"""The light / rad pixel stages (csrc/lightrad.cu) read back with epid_lightrad_stages and compared pixel for pixel with a plain
reference built from numpy, scipy and the restated equalize_adapthist (tests/golden/clahe_restated.py, whose parity with scikit-image
is UNPINNED).

The reference follows the reference's own float pipeline: ground, normalize, invert() (check_inversion, then the `invert` argument),
median_filter on the float image, img_as_uint, the 14-bit rescale and the contextual-region CLAHE.  The device works on the integer
frame through an affine map (DESIGN 2.1), so equal planes here also test that argument.

The BB centres of test_gpu_lightrad.py depend only on the equalised pixels inside each BB window.  These tests check every pixel of
every stage, at kernel sizes from 1 to just below the frame edge (every clip regime of clip_histogram, kernels that divide the frame)
and at frame shapes with partial tiles."""
import numpy as np
import pytest
from scipy import ndimage

from pylinac_b200 import _native as nat
from pylinac_b200 import planar_imaging as pi
from pylinac_b200.contrib.quasar import QuasarLightRadScaling
from tests.golden import clahe_restated as sk
from tests.golden.lightrad_cases import ISOALIGN, SI_10, lightrad_case, multiplier_for, synth_frame

FC2 = pi.StandardImagingFC2
NEAR_10 = (99.6, 99.4)          # a 10 x 10 field whose corner BBs lie within 10 mm of the field edge

# id: (class, (h, w), pixel mm, field mm, k, inverted raw frame, ctor kwargs, analyze kwargs)
_S = {
    "1280_k9": (FC2, (1280, 1280), 0.336, NEAR_10, 9, False, {}, {}),
    "1280_k12": (FC2, (1280, 1280), 0.336, NEAR_10, 12, False, {}, {}),
    "1280_k31": (FC2, (1280, 1280), 0.336, NEAR_10, 31, False, {}, {}),
    "1280_k32": (FC2, (1280, 1280), 0.336, NEAR_10, 32, False, {}, {}),
    "1280_k33": (FC2, (1280, 1280), 0.336, NEAR_10, 33, False, {}, {}),
    "1280_k64": (FC2, (1280, 1280), 0.336, NEAR_10, 64, False, {}, {}),
    "1280_k100": (FC2, (1280, 1280), 0.336, NEAR_10, 100, False, {}, {}),
    "1280_k160": (FC2, (1280, 1280), 0.336, NEAR_10, 160, False, {}, {}),
    "241x199_k1": (FC2, (241, 199), 0.6, NEAR_10, 1, False, {}, {}),
    "241x199_k2": (FC2, (241, 199), 0.6, NEAR_10, 2, False, {}, {}),
    "241x199_k3": (FC2, (241, 199), 0.6, NEAR_10, 3, False, {}, {}),
    "241x199_k9": (FC2, (241, 199), 0.6, NEAR_10, 9, False, {}, {}),
    "241x199_k198": (FC2, (241, 199), 0.6, NEAR_10, 198, False, {}, {}),
    "768x1024_k12": (FC2, (768, 1024), 0.392, NEAR_10, 12, False, {}, {}),
    "768x1024_k33": (FC2, (768, 1024), 0.392, NEAR_10, 33, False, {}, {}),
    "768x1024_k64": (FC2, (768, 1024), 0.392, NEAR_10, 64, False, {}, {}),
    "1024x768_k12": (FC2, (1024, 768), 0.392, NEAR_10, 12, False, {}, {}),
    "1024x768_k32": (FC2, (1024, 768), 0.392, NEAR_10, 32, False, {}, {}),
    "1024x768_k100": (FC2, (1024, 768), 0.392, NEAR_10, 100, False, {}, {}),
    "1190_k12": (FC2, (1190, 1190), 0.336, NEAR_10, 12, False, {}, {}),
    "1190_k32": (FC2, (1190, 1190), 0.336, NEAR_10, 32, False, {}, {}),
    "1190_k64": (FC2, (1190, 1190), 0.336, NEAR_10, 64, False, {}, {}),
    "inverted_raw_k48": (FC2, (1280, 1280), 0.336, NEAR_10, 48, True, {}, {}),
    "invert_kw_k32": (FC2, (1280, 1280), 0.336, NEAR_10, 32, True, {}, {"invert": True}),
    "invert_kw_upright_k12": (FC2, (1280, 1280), 0.336, NEAR_10, 12, False, {}, {"invert": True}),
    "no_normalize_k64": (FC2, (768, 1024), 0.392, NEAR_10, 64, False, {"normalize": False}, {}),
    "no_normalize_inverted_k12": (FC2, (1280, 1280), 0.336, NEAR_10, 12, True, {"normalize": False}, {}),
    "isoalign_k33": (pi.IsoAlign, (1280, 1280), 0.336, (100.4, 100.2), 33, False, {}, {"bb_edge_threshold_mm": 26}),
    "quasar_k40": (QuasarLightRadScaling, (1280, 1280), 0.336, (150.3, 150.8), 40, False, {}, {"bb_edge_threshold_mm": 12}),
}


def _stage_case(name):
    cls, shape, ps, field, k, inverted, ctor, ak = _S[name]
    bbs = ISOALIGN if cls is pi.IsoAlign else SI_10
    frame, _ = synth_frame(cls.__name__, shape, ps, field, seed=100 + list(_S).index(name), bbs=bbs, bb_diameter_mm=cls.bb_size_mm,
                           inverted=inverted)
    normalize = ctor.get("normalize", True)
    invert = ak.get("invert", False)
    p = pi._params(cls, 1.0 / ps, normalize, invert, 50, ak.get("bb_edge_threshold_mm", 10), multiplier_for(k, cls.bb_size_mm, ps))
    assert p.clahe_kernel == k
    return frame, p, normalize, invert, k


# ------------------------------------------------------------------------------------------- the plain reference
def _corners(a):
    return [a[1:21, 1:21], a[1:21, -21:-1], a[-21:-1, 1:21], a[-21:-1, -21:-1]]


def _invert(a):
    return -a + a.max() + a.min()            # core/array_utils.invert, in the image's own dtype


def reference_stages(frame, normalize, invert, k):
    """the reference's float pipeline up to the second median of the equalised image"""
    img = frame.copy()
    if normalize:
        img = img - img.min()                # ground (uint16, exact)
        img = img / img.max()                # normalize -> float64
    checked = bool(np.mean(_corners(img)) > np.mean(img.flatten()))
    if checked:
        img = _invert(img)
    if invert:
        img = _invert(img)
    filt = ndimage.median_filter(img, size=3)
    u16 = sk._img_as_uint(filt)
    img14 = np.round(sk._rescale_intensity(u16, (0, sk.NR_OF_GRAY - 1))).astype(np.uint16)
    eq = sk.clahe_u14(img14, k)
    return {"checked": checked, "inv": checked ^ invert, "u16": u16, "eq": eq, "eqf": ndimage.median_filter(eq, size=3)}


def _device_u16(T, mn, mx, inv, normalize):
    """img_as_uint of the once-filtered image from the device's median T of the mapped integer frame (DESIGN 2.1)"""
    T = T.astype(np.int64)
    if not normalize:
        return T.astype(np.uint16)
    D = float(mx - mn)
    a = -((mx - T) / D) + 1.0 + 0.0 if inv else (T - mn) / D
    return np.rint(a * 65535.0).astype(np.uint16)


def _assert_planes_equal(dev, ref, what):
    assert dev.shape == ref.shape, (what, dev.shape, ref.shape)
    bad = np.argwhere(dev != ref)
    if len(bad):
        d = dev.astype(np.int64) - ref.astype(np.int64)
        first = [(int(y), int(x), int(dev[y, x]), int(ref[y, x])) for y, x in bad[:8]]
        raise AssertionError(f"{what}: {len(bad)} of {dev.size} pixels differ, max |diff| {int(np.abs(d).max())}, "
                             f"rows {int(bad[:, 0].min())}..{int(bad[:, 0].max())}, cols {int(bad[:, 1].min())}..{int(bad[:, 1].max())}, "
                             f"first (y, x, device, reference) {first}")


def _stages(frames, p):
    return nat.lightrad_stages(nat.Context.default(), frames, p)


# ------------------------------------------------------------------------------------------- every stage of one frame
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_S))
def test_lightrad_stages_match_reference(name):
    frame, p, normalize, invert, k = _stage_case(name)
    out = _stages(frame[None], p)
    info = {f: int(v[0]) for f, v in out["info"].items()}
    ref = reference_stages(frame, normalize, invert, k)
    raw = frame.astype(np.int64)
    # front: raw range, exact sum, corner boxes, check_inversion of the image the reference sees
    assert info["mn"] == raw.min() and info["mx"] == raw.max()
    assert info["sum"] == raw.sum()
    assert info["corner"] == sum(int(c.sum()) for c in _corners(raw))
    assert info["checked"] == ref["checked"] and info["inv"] == ref["inv"]
    assert info["near_mask"] != 0, "the case must reach the equalisation"
    # first median of the mapped integer frame, and its 16-bit value as the float pipeline has it
    mapped = info["mx"] + info["mn"] - raw if info["inv"] else raw
    T = out["filtered"][0]
    _assert_planes_equal(T, ndimage.median_filter(mapped, size=3).astype(np.uint16), "filtered")
    _assert_planes_equal(_device_u16(T, info["mn"], info["mx"], info["inv"], normalize), ref["u16"], "img_as_uint(filtered)")
    assert (info["fmn"], info["fmx"]) == (int(T.min()), int(T.max()))
    # equalize_adapthist up to the cast back to integers, then the second median
    eq = out["equalised"][0]
    _assert_planes_equal(eq, ref["eq"], f"equalised (k={k})")
    assert (info["umin"], info["umax"]) == (int(ref["eq"].min()), int(ref["eq"].max()))
    _assert_planes_equal(out["equalised_filtered"][0], ref["eqf"], f"equalised_filtered (k={k})")
    # the read-back runs the production launch sequence
    assert out["results"].tobytes() == nat.lightrad_analyze(nat.Context.default(), frame[None], p).tobytes()


def test_lightrad_stages_cover_every_clip_regime():
    """the matrix above reaches clip limit 1 without excess redistribution rounds, limits above 1 with bin_incr > 0, and the mid
    branch of clip_histogram (bins lifted to between upper and the limit); counted on the restated operator's own histograms"""
    seen = set()
    for name in ("1280_k12", "1280_k32", "1280_k64"):
        frame, p, normalize, invert, k = _stage_case(name)
        ref = reference_stages(frame, normalize, invert, k)
        img14 = np.round(sk._rescale_intensity(ref["u16"], (0, sk.NR_OF_GRAY - 1))).astype(np.uint16)
        ps = k // 2
        pe = [(k - s % k) % k + int(np.ceil(k / 2.0)) for s in img14.shape]
        img = np.pad(img14, [[ps, pe[0]], [ps, pe[1]]], mode="reflect") // (1 + sk.NR_OF_GRAY // 256)
        nh = [s // k - 1 for s in img.shape]
        clim = int(max(0.01 * k * k, 1))
        for ti in range(0, nh[0], 7):
            for tj in range(0, nh[1], 7):
                h = np.bincount(img[ps + ti * k:ps + (ti + 1) * k, ps + tj * k:ps + (tj + 1) * k].ravel(), minlength=256)
                n_excess = int(np.maximum(h - clim, 0).sum())
                incr = n_excess // 256
                hc = np.minimum(h, clim)
                hc[hc < clim - incr] += incr
                seen.add(("limit1" if clim == 1 else "limit>1", incr > 0, bool(np.any((hc >= clim - incr) & (hc < clim)) and incr > 0)))
    assert ("limit1", False, False) in seen
    assert any(s[0] == "limit>1" and s[1] for s in seen)
    assert any(s[2] for s in seen), seen


# ------------------------------------------------------------------------------------------- batches of more than one chunk
@pytest.mark.gpu
def test_lightrad_stages_batch_equals_single_frames():
    """70 frames of one shape (more than one 64-frame chunk), near-edge and not, inverted and not: every frame's planes and
    accumulators equal those of its one-frame call"""
    names = ["fc2_10_near", "fc2_10_far", "fc2_inverted", "fc2_15_near", "fc2_k32", "fc2_no_bb"]
    base = [lightrad_case(n)["frame"] for n in names]
    order = [i % len(names) for i in range(70)]
    frames = np.stack([base[i] for i in order])
    p = pi._params(FC2, lightrad_case(names[0])["dpmm"], True, False, 50, 10, 2.0)
    batch = _stages(frames, p)
    singles = [_stages(f[None], p) for f in base]
    assert any(s["info"]["near_mask"][0] for s in singles) and not all(s["info"]["near_mask"][0] for s in singles)
    for i, j in enumerate(order):
        one = singles[j]
        near = one["info"]["near_mask"][0] != 0
        assert batch["results"][i].tobytes() == one["results"][0].tobytes(), (i, names[j])
        fields = nat.LR_INFO_FIELDS if near else nat.LR_INFO_FIELDS[:7]
        assert [int(batch["info"][f][i]) for f in fields] == [int(one["info"][f][0]) for f in fields], (i, names[j])
        assert np.array_equal(batch["filtered"][i], one["filtered"][0]), (i, names[j])
        if near:
            assert np.array_equal(batch["equalised"][i], one["equalised"][0]), (i, names[j])
            assert np.array_equal(batch["equalised_filtered"][i], one["equalised_filtered"][0]), (i, names[j])
