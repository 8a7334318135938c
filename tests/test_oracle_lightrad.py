"""CPU checks of the light/rad goldens, the restated equalize_adapthist (tests/golden/clahe_restated.py) and the host bookkeeping of
pylinac_b200/planar_imaging.py.

scikit-image is not installed, so the CLAHE restatement is UNPINNED: these tests check its own properties (a constant image, no
clipping, a single contextual region computed by hand, the output range), not agreement with scikit-image."""
import hashlib
import os

import numpy as np
import pytest

from oracle.refstub import REFERENCE_ROOT
from pylinac_b200 import _native as nat
from pylinac_b200 import planar_imaging as pi
from pylinac_b200.contrib.quasar import QuasarLightRadScaling
from tests.golden import clahe_restated as sk
from tests.golden.lightrad_cases import CASES, lightrad_case

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "lightrad_golden.npz"))
CLASSES = {"StandardImagingFC2": pi.StandardImagingFC2, "IMTLRad": pi.IMTLRad, "DoselabRLf": pi.DoselabRLf, "IsoAlign": pi.IsoAlign,
           "SNCFSQA": pi.SNCFSQA, "QuasarLightRadScaling": QuasarLightRadScaling}


def _golden(name):
    return {k.split("/", 1)[1]: G[k] for k in G.files if k.startswith(name + "/")}


@pytest.mark.parametrize("name", CASES)
def test_lightrad_case_inputs_reproduce(name):
    c = lightrad_case(name)
    assert hashlib.sha1(c["frame"].tobytes()).digest() == _golden(name)["input_sha1"].tobytes()


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE_ROOT, "pylinac")), reason="needs the reference source tree")
@pytest.mark.parametrize("name", ["fc2_10_near", "fc2_mismatch", "quasar", "snc", "fc2_k1", "fc2_k64", "fc2_odd_small"])
def test_lightrad_golden_reproduces_from_reference(name):
    import warnings

    from tests.golden.make_lightrad_golden import reference_lightrad

    c = lightrad_case(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = reference_lightrad(c["cls"], c["frame"], c["dpmm"], c["ctor"], c["analyze"])
    g = _golden(name)
    for k, v in ref.items():
        assert np.array_equal(np.asarray(v), g[k]), (name, k)


# ------------------------------------------------------------------------------------------- restated CLAHE
def test_clahe_constant_image():
    """one bin everywhere: every region has the same map, so every pixel is that map value, or one count below it where the float32
    sum of the four bilinear weights rounds under 1 before the cast back to integers"""
    img14 = np.full((40, 50), 9000, np.uint16)
    u = sk.clahe_u14(img14, 10).astype(int)
    assert u.max() - u.min() <= 1
    out = sk.equalize_adapthist(np.full((40, 50), 0.3), kernel_size=10)
    assert out.shape == (40, 50) and set(np.unique(out)) <= {0.0, 1.0}


def test_clahe_output_range():
    rng = np.random.default_rng(3)
    img = rng.random((61, 47))
    out = sk.equalize_adapthist(img, kernel_size=8)
    assert out.min() == 0.0 and out.max() == 1.0
    u16 = (rng.random((33, 29)) * 65535).astype(np.uint16)
    out = sk.equalize_adapthist(u16, kernel_size=7)
    assert out.min() >= 0.0 and out.max() <= 1.0


def test_clahe_no_clipping_keeps_histograms():
    """clip_limit=1: the clip count is k * k, which no bin of a k x k region exceeds, so clip_histogram returns it unchanged"""
    rng = np.random.default_rng(5)
    h = np.bincount(rng.integers(0, 256, 100), minlength=256)
    assert np.array_equal(sk.clip_histogram(h.copy(), 100), h)


def test_clahe_single_region_is_its_clipped_equalisation():
    """a k x k image with kernel k has one contextual region: every pixel takes that region's map of its bin (the float32 sum of the
    four equal maps may round one count down before the cast back to integers)"""
    k = 12
    rng = np.random.default_rng(7)
    img14 = rng.integers(0, sk.NR_OF_GRAY, (k, k)).astype(np.uint16)
    bins = img14 // (1 + sk.NR_OF_GRAY // 256)
    hist = np.bincount(bins.ravel(), minlength=256)
    clim = int(max(0.01 * k * k, 1))
    # clip_histogram by hand: clip at clim, then hand out the excess one count per bin below clim, left to right, repeatedly
    excess = int(np.sum(np.maximum(hist - clim, 0)))
    hist = np.minimum(hist, clim)
    while excess > 0:
        under = np.flatnonzero(hist < clim)
        if len(under) == 0:
            break
        step = max(1, len(under) // excess)
        picked = [b for b in range(0, 256, step) if hist[b] < clim]
        hist[picked] += 1
        excess -= len(picked)
    cdf = np.cumsum(hist)
    mapping = np.minimum(cdf * ((sk.NR_OF_GRAY - 1) / (k * k)), sk.NR_OF_GRAY - 1).astype(int)
    out = sk.clahe_u14(img14, k).astype(int)
    expected = mapping[bins]
    assert np.all((out == expected) | (out == expected - 1))


# ------------------------------------------------------------------------------------------- host bookkeeping
def test_bb_sets_match_the_reference_classes():
    assert list(pi.StandardImagingFC2._device_bb_set()[0]) == ["TL", "BL", "TR", "BR"]
    assert pi.StandardImagingFC2._device_bb_set()[1] == 1
    assert pi.StandardImagingFC2.bb_positions_15x15["BR"] == [65, 65]
    assert list(pi.IMTLRad._device_bb_set()[0]) == ["Center"] and pi.IMTLRad.bb_size_mm == 3
    assert pi.DoselabRLf._device_bb_set()[0]["TL"] == [-17, -45]
    assert list(pi.IsoAlign._device_bb_set()[0]) == ["Center", "Top", "Bottom", "Left", "Right"]
    assert pi.SNCFSQA._device_bb_set()[0] == {"TR": [40, -40]}
    assert QuasarLightRadScaling._device_bb_set()[1] == 2


def test_lightrad_params_kernel_size():
    p = pi._params(pi.StandardImagingFC2, 2.9761904761904763, True, False, 50, 10, 2.0)
    assert p.clahe_kernel == int(round(4 / 2 * 2.9761904761904763 * 2.0)) == 12
    assert p.nbb == 4 and p.set_mode == 1 and p.scaling == 0
    q = pi._params(QuasarLightRadScaling, 2.5, True, False, 50, 10, 2.0)
    assert q.scaling == 1 and q.quasar_offset_mm == 11 and q.strip_width_mm == 20


def _row_from_golden(name, g, phantom):
    r = np.zeros(1, nat.LR_RESULT_DTYPE)[0]
    r["field_center_x"], r["field_center_y"] = g["field_center"]
    r["field_width_x_mm"], r["field_width_y_mm"] = g["field_width"]
    nbb = len(g["bb_keys"]) - (1 if phantom._virtual_center else 0)
    r["bb_x"][:nbb] = g["bb_centers"][:nbb, 0]
    r["bb_y"][:nbb] = g["bb_centers"][:nbb, 1]
    r["large_set"] = int(str(g["bb_keys"][0]) == "TL" and abs(g["bb_centers"][0, 0] - g["epid_center"][0]) > 50 * g["dpmm"])
    return r


@pytest.mark.parametrize("name", [n for n in CASES if "error_type" not in _golden(n)])
def test_host_bookkeeping_from_golden_points(name):
    """virtual centre, BB centroid, offsets, near-edge decisions and results() text from the reference's own points"""
    c = lightrad_case(name)
    g = _golden(name)
    phantom = CLASSES[c["cls"]]
    fr = pi.LightRadFrame(_row_from_golden(name, g, phantom), phantom, float(g["dpmm"]), c["frame"].shape)
    np.testing.assert_allclose([[p.x, p.y] for p in fr.bb_centers.values()], g["bb_centers"], rtol=0, atol=1e-9)
    assert list(fr.bb_centers) == [str(k) for k in g["bb_keys"]]
    np.testing.assert_allclose([fr.bb_center.x, fr.bb_center.y], g["bb_center"], rtol=0, atol=1e-9)
    np.testing.assert_allclose([fr.epid_center.x, fr.epid_center.y], g["epid_center"], rtol=0, atol=0)
    np.testing.assert_allclose([fr.field_bb_offset_mm.x, fr.field_bb_offset_mm.y], g["field_bb_offset_mm"], rtol=0, atol=1e-12)
    np.testing.assert_allclose([fr.field_epid_offset_mm.x, fr.field_epid_offset_mm.y], g["field_epid_offset_mm"], rtol=0, atol=1e-12)
    # near-edge decisions from the reference's widths and BB set
    ph = phantom.__new__(phantom)
    ph.bb_edge_threshold_mm = c["analyze"].get("bb_edge_threshold_mm", 10)
    ph.field_width_x, ph.field_width_y = g["field_width"]
    if phantom is QuasarLightRadScaling:
        fx, fy = g["field_width"] / 2
        positions = [(-fx + 11, -fy + 11), (-fx + 11, fy - 11), (fx - 11, fy - 11), (fx - 11, -fy + 11)]
    else:
        bb_set = phantom._device_bb_set()[0]
        if phantom is pi.StandardImagingFC2 and g["field_width"][0] > 140:
            bb_set = phantom.bb_positions_15x15
        positions = list(bb_set.values())
    assert [ph._is_bb_near_edge(p) for p in positions] == list(g["near_edge"])
    # results() text, except the file line
    ph.image = type("Img", (), {"dpmm": float(g["dpmm"]), "path": ""})()
    ph.field_center, ph.bb_center, ph.epid_center = fr.field_center, fr.bb_center, fr.epid_center
    lines = ph.results(as_list=True)
    ref = [str(s) for s in g["results"]]
    assert lines[0] == ref[0] and lines[2:] == ref[2:]


def test_mismatch_message_matches_reference():
    g = _golden("fc2_mismatch")
    r = np.zeros(1, nat.LR_RESULT_DTYPE)[0]
    r["status"] = 2
    r["field_width_x_mm"], r["field_width_y_mm"] = 100.0, 150.0
    fr = pi.LightRadFrame(r, pi.StandardImagingFC2, 3.0, (1280, 1280))
    with pytest.raises(ValueError) as ei:
        fr.raise_for_status()
    assert str(ei.value).split("Detected")[0] == str(g["error_message"]).split("Detected")[0]
