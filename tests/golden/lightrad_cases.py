"""Seeded synthetic light/radiation-field coincidence frames (planar_imaging.StandardImagingFC2 and its subclasses, Quasar).

A frame is an open rectangular field with erf penumbrae on a low background, attenuating BBs (dark disks with soft edges) at the
phantom's nominal positions, and gaussian noise.  Every case keeps its true field edges and BB centres (pixels, image coordinates),
so results can be checked against the geometry as well as against the reference.
"""
from __future__ import annotations

import math

import numpy as np

SI_10 = [(-40, -40), (-40, 40), (40, -40), (40, 40)]
SI_15 = [(-65, -65), (-65, 65), (65, -65), (65, 65)]
DOSELAB = [(-17, -45), (-45, 17), (45, -17), (17, 45)]
ISOALIGN = [(0, 0), (0, -25), (0, 25), (-25, 0), (25, 0)]
QUASAR_SCALING = [(0, 0), (-10, -8), (10, -8), (-10, 8), (10, 8)]

# name: (class, (h, w), pixel mm, field x / y mm, field centre offset mm (x, y), bb offset mm (x, y), bb diameter, bbs, seed,
#        inverted raw frame, analyze kwargs, ctor kwargs)
_C = {
    "fc2_10_near": ("StandardImagingFC2", (1280, 1280), 0.336, 99.6, 99.4, (0.3, -0.2), (0.0, 0.0), 4, SI_10, 1, False, {}, {}),
    "fc2_10_far": ("StandardImagingFC2", (1280, 1280), 0.336, 101.0, 100.8, (-0.4, 0.3), (0.2, 0.1), 4, SI_10, 2, False, {}, {}),
    "fc2_15": ("StandardImagingFC2", (1280, 1280), 0.336, 150.5, 150.2, (0.5, 0.4), (-0.3, 0.2), 4, SI_15, 3, False, {}, {}),
    "fc2_15_near": ("StandardImagingFC2", (1280, 1280), 0.336, 149.2, 149.5, (0.1, 0.2), (0.0, -0.2), 4, SI_15, 4, False, {}, {}),
    "fc2_small_near": ("StandardImagingFC2", (768, 1024), 0.392, 99.2, 99.7, (-0.6, 0.4), (0.25, -0.15), 4, SI_10, 5, False, {}, {}),
    "fc2_small_far": ("StandardImagingFC2", (768, 1024), 0.392, 100.6, 100.9, (0.2, -0.5), (-0.2, 0.3), 4, SI_10, 6, False, {}, {}),
    "fc2_inverted": ("StandardImagingFC2", (1280, 1280), 0.336, 100.7, 100.9, (0.2, 0.2), (0.1, 0.0), 4, SI_10, 7, True, {}, {}),
    "fc2_invert_kw": ("StandardImagingFC2", (1280, 1280), 0.336, 101.2, 101.0, (0.0, 0.3), (0.0, 0.2), 4, SI_10, 8, True,
                      {"invert": True}, {}),
    "fc2_no_normalize": ("StandardImagingFC2", (1280, 1280), 0.336, 99.5, 99.8, (0.2, -0.3), (0.1, 0.1), 4, SI_10, 9, False, {},
                         {"normalize": False}),
    "fc2_no_normalize_far": ("StandardImagingFC2", (768, 1024), 0.392, 101.5, 101.1, (0.2, -0.3), (0.1, 0.1), 4, SI_10, 10, False,
                             {}, {"normalize": False}),
    "fc2_threshold": ("StandardImagingFC2", (1280, 1280), 0.336, 101.0, 100.6, (0.1, 0.1), (0.0, 0.0), 4, SI_10, 11, False,
                      {"bb_edge_threshold_mm": 5, "kernel_size_multiplier": 1.5}, {}),
    "fc2_mismatch": ("StandardImagingFC2", (1280, 1280), 0.336, 100.0, 150.0, (0.0, 0.0), (0.0, 0.0), 4, SI_10, 12, False, {}, {}),
    "fc2_no_bb": ("StandardImagingFC2", (1280, 1280), 0.336, 101.0, 101.0, (0.0, 0.0), (0.0, 0.0), 4, [], 13, False, {}, {}),
    "imt": ("IMTLRad", (1280, 1280), 0.336, 100.5, 100.3, (0.3, 0.1), (0.2, -0.1), 3, [(0, 0)], 14, False, {}, {}),
    "doselab": ("DoselabRLf", (1280, 1280), 0.336, 100.8, 100.4, (-0.2, 0.3), (0.1, 0.2), 4, DOSELAB, 15, False, {}, {}),
    "doselab_near": ("DoselabRLf", (1280, 1280), 0.336, 99.0, 99.3, (0.2, 0.1), (0.0, 0.1), 4, DOSELAB, 16, False, {}, {}),
    "isoalign": ("IsoAlign", (1280, 1280), 0.336, 100.4, 100.2, (0.1, -0.2), (-0.1, 0.2), 4, ISOALIGN, 17, False, {}, {}),
    "snc": ("SNCFSQA", (1280, 1280), 0.336, 150.6, 150.3, (0.3, 0.2), (0.2, 0.2), 4, [(40, -40)], 18, False, {}, {}),
    "quasar": ("QuasarLightRadScaling", (1280, 1280), 0.336, 150.3, 150.8, (0.2, -0.1), (0.0, 0.0), 5, None, 19, False, {}, {}),
}


def multiplier_for(k: int, bb_size_mm: float, pixel_mm: float) -> float:
    """the kernel_size_multiplier that makes the reference's CLAHE kernel int(round(bb_radius_px * multiplier)) equal k"""
    return k / (bb_size_mm / 2 / pixel_mm)


def _k(k, pixel_mm, bb_size_mm=4):
    return {"kernel_size_multiplier": multiplier_for(k, bb_size_mm, pixel_mm)}


# kernel sizes and frame shapes beyond the default k = int(round(bb_radius_px * 2)) in {9, 10, 12}: clip limits above 1, kernels that
# divide the frame, partial tiles of odd frames, and k = 1, where every contextual region is one pixel
_C.update({
    "fc2_k1": ("StandardImagingFC2", (1280, 1280), 0.336, 99.6, 99.4, (0.3, -0.2), (0.0, 0.0), 4, SI_10, 20, False, _k(1, 0.336), {}),
    "fc2_k32": ("StandardImagingFC2", (1280, 1280), 0.336, 99.5, 99.7, (-0.2, 0.1), (0.1, -0.1), 4, SI_10, 21, False, _k(32, 0.336),
                {}),
    "fc2_k64": ("StandardImagingFC2", (1280, 1280), 0.336, 99.3, 99.6, (0.1, 0.3), (-0.1, 0.1), 4, SI_10, 22, False, _k(64, 0.336),
                {}),
    "fc2_k160": ("StandardImagingFC2", (1280, 1280), 0.336, 99.7, 99.5, (0.2, 0.2), (0.0, 0.1), 4, SI_10, 23, False, _k(160, 0.336),
                 {}),
    "fc2_1190_near": ("StandardImagingFC2", (1190, 1190), 0.336, 99.4, 99.6, (-0.3, 0.2), (0.1, 0.0), 4, SI_10, 24, False, {}, {}),
    "fc2_odd_small": ("StandardImagingFC2", (241, 199), 0.6, 99.5, 99.3, (0.2, -0.3), (0.1, 0.2), 4, SI_10, 25, False, {}, {}),
    "fc2_no_normalize_k64": ("StandardImagingFC2", (1280, 1280), 0.336, 99.6, 99.2, (0.1, -0.1), (0.0, 0.2), 4, SI_10, 26, False,
                             _k(64, 0.336), {"normalize": False}),
    "fc2_inverted_k48": ("StandardImagingFC2", (1280, 1280), 0.336, 99.4, 99.5, (-0.1, 0.2), (0.2, 0.0), 4, SI_10, 27, True,
                         _k(48, 0.336), {}),
})
CASES = list(_C)


def _bbs_for(cls, fwx, fwy, bbs):
    if cls == "QuasarLightRadScaling":
        fx, fy = fwx / 2, fwy / 2
        corners = [(-fx + 11, -fy + 11), (-fx + 11, fy - 11), (fx - 11, fy - 11), (fx - 11, -fy + 11)]
        return corners + QUASAR_SCALING
    return bbs


def _erf_edge(x, lo, hi, sigma):
    s = sigma * math.sqrt(2.0)
    from scipy.special import erf

    return 0.5 * (erf((x - lo) / s) - erf((x - hi) / s))


def synth_frame(cls, shape, pixel_mm, field_mm, field_offset_mm=(0.0, 0.0), bb_offset_mm=(0.0, 0.0), bb_diameter_mm=4, bbs=SI_10,
                seed=0, inverted=False):
    """-> (frame uint16 [h, w], truth) for one synthetic light/rad frame: field_mm = (x, y) widths, bbs = nominal BB positions (mm)
    (ignored for Quasar, whose corner BBs follow the field)"""
    h, w = shape
    ps = pixel_mm
    fwx, fwy = field_mm
    fcx, fcy = field_offset_mm
    box, boy = bb_offset_mm
    bbd = bb_diameter_mm
    rng = np.random.default_rng(1000 + seed)
    dpmm = 1.0 / ps
    # pixel coordinates of the image centre as the reference places the nominal BBs (shape / 2)
    cx, cy = w / 2 + fcx * dpmm, h / 2 + fcy * dpmm
    xs = np.arange(w, dtype=np.float64)
    ys = np.arange(h, dtype=np.float64)
    sig = 2.0 * dpmm              # 2 mm penumbra sigma
    px = _erf_edge(xs, cx - fwx / 2 * dpmm, cx + fwx / 2 * dpmm, sig)
    py = _erf_edge(ys, cy - fwy / 2 * dpmm, cy + fwy / 2 * dpmm, sig)
    img = 1500.0 + 28000.0 * np.outer(py, px)
    bb_px = []
    r = bbd / 2 * dpmm
    yy, xx = np.mgrid[0:h, 0:w]
    for bx, by in _bbs_for(cls, fwx, fwy, bbs):
        x0, y0 = w / 2 + (bx + box) * dpmm, h / 2 + (by + boy) * dpmm
        x0 += rng.uniform(-0.3, 0.3)
        y0 += rng.uniform(-0.3, 0.3)
        bb_px.append((x0, y0))
        y_lo, y_hi = int(max(y0 - r - 4, 0)), int(min(y0 + r + 5, h))
        x_lo, x_hi = int(max(x0 - r - 4, 0)), int(min(x0 + r + 5, w))
        d = np.hypot(xx[y_lo:y_hi, x_lo:x_hi] - x0, yy[y_lo:y_hi, x_lo:x_hi] - y0)
        att = 1.0 - 0.6 * np.clip(r + 0.5 - d, 0.0, 1.0)
        img[y_lo:y_hi, x_lo:x_hi] *= att
    img += rng.normal(0.0, 40.0, img.shape)
    if inverted:
        img = 32000.0 - img
    frame = np.clip(np.rint(img), 0, 65535).astype(np.uint16)
    truth = {
        "field_edges_px": np.array([cx - fwx / 2 * dpmm, cx + fwx / 2 * dpmm, cy - fwy / 2 * dpmm, cy + fwy / 2 * dpmm]),
        "field_size_mm": np.array([fwx, fwy]),
        "field_center_px": np.array([cx, cy]),
        "bb_px": np.array(bb_px, dtype=np.float64).reshape(-1, 2),
    }
    return frame, truth


def lightrad_case(name):
    """-> dict(cls, frame uint16 [h, w], dpmm, ctor, analyze, truth) for one named case"""
    cls, shape, ps, fwx, fwy, fc, bo, bbd, bbs, seed, inverted, ak, ck = _C[name]
    frame, truth = synth_frame(cls, shape, ps, (fwx, fwy), fc, bo, bbd, bbs, seed, inverted)
    return {"cls": cls, "frame": frame, "dpmm": 1.0 / ps, "ctor": dict(ck), "analyze": dict(ak), "truth": truth}
