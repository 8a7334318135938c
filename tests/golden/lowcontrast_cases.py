"""Seeded arrays and settings for the LowContrastDiskROI / core.contrast / low-contrast batch goldens (make_lowcontrast_golden.py) and the
tests that check them.

ROI_CASES: name -> (array builder, [roi spec, ...]).  A roi spec is (centre row, centre col, radius, LowContrastDiskROI keyword
arguments); every ROI records its statistics, contrasts, pass flags, as_dict and the percentiles of Q.
BATCH_CASES: name -> (frames builder, geometry, settings keyword arguments).  The reference's ImagePhantomBase stage runs on each frame.
CONTRAST_CASES: direct calls of the core.contrast functions, (function name, args)."""
from __future__ import annotations

import numpy as np

# q = 100.5 is out of range; 99.99999999 rounds to 1.0 in float32 (in range there) but not in float64
Q = [0, 1, 2.5, 50, 99, 99.5, 100, 99.99999999, 100.5]

METHODS = ["Michelson", "Weber", "Ratio", "Root Mean Square", "Difference", "michelson", "Nonsense"]


def _noise(seed: int, shape, dtype, nan: bool = False) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if np.issubdtype(dtype, np.floating):
        a = (rng.standard_normal(shape) * 300 + 1000).astype(dtype)
        if nan:
            a[20, 30] = np.nan
        return a
    info = np.iinfo(dtype)
    lo, hi = max(int(info.min), -30000), min(int(info.max), 30000)
    return rng.integers(lo, hi + 1, shape).astype(dtype)


def _unit(seed: int) -> np.ndarray:
    """values in [0, 1] for the RMS contrast"""
    return np.random.default_rng(seed).uniform(0.2, 0.8, (48, 64))


def _flat(value, dtype) -> np.ndarray:
    """a constant array: the std is 0"""
    return np.full((48, 64), value, dtype)


_BASE = {"contrast_reference": 900.0, "contrast_threshold": 0.05, "cnr_threshold": 2.0}
_GEOM = [
    (20.3, 30.1, 6.2, _BASE),                                                   # odd count, holds the NaN of the NaN cases
    (24.0, 24.0, 2.0, _BASE),                                                   # 12 pixels: an even count
    (10.0, 40.0, 1.0, _BASE),                                                   # one pixel
    (-3.5, 10.2, 6.3, _BASE),                                                   # across the top edge: negative rows wrap
    (20.0, -2.7, 5.0, _BASE),                                                   # across the left edge
    (12.5, 40.5, 0.3, _BASE),                                                   # empty
    (46.0, 60.0, 5.0, _BASE),                                                   # beyond the frame: IndexError
    (30.0, 30.0, 9.7, {**_BASE, "contrast_reference": None}),
    (30.0, 30.0, 9.7, {**_BASE, "contrast_reference": 0.0}),
    (30.0, 30.0, 9.7, {**_BASE, "contrast_reference": 0}),                      # a Python int zero
    (30.0, 30.0, 9.7, {**_BASE, "contrast_reference": -250.0}),
    (30.0, 30.0, 9.7, {**_BASE, "contrast_threshold": None, "cnr_threshold": None}),
    (30.0, 30.0, 9.7, {**_BASE, "visibility_threshold": 1e9}),
] + [(22.2, 33.3, 7.5, {**_BASE, "contrast_method": m}) for m in METHODS]

ROI_CASES = {
    "uint8": (lambda: _noise(31, (48, 64), np.uint8), _GEOM),
    "uint16": (lambda: _noise(32, (48, 64), np.uint16), _GEOM),
    "int16": (lambda: _noise(33, (48, 64), np.int16), _GEOM),       # values of both signs: b - a wraps in int16
    "int32": (lambda: _noise(34, (48, 64), np.int32), _GEOM),
    "float32": (lambda: _noise(35, (48, 64), np.float32), _GEOM),
    "float64": (lambda: _noise(36, (48, 64), np.float64), _GEOM),
    "float32_nan": (lambda: _noise(37, (48, 64), np.float32, nan=True), _GEOM[:3]),
    "float64_nan": (lambda: _noise(38, (48, 64), np.float64, nan=True), _GEOM[:3]),
    "flat_uint16": (lambda: _flat(1000, np.uint16), _GEOM[:3] + _GEOM[7:12]),
    "flat_float64_zero": (lambda: _flat(0.0, np.float64), _GEOM[:3] + _GEOM[7:12]),
    # np.percentile of bool pixels raises TypeError (an empty disk IndexError); the statistics are numpy's of bool arrays
    "bool": (lambda: _noise(40, (48, 64), np.uint8) > 128, _GEOM[:7]),
    "unit_rms": (lambda: _unit(39), [(22.2, 33.3, 7.5, {**_BASE, "contrast_reference": r, "contrast_method": "Root Mean Square"})
                                     for r in (0.5, 1.5, -0.1)]),
}


# --------------------------------------------------------------------------------------------------------------- batch cases
def phantom(seed: int, n: int = 3, shape=(256, 256), center=(128.4, 127.6), radius=100.0, angle=0.0, dtype=np.uint16,
            contrast=0.004) -> np.ndarray:
    """Poisson noise around 1000 counts with the 18 low-contrast disks of LEEDS_LIKE, each brighter than the last"""
    rng = np.random.default_rng(seed)
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w]
    lam = np.full(shape, 1000.0)
    for i, st in enumerate(LEEDS_LIKE.values()):
        a = np.deg2rad(angle + st["angle"])
        cx, cy = center[0] + np.cos(a) * radius * st["distance from center"], center[1] + np.sin(a) * radius * st["distance from center"]
        lam[(yy - cy) ** 2 + (xx - cx) ** 2 < (radius * st["roi radius"]) ** 2] *= 1 + contrast * (i + 1)
    out = rng.poisson(lam, (n, h, w))
    return out.astype(dtype)


LEEDS_LIKE = {f"{i}": {"angle": i * 20.0, "distance from center": 0.7, "roi radius": 0.045} for i in range(18)}
LEEDS_BG = {"0": {"angle": 30, "distance from center": 0.35, "roi radius": 0.045},
            "1": {"angle": 210, "distance from center": 0.35, "roi radius": 0.045}}

BATCH_CASES = {
    "leeds_u16": (lambda: phantom(41), {"center": (128.4, 127.6), "angle": 0.0, "radius": 100.0}, {}),
    "leeds_rotated_weber": (lambda: phantom(42, angle=7.5), {"center": (128.4, 127.6), "angle": 7.5, "radius": 100.0},
                            {"contrast_method": "Weber", "visibility_threshold": 0.5, "roi_size_factor": 0.8}),
    "leeds_float32_ratio": (lambda: phantom(43, dtype=np.float32), {"center": (128.4, 127.6), "angle": 0.0, "radius": 100.0},
                            {"contrast_method": "Ratio", "percentiles": (2.5, 97.5)}),
    "leeds_int16_difference": (lambda: phantom(44, dtype=np.int16), {"center": (128.4, 127.6), "angle": -3.0, "radius": 101.5},
                               {"contrast_method": "Difference", "contrast_threshold": 10.0}),
    "leeds_float64_odd": (lambda: phantom(45, shape=(251, 263), center=(131.5, 125.5), dtype=np.float64),
                          {"center": (131.5, 125.5), "angle": 0.0, "radius": 100.0}, {"percentiles": (0, 100)}),
}

# direct calls of core.contrast: (function, args)
CONTRAST_CASES = [
    ("michelson", ([1.0, 3.0],)), ("michelson", ([np.nan, 2.0, 5.0],)), ("michelson", ([np.nan, np.nan],)),
    ("michelson", ([0.0, 0.0],)), ("michelson", ([-1.0, 1.0],)),
    ("weber", (5.0, 2.0)), ("weber", (5.0, 0.0)), ("weber", (5, 0)), ("weber", (np.float64(5.0), np.float64(0.0))),
    ("weber", (np.float64(0.0), np.float64(0.0))), ("ratio", (3.0, 0.0)), ("ratio", (np.float64(3.0), np.float64(0.0))),
    ("ratio", (7.0, 2.0)), ("difference", (2.0, 7.5)),
    ("rms", ([0.1, 0.9, 0.5],)), ("rms", ([0.0, 1.0],)), ("rms", ([-0.1, 0.5],)), ("rms", ([0.5, 1.1],)), ("rms", ([np.nan, 0.5],)),
    ("contrast", ([1.0, 2.0, 3.0], "Weber")), ("contrast", ([1.0, 2.0, 3.0], "Ratio")), ("contrast", ([1.0, 2.0, 3.0], "Difference")),
    ("contrast", ([1.0, 2.0, 3.0], "Michelson")), ("contrast", ([1.0, 2.0], "unknown")), ("contrast", ([0.25, 0.5], "ROOT MEAN SQUARE")),
    ("visibility", ([1000.0, 900.0], 5.0, 30.0, "Michelson")), ("visibility", ([1000.0, 900.0], 5.0, 0.0, "Weber")),
    ("visibility", ([1000.0, 900.0], 5.0, 30.0, "Difference")),
]
