"""Seeded four-quadrant bar-phantom frames for the pylinac.nuclear.QuadrantResolution goldens (make_quadrant_golden.py) and the tests
that check them, and seeded arrays for the DiskROI goldens.

CASES: name -> (frames builder, QuadrantResolution.analyze kwargs).  Each builder returns [n, h, w] frames that are written to an NM
file; only frame 0 is analysed.  DISK_CASES: name -> (array builder, [(centre row, centre col, radius), ...]) for DiskROI directly.

A QuadrantResolution disk cannot wrap without another one raising: its four disks reach e = distance * cos 45 + radius beyond the
centre (Rows / 2, Columns / 2) on both axes, and a wrap needs e > Columns / 2 (rows) or e > Rows / 2 (columns) while staying inside
needs Columns / 2 + e < Rows and Rows / 2 + e < Columns.  Those contradict each other, so wrapping is covered by DISK_CASES and the
fuzz, and the non-square cases here sit off-centre or raise."""
from __future__ import annotations

import numpy as np

WIDTHS = [4.23, 3.18, 2.54, 2.12]


def bars(seed: int, shape=(512, 512), widths_px=(7, 5, 4, 3), high=140, low=60, dtype=np.uint16, frames=1) -> np.ndarray:
    """Poisson counts of a bar pattern: one bar width per quadrant of the frame, vertical bars in two quadrants and horizontal
    bars in the other two.  The contrast keeps the moments MTF below 1, where its FWHM is defined."""
    rng = np.random.default_rng(seed)
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w]
    q = (yy >= h / 2).astype(int) * 2 + (xx >= w / 2)
    wp = np.asarray(widths_px)[q]
    along = np.where(q % 3 == 0, xx, yy)
    lam = np.where((along // wp) % 2 == 0, high, low)
    out = rng.poisson(lam, (frames, h, w))
    return np.minimum(out, np.iinfo(dtype).max).astype(dtype)


def flat(seed: int, shape=(512, 512), counts=100) -> np.ndarray:
    """a flat Poisson flood: std**2 is about the mean, so the moments MTF takes the square root of a negative number"""
    return np.random.default_rng(seed).poisson(counts, (1,) + shape).astype(np.uint16)


CASES = {
    "u16_512": (lambda: bars(1), {"bar_widths": WIDTHS}),
    "u16_1024": (lambda: bars(2, (1024, 1024), widths_px=(12, 9, 7, 5), high=700, low=300), {"bar_widths": WIDTHS}),
    "u8_512": (lambda: bars(3, dtype=np.uint8, high=150, low=50), {"bar_widths": WIDTHS}),
    "multiframe": (lambda: bars(4, frames=3), {"bar_widths": WIDTHS}),
    # 511 / 2 = 255.5: every centre is on a half pixel
    "odd_511": (lambda: bars(5, (511, 511)), {"bar_widths": WIDTHS}),
    # Rows 301 give x = 150.5, Columns 333 give y = 166.5: the disks sit off the phantom's centre
    "non_square_301x333": (lambda: bars(6, (301, 333)), {"bar_widths": WIDTHS, "roi_diameter_mm": 40, "distance_from_center_mm": 80}),
    "non_square_raises": (lambda: bars(7, (300, 600)), {"bar_widths": WIDTHS}),
    "default_raises_256": (lambda: bars(8, (256, 256)), {"bar_widths": WIDTHS}),
    "duplicate_widths": (lambda: bars(9), {"bar_widths": [3.18, 2.54, 3.18, 2.12]}),
    "all_equal_widths": (lambda: bars(10), {"bar_widths": [2.5, 2.5, 2.5, 2.5]}),
    "three_widths": (lambda: bars(11), {"bar_widths": [4.23, 3.18, 2.54]}),
    "five_widths": (lambda: bars(12), {"bar_widths": [4.23, 3.18, 2.54, 2.12, 1.5]}),
    "flat_poisson": (lambda: flat(13), {"bar_widths": WIDTHS}),
    "blank": (lambda: np.zeros((1, 512, 512), np.uint16), {"bar_widths": WIDTHS}),
    # a high contrast: the moments MTF exceeds 1 and its FWHM takes the square root of a negative logarithm
    "mtf_above_one": (lambda: bars(17, high=190, low=10), {"bar_widths": WIDTHS}),
    "diameter_distance": (lambda: bars(14), {"bar_widths": WIDTHS, "roi_diameter_mm": 50.5, "distance_from_center_mm": 120.25}),
    # a radius of 0.3 px around centres half a pixel off the grid: every disk is empty, so every statistic is numpy's empty-array
    # result
    "empty_disks": (lambda: bars(15), {"bar_widths": WIDTHS, "roi_diameter_mm": 0.3, "distance_from_center_mm": 70.5 * 2 ** 0.5}),
    "one_pixel_disks": (lambda: bars(16), {"bar_widths": WIDTHS, "roi_diameter_mm": 1, "distance_from_center_mm": 100 * 2 ** 0.5}),
}


def _noise(seed: int, shape, dtype) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if np.issubdtype(dtype, np.floating):
        return (rng.standard_normal(shape) * 1000 + 50).astype(dtype)
    return rng.integers(0, 4000, shape).astype(dtype)


_DISKS = [(-3.5, 10.2, 6.3), (20.0, -2.7, 5.0), (-60.25, -70.5, 3.7), (30.5, 40.5, 0.4), (10.0, 10.0, 1.0), (31.2, 39.9, 17.6),
          (63.0, 79.0, 2.2), (70.0, 10.0, 5.0), (10.0, -85.0, 6.0)]

DISK_CASES = {
    "uint16": (lambda: _noise(21, (64, 80), np.uint16), _DISKS),
    "float32": (lambda: _noise(22, (64, 80), np.float32), _DISKS),
    "float64": (lambda: _noise(23, (64, 80), np.float64), _DISKS),
    "int32": (lambda: _noise(24, (64, 80), np.int32), _DISKS),
}
