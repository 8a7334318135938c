"""Seeded SPECT volumes for the pylinac.nuclear.TomographicUniformity goldens (make_tomo_uniformity_golden.py) and the tests that
check them.  CASES: name -> (volume builder, pixel size mm, TomographicUniformity.analyze kwargs, number of analyze() calls).  The
volumes are tomo_contrast_cases.jaszczak phantoms; every builder is deterministic in its seed."""
from __future__ import annotations

import numpy as np

from tests.golden.tomo_contrast_cases import jaszczak


def _hot_spot():
    """one voxel far above the cylinder in every slice of the slab: it sets the threshold's 10 % level and the FOV maximum"""
    v = jaszczak(21)
    v[:, 30, 33] = 9000
    return v


CASES = {
    # bin 2, the default slab (the last slice is dropped: 31 slices)
    "default_4p4": (lambda: jaszczak(1), 4.4, {}, 1),
    # bin 1, an explicit 7-slice slab
    "bin1_6p0": (lambda: jaszczak(3, shape=(24, 48, 56), pixel_size=6.0, z_extent=(2, 22), counts=150), 6.0,
                 {"first_frame": 2, "last_frame": 9}, 1),
    # bin 2, 75 x 69 is not a multiple of the bin; a 3-slice slab
    "bin2_3p3_odd": (lambda: jaszczak(2, shape=(28, 75, 69), pixel_size=3.3, z_extent=(3, 25)), 3.3,
                     {"first_frame": 10, "last_frame": 13}, 1),
    # bin 4, 130 x 126 is not a multiple of the bin; a 25-slice slab
    "bin4_2p2": (lambda: jaszczak(4, shape=(30, 130, 126), pixel_size=2.2, z_extent=(2, 28), counts=40), 2.2,
                 {"first_frame": 2, "last_frame": 27}, 1),
    # bin 1, a 128 x 128 frame (16 bytes a pixel is beyond shared memory); a 16-slice slab
    "large_bin1": (lambda: jaszczak(5, shape=(20, 128, 128), pixel_size=6.0, z_extent=(1, 19), counts=90), 6.0,
                   {"first_frame": 2, "last_frame": 18}, 1),
    "default_last_first5": (lambda: jaszczak(6), 4.4, {"first_frame": 5}, 1),
    "ratios": (lambda: jaszczak(7), 4.4, {"ufov_ratio": 0.9, "cfov_ratio": 0.6, "center_ratio": 0.5, "threshold": 0.6}, 1),
    "window3": (lambda: jaszczak(8), 4.4, {"window_size": 3}, 1),
    "window7": (lambda: jaszczak(9), 4.4, {"window_size": 7, "first_frame": 4, "last_frame": 11}, 1),
    "window_too_large": (lambda: jaszczak(10), 4.4, {"window_size": 40}, 1),
    "center_empty": (lambda: jaszczak(11), 4.4, {"center_ratio": 0.0}, 1),
    "ring_empty": (lambda: jaszczak(12), 4.4, {"cfov_ratio": 1.0}, 1),
    "hot_spot": (_hot_spot, 4.4, {}, 1),
    "uint8": (lambda: jaszczak(13, counts=60, dtype=np.uint8), 4.4, {"first_frame": 3, "last_frame": 28}, 1),
    "first_negative": (lambda: jaszczak(14), 4.4, {"first_frame": -1}, 1),
    "last_beyond": (lambda: jaszczak(15), 4.4, {"last_frame": 32}, 1),
    "last_before_first": (lambda: jaszczak(16), 4.4, {"first_frame": 9, "last_frame": 4}, 1),
    "one_slice": (lambda: jaszczak(17, shape=(1, 64, 64), z_extent=(0, 1)), 4.4, {}, 1),
    "second_analyze": (lambda: jaszczak(18), 4.4, {}, 2),
    "blank": (lambda: np.zeros((8, 32, 32), np.uint16), 4.4, {}, 1),
}
