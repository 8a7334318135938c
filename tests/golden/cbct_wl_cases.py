"""Seeded CT volumes for WinstonLutz.from_cbct (winston_lutz.py:1444-1509): the reference's generated sphere phantom
(tests_basic/test_winstonlutz.py create_sphere / GeneratedWLCBCT, 100^3 voxels of 1 mm, BB radius 5) and physical-unit variants
that exercise what the reference's own cases do not: int16 slices with negative values, a non-unit slice / pixel ratio, ratio 0.5
(exact halves in the linear zoom) and non-square slices.

case_volume(name) -> (volume [N, H, W] in the slice dtype, slice_thickness_mm, pixel_spacing_mm): slice n of the volume is the
reference's ``array[..., n]``."""
from __future__ import annotations

import numpy as np

# name: (offset along axes 0 / 1 / 2 in mm: + left / + up / + in, as create_sphere documents it)
SPHERES = {
    "sphere_perfect": (0, 0, 0),
    "sphere_left5": (5, 0, 0),
    "sphere_up_m5": (0, -5, 0),
    "sphere_in5": (0, 0, 5),
}

# name: (shape H, W, N, pixel mm, slice mm, offset mm, dtype, background, noise amplitude, seed)
PHYSICAL = {
    "int16_negative": ((100, 100, 100), 1.0, 1.0, (1.0, -2.0, 1.5), np.int16, -1000, 3, 11),
    "ratio_2p0_0p9": ((110, 110, 50), 0.9, 2.0, (1.5, -1.0, 2.0), np.uint16, 100, 4, 12),
    "ratio_half": ((100, 100, 200), 1.0, 0.5, (-1.0, 2.0, 1.0), np.uint16, 50, 2, 13),
    "nonsquare": ((80, 120, 100), 1.0, 1.25, (2.0, 1.0, -1.0), np.uint16, 20, 3, 14),
}

CASES = list(SPHERES) + list(PHYSICAL)

# the reference's own expectations for its generated-sphere classes (TestPerfectCBCT / TestOffset*CBCT,
# tests_basic/test_winstonlutz.py:2186-2218): cax2bb max / median / mean, cax2epid max, bb_shift_vector (x, y, z)
SPHERE_EXPECT = {
    "sphere_perfect": (0, 0, 0, 0, (0, 0, 0)),
    "sphere_left5": (5, 2.5, 2.5, 5, (-5, 0, 0)),
    "sphere_up_m5": (5, 2.5, 2.5, 5, (0, 0, 5)),
    "sphere_in5": (5, 5, 5, 5, (0, -5, 0)),
}


def create_sphere(radius, shape, offset=(0, 0, 0)):
    """tests_basic/test_winstonlutz.py:2078-2101, restated: radius - distance from the (offset) centre, clamped at 0, through a
    sigmoid, times 1000, background shifted to 0."""
    center = np.array(shape) / 2 - 0.5 + np.array(offset)
    indices = np.indices(shape)
    distances = np.sqrt(np.sum((indices - center[:, np.newaxis, np.newaxis, np.newaxis]) ** 2, axis=0))
    arr = radius - distances
    arr[arr <= 0] = 0
    arr = 1 / (1 + np.exp(-1.0 * arr))
    arr *= 1000
    arr -= arr.min()
    return arr


def _physical(shape, ps, st, offset, dtype, background, noise, seed, radius=5.0):
    h, w, n = shape
    ax = [(np.arange(k) - (k / 2 - 0.5)) * s for k, s in zip(shape, (ps, ps, st))]
    y, x, z = np.meshgrid(*ax, indexing="ij")
    d = np.sqrt((y - offset[0]) ** 2 + (x - offset[1]) ** 2 + (z - offset[2]) ** 2)
    arr = radius - d
    arr[arr <= 0] = 0
    arr = 1000 * (1 / (1 + np.exp(-arr)) - 0.5)
    rng = np.random.default_rng(seed)
    arr = np.round(arr) + background + rng.integers(-noise, noise + 1, size=arr.shape)
    return arr.astype(dtype)


def case_volume(name):
    if name in SPHERES:
        arr = create_sphere(5, (100, 100, 100), offset=SPHERES[name])
        # create_dicom_files_from_3d_array (core/array_utils.py:314-362): slice i = array[..., i].astype(uint16), 1 mm / 1 mm
        return np.ascontiguousarray(np.moveaxis(arr, -1, 0).astype(np.uint16)), 1.0, 1.0
    shape, ps, st, offset, dtype, background, noise, seed = PHYSICAL[name]
    arr = _physical(shape, ps, st, offset, dtype, background, noise, seed)
    return np.ascontiguousarray(np.moveaxis(arr, -1, 0)), st, ps
