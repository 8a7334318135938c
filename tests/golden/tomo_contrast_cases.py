"""Seeded SPECT volumes for the pylinac.nuclear.TomographicContrast goldens (make_tomo_contrast_golden.py) and the tests that check
them.  CASES: name -> (volume builder, pixel size mm, TomographicContrast.analyze kwargs).  Every builder is deterministic in its seed."""
from __future__ import annotations

import math

import numpy as np

DEFAULT_DIAMETERS = (38, 31.8, 25.4, 19.1, 15.9, 12.7)
DEFAULT_ANGLES = (-10, -70, -130, -190, 110, 50)


def jaszczak(seed, shape=(32, 64, 64), *, pixel_size=4.4, frac=0.8, counts=300.0, background=0.5, z_extent=(3, 29), sphere_z=None,
             diameters=DEFAULT_DIAMETERS, angles=DEFAULT_ANGLES, sphere_gain=0.1, offset=(0.0, 0.0), dtype=np.uint16):
    """A Jaszczak-like volume: a uniform cylinder (radius frac x half the smaller side, slices z_extent[0] .. z_extent[1] - 1) of
    `counts` mean counts over a `background` level, with cold spheres of `diameters` (mm) at `angles` (degrees) on a ring at 0.65 of
    the cylinder radius, centred on slice `sphere_z`; Poisson noise."""
    rng = np.random.default_rng(seed)
    nz, h, w = shape
    z, y, x = np.mgrid[0:nz, 0:h, 0:w].astype(float)
    cy, cx = (h - 1) / 2 + offset[0], (w - 1) / 2 + offset[1]
    rad = frac * min(h, w) / 2
    # the two slices at each end of the cylinder are narrower, as partial-volume slices are: slice_data drops them
    end = (z < z_extent[0] + 2) | (z >= z_extent[1] - 2)
    inside = ((y - cy) ** 2 + (x - cx) ** 2 <= (np.where(end, 0.6, 1.0) * rad) ** 2) & (z >= z_extent[0]) & (z < z_extent[1])
    lam = np.where(inside, counts, background)
    sz = (z_extent[0] + z_extent[1]) / 2 if sphere_z is None else sphere_z
    for d, a in zip(diameters, angles):
        r = d / 2 / pixel_size
        sx, sy = cx + 0.65 * rad * math.cos(math.radians(a)), cy + 0.65 * rad * math.sin(math.radians(a))
        lam = np.where((x - sx) ** 2 + (y - sy) ** 2 + (z - sz) ** 2 <= r ** 2, lam * sphere_gain, lam)
    return np.clip(rng.poisson(lam), 0, np.iinfo(dtype).max).astype(dtype)


def _blank_slices():
    """empty edge slices (no component), and one slice whose only component is a one-pixel-wide line: its FOV is empty"""
    v = jaszczak(31, z_extent=(4, 28))
    v[:2] = 0
    v[2] = 0
    v[2, 30, 5:55] = 300
    return v


def _tied_largest():
    """a slice with two components of equal area: the first in raster order is the largest"""
    v = jaszczak(32, z_extent=(2, 30))
    v[0] = 0
    v[0, 10:20, 5:15] = 300
    v[0, 40:50, 45:55] = 300
    v[1] = 0
    v[1, 5:9, 40:55] = 300
    v[1, 30:45, 10:14] = 300
    return v


def _edge_volume():
    """the cylinder close to the x / y edges and the sphere slice at the top of the volume: search boxes cross every edge"""
    return jaszczak(33, frac=0.98, z_extent=(0, 32), sphere_z=1.0, offset=(2.0, -2.0))


CASES = {
    "default_4p4": (lambda: jaszczak(1), 4.4, {}),
    "default_3p3": (lambda: jaszczak(2, shape=(36, 80, 80), pixel_size=3.3, z_extent=(4, 32)), 3.3, {}),
    "default_6p0": (lambda: jaszczak(3, shape=(24, 48, 56), pixel_size=6.0, z_extent=(2, 22), counts=150), 6.0, {}),
    "edges": (_edge_volume, 4.4, {"search_window_px": 8, "search_slices": 5}),
    "empty_sphere": (lambda: jaszczak(4), 4.4, {"sphere_diameters_mm": (0.5, 25.4), "sphere_angles": (-10, 110)}),
    "blank_and_empty_fov_slices": (_blank_slices, 4.4, {}),
    "tied_largest": (_tied_largest, 4.4, {}),
    "custom": (lambda: jaszczak(5, diameters=(30, 20, 10), angles=(0, 120, 240), sphere_gain=0.3), 4.4,
               {"sphere_diameters_mm": (30, 20, 10), "sphere_angles": (0, 120, 240), "ufov_ratio": 0.7, "search_window_px": 3,
                "search_slices": 2}),
    "hot_spheres_u8": (lambda: jaszczak(6, counts=60, sphere_gain=3.0, dtype=np.uint8), 4.4, {}),
    "length_mismatch": (lambda: jaszczak(7), 4.4, {"sphere_diameters_mm": (38, 31.8), "sphere_angles": (-10,)}),
    "no_slice": (lambda: np.zeros((8, 32, 32), np.uint16), 4.4, {}),
    "large_slice": (lambda: jaszczak(8, shape=(10, 160, 150), pixel_size=2.2, z_extent=(1, 9), counts=80), 2.2, {"search_slices": 2}),
}
