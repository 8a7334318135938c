"""Seeded synthetic ACR CT 464 series for tests/golden/acr_golden.npz (make_acr_golden.py), the GPU tests and tools/bench_acr.py.

A 200 mm water cylinder with the four modules at z = origin + 0, 30, 70 and 100 mm, each a few slices thick, water between them and
air (-1000 HU) beyond the phantom.  The HU module holds the five material inserts and the two air bubbles the roll is read from (both
right of the centre, one above the other, rotated by the roll); the uniformity module is plain water; the resolution module holds eight
striped disks (1000 HU +- a contrast that falls with their line-pair spacing); the low-contrast module one +6 HU disk.  Stored as
raw = (HU - intercept) / slope in int16 or uint16 with Gaussian noise.
"""
from __future__ import annotations

import numpy as np

# name: n slices, size px, pixel mm, slice mm, dtype, intercept (None: per slice), extras
CASES = {
    "acr_512": dict(n=48, size=512, px=0.5, thk=2.5, dtype="int16", intercept=-1024.0),
    "acr_256_roll3": dict(n=46, size=256, px=1.0, thk=2.5, dtype="uint16", intercept=None, roll=3.0, slope=0.5),
    "acr_256_roll_m2": dict(n=46, size=256, px=1.0, thk=2.5, dtype="int16", intercept=-1000.0, roll=-2.0, drift=(3.0, -2.0)),
    # a 216 mm field of view: the 110 mm Otsu disk reaches past the image on every side; air-only end slices
    "acr_small_fov": dict(n=48, size=240, px=0.9, thk=2.5, dtype="int16", intercept=-1024.0, air_ends=3),
    # no inserts and no air bubbles on the given origin slice: fewer than two qualifying regions -> the roll warning and 0.0
    "acr_no_bubbles": dict(n=46, size=256, px=1.0, thk=2.5, dtype="int16", intercept=-1024.0, no_hu=True),
    # the series stops 60 mm past the HU module: the other modules are not scanned
    "acr_short": dict(n=30, size=256, px=1.0, thk=2.5, dtype="int16", intercept=-1024.0),
    # no HU module at all
    "acr_no_hu": dict(n=46, size=256, px=1.0, thk=2.5, dtype="int16", intercept=-1024.0, no_hu=True),
    # striped disks of equal contrast: the MTF does not drop monotonically
    "acr_flat_mtf": dict(n=46, size=256, px=1.0, thk=2.5, dtype="int16", intercept=-1024.0, flat_mtf=True),
}

ORIGIN_Z_MM = 10.0      # the HU module's z above the first slice

# analyze() variants per case (kwargs); every case also runs analyze() once more on the same object with the first set, and a second
# instance of the case runs the first set after the first instance
ANALYZE = {
    "acr_512": [{}],
    "acr_256_roll3": [{}],
    "acr_256_roll_m2": [{"x_adjustment": 1.5, "y_adjustment": -1.0, "angle_adjustment": 1.0, "roi_size_factor": 0.9,
                         "scaling_factor": 1.02}],
    "acr_small_fov": [{}],
    "acr_no_bubbles": [{"origin_slice": 4}],
    "acr_short": [{}],
    "acr_no_hu": [{}, {"origin_slice": 4}],
    "acr_flat_mtf": [{"origin_slice": 5}],
}

# what each case must reach (checked when the goldens are made and by tests/test_oracle_acr.py): "error" the exception type of the
# first analyze(), "warnings" messages the first analyze() must warn (substrings), "roll" the range of the first roll, "beyond" the
# Otsu disk reaches past the image, "statuses" localization statuses that must occur
EXPECT = {
    "acr_512": dict(statuses={0}, roll=(-0.5, 0.5)),
    "acr_256_roll3": dict(statuses={0}, roll=(2.0, 4.0)),
    "acr_256_roll_m2": dict(statuses={0}, roll=(-2.0, 0.0)),
    "acr_small_fov": dict(statuses={0, 1}, beyond=True),
    "acr_no_bubbles": dict(statuses={0}, warnings=["Could not determine phantom roll"], roll=(0.0, 0.0)),
    "acr_short": dict(error="ValueError"),
    "acr_no_hu": dict(error="ValueError"),
    "acr_flat_mtf": dict(warnings=["does not drop monotonically"]),
}

HU_INSERTS = [(45, -1000.0), (225, -95.0), (135, 120.0), (-45, 955.0), (180, 0.0)]
LP = [(-135, 0.4), (-180, 0.5), (135, 0.6), (90, 0.7), (45, 0.8), (0, 0.9), (-45, 1.0), (-90, 1.2)]


def case_series(name):
    """-> (raw volume [n, h, w], slopes [n], intercepts [n], pixel mm, slice mm)"""
    c = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)) + 17)
    n, size, px, thk = c["n"], c["size"], c["px"], c["thk"]
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float64)
    roll = c.get("roll", 0.0)
    vol = np.empty((n, size, size))
    for z in range(n):
        dx, dy = c.get("drift", (0.0, 0.0))
        cx = size / 2 - 0.5 + 2.3 / px + dx * z / n
        cy = size / 2 - 0.5 - 1.7 / px + dy * z / n
        r = np.hypot(xx - cx, yy - cy) * px
        hu = np.full((size, size), -1000.0)
        hu[r <= 100.0] = 0.0
        zmm = z * thk - ORIGIN_Z_MM

        def blob(ang, dist, rad, val):
            a = np.deg2rad(ang + roll)
            ix, iy = cx + np.cos(a) * dist / px, cy + np.sin(a) * dist / px
            m = np.hypot(xx - ix, yy - iy) * px <= rad
            hu[m] = val
            return m, ix, iy

        if abs(zmm) <= 6 and not c.get("no_hu"):
            for ang, val in HU_INSERTS:
                blob(ang, 63.0, 12.5, val)
            if c.get("bubbles", True):
                blob(-59.0, 29.2, 9.0, -1000.0)          # right of centre, above
                blob(59.0, 29.2, 9.0, -1000.0)           # right of centre, below
        elif abs(zmm - 100) <= 6:
            for k, (ang, lp) in enumerate(LP):
                m, ix, iy = blob(ang, 70.0, 7.0, 0.0)
                period = 1.0 / lp
                amp = 400.0 if c.get("flat_mtf") else 800.0 * (1.0 - 0.1 * k)
                stripes = np.where(np.floor((xx - ix) * px / (period / 2)) % 2 == 0, 1000.0 + amp, 1000.0 - amp)
                hu[m] = stripes[m]
        elif abs(zmm - 30) <= 6:
            blob(-90, 60.0, 6.5, 6.0)
        ends = c.get("air_ends", 0)
        if z < ends or z >= n - ends:
            hu[:] = -1000.0
        else:
            hu = hu + rng.normal(0, 4.0, hu.shape)
        vol[z] = hu
    if c["intercept"] is None:
        intercepts = np.where(np.arange(n) % 2 == 0, -1024.0, -1000.0)
    else:
        intercepts = np.full(n, c["intercept"])
    slopes = np.full(n, c.get("slope", 1.0))
    raw = np.rint((vol - intercepts[:, None, None]) / slopes[:, None, None])
    dt = np.dtype(c["dtype"])
    raw = np.clip(raw, np.iinfo(dt).min, np.iinfo(dt).max).astype(dt)
    return raw, slopes, intercepts, px, thk
