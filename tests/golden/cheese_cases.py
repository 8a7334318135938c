"""Seeded synthetic cheese-phantom CT series for tests/golden/cheese_golden.npz (make_cheese_golden.py) and the GPU tests.

A water cylinder of the phantom's radius (plus 2 mm) with its inserts over the middle slices, air (-1000 HU) elsewhere, stored as
raw = (HU - intercept) / slope in int16 or uint16 with Gaussian noise.  Options: a couch slab touching the bottom border, a metal insert
above 1000 HU, a roll of the inserts, a phantom axis drifting across the series, per-slice rescale tags, another body value and
air-only end slices."""
from __future__ import annotations

import numpy as np

TOMO_OUTER = [-75, -45, -15, 15, 45, 75, 105, 135, 165, -165, -135, -105]
CIRS_OUTER = [-90, -45, 0, 45, 90, 135, 180, -135]

# name: phantom, n slices, size px, pixel mm, slice mm, dtype, intercept (None: per-slice), extras
CASES = {
    "tomo_512": dict(phantom="TomoCheese", n=24, size=512, px=0.8, thk=2.0, dtype="int16", intercept=-1024.0),
    "tomo_256_roll3": dict(phantom="TomoCheese", n=16, size=256, px=1.4, thk=3.0, dtype="uint16", intercept=-1000.0, roll=3.0),
    # a couch touching the border: with clear_border on it takes the phantom with it, so no slice is in view
    "tomo_couch": dict(phantom="TomoCheese", n=12, size=448, px=0.9, thk=2.5, dtype="int16", intercept=-1024.0, couch=True),
    # a 2600 HU insert: clipping changes the Otsu threshold of the slices that hold it; the phantom still localizes
    "tomo_metal": dict(phantom="TomoCheese", n=20, size=448, px=0.9, thk=2.5, dtype="int16", intercept=-1024.0, metal=True,
                       roll=-3.0, drift=(6.0, -4.0)),
    # the brightest insert at 34 degrees, 11 degrees from the nearest nominal insert angle: the "> 5 degrees" message
    "tomo_roll19": dict(phantom="TomoCheese", n=12, size=480, px=0.85, thk=2.0, dtype="int16", intercept=-1024.0, roll=19.0),
    # no inserts and a -60 HU body: the profile is all zeros after the negatives are cleared, so find_fwxm_peaks finds no peak and
    # the reference's `if peak_idxs:` on the empty array raises numpy's ValueError (its "No low-HU regions" message is printed only
    # for a single peak at index 0)
    "tomo_noinsert": dict(phantom="TomoCheese", n=12, size=480, px=0.85, thk=2.0, dtype="int16", intercept=-1024.0, flat=True,
                          body=-60.0),
    # 72 slices of 512 x 512 (more than one device chunk of 64) with air-only ends: constant slices (no edges at all) and slices
    # with 0.1 HU steps (slope 0.1), whose Scharr maximum is above 0 and below 0.1
    "tomo_long": dict(phantom="TomoCheese", n=72, size=512, px=0.8, thk=1.0, dtype="int16", intercept=-1024.0, slope=0.1,
                      air_ends=8),
    "cirs_512": dict(phantom="CIRS062M", n=20, size=512, px=0.8, thk=2.0, dtype="int16", intercept=None, couch=True),
    "cirs_uint16": dict(phantom="CIRS062M", n=14, size=400, px=1.0, thk=1.0, dtype="uint16", intercept=-1024.0, slope=0.5),
    "tomo_edge_origin": dict(phantom="TomoCheese", n=12, size=480, px=0.85, thk=2.0, dtype="int16", intercept=-1024.0,
                             inserts=(0, 3)),
    "tomo_air_only": dict(phantom="TomoCheese", n=10, size=256, px=1.4, thk=2.0, dtype="int16", intercept=-1024.0, empty=True),
}

# analyze() variants per case (kwargs); every case also runs analyze() once more with the first set
ANALYZE = {
    "tomo_512": [{}, {"x_adjustment": 1.5, "y_adjustment": -2.0, "angle_adjustment": 1.0, "roi_size_factor": 0.8,
                      "scaling_factor": 1.02}],
    "tomo_256_roll3": [{}],
    "tomo_couch": [{}],
    "tomo_metal": [{}, {"origin_slice": 9}],
    "tomo_roll19": [{}],
    "tomo_noinsert": [{"origin_slice": 6}],
    "tomo_long": [{}],
    "cirs_512": [{}, {"roi_size_factor": 1.2}],
    "cirs_uint16": [{}],
    "tomo_edge_origin": [{}],
    "tomo_air_only": [{}],
}

# what each case must reach (checked when the goldens are made and by tests/test_oracle_cheese.py): "stdout" a printed message,
# "error" the exception type of the first analyze(), "statuses" localization statuses that must occur, "small_edges" a NO_EDGES row
# with a Scharr maximum above 0, "clipped" slices whose Otsu threshold clipping changes, "roll" the first analyze()'s roll
EXPECT = {
    "tomo_512": dict(statuses={0}),
    "tomo_256_roll3": dict(statuses={0}, roll=(2.0, 4.0)),
    "tomo_couch": dict(error="TypeError", statuses={2, 3}, only=True),
    "tomo_metal": dict(statuses={0}, clipped=True, roll=(-4.0, -2.0)),
    "tomo_roll19": dict(stdout="Detected shift of ", roll=(0.0, 0.0)),
    "tomo_noinsert": dict(error="ValueError"),
    "tomo_long": dict(statuses={0, 1}, small_edges=True),
    "cirs_512": dict(statuses={0}),
    "cirs_uint16": dict(statuses={0}),
    "tomo_edge_origin": dict(error="ValueError"),
    "tomo_air_only": dict(error="TypeError"),
}


def case_series(name):
    """-> (raw volume [n, h, w], slopes [n], intercepts [n], pixel mm, slice mm)"""
    c = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    n, size, px = c["n"], c["size"], c["px"]
    tomo = c["phantom"] == "TomoCheese"
    radius_mm = 152.0 if tomo else 157.0
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float64)
    first, last = c.get("inserts", (n // 4, n - n // 4))
    vol = np.empty((n, size, size))
    for z in range(n):
        dx, dy = c.get("drift", (0.0, 0.0))
        cx = size / 2 - 0.5 + 3.3 + dx * z / n
        cy = size / 2 - 0.5 - 2.1 + dy * z / n
        r = np.hypot(xx - cx, yy - cy) * px
        hu = np.full((size, size), -1000.0)
        if not c.get("empty"):
            hu[r <= radius_mm] = c.get("body", 2.0)
            if first <= z < last and not c.get("flat"):
                roll = c.get("roll", 0.0)
                outer = TOMO_OUTER if tomo else CIRS_OUTER
                dist = 110.0 if tomo else 115.0
                for k, ang in enumerate(outer):
                    val = {0: -850.0, 3: 950.0}.get(k, 10.0 * ((k % 3) - 1))
                    if c.get("metal") and k == 3:
                        val = 2600.0
                    a = np.deg2rad(ang + roll)
                    ix, iy = cx + np.cos(a) * dist / px, cy + np.sin(a) * dist / px
                    hu[np.hypot(xx - ix, yy - iy) * px <= (12.5 if tomo else 10.5)] = val
                inner = [-67.5, -22.5, 22.5, 67.5, 112.5, 157.5, -157.5, -112.5] if tomo else [-90, -45, 0, 45, 90, 135, 180, -135]
                for k, ang in enumerate(inner):
                    a = np.deg2rad(ang + roll)
                    d = 65.0 if tomo else 60.0
                    ix, iy = cx + np.cos(a) * d / px, cy + np.sin(a) * d / px
                    hu[np.hypot(xx - ix, yy - iy) * px <= 11.0] = 40.0 * k - 150.0
        if c.get("couch"):
            hu[int(cy + radius_mm / px) + 3:, :] = np.maximum(hu[int(cy + radius_mm / px) + 3:, :], -300.0)
        ends = c.get("air_ends", 0)
        if z < ends or z >= n - ends:
            hu[:] = -1000.0             # air only, without noise (every other such slice gets 0.1 HU steps below)
        else:
            hu = hu + rng.normal(0, 6.0, hu.shape)
        vol[z] = hu
    if c["intercept"] is None:
        intercepts = np.where(np.arange(n) % 2 == 0, -1024.0, -1000.0)
    else:
        intercepts = np.full(n, c["intercept"])
    slopes = np.full(n, c.get("slope", 1.0))
    raw = np.rint((vol - intercepts[:, None, None]) / slopes[:, None, None])
    dt = np.dtype(c["dtype"])
    raw = np.clip(raw, np.iinfo(dt).min, np.iinfo(dt).max).astype(dt)
    ends = c.get("air_ends", 0)
    for z in [*range(1, ends, 2), *range(n - ends + 1, n, 2)]:
        raw[z][rng.random(raw[z].shape) < 0.01] += 1        # one stored step: slope x 1 HU
    return raw, slopes, intercepts, px, c["thk"]
