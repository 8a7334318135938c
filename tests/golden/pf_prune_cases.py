"""Seeded synthetic PF cases for the leaf-row pruning of the reference (picketfence.py:810-828) and for picket counts at the
edges of the CUDA path's limits (1, 2 and 32 pickets).  Shared by the golden generator, the oracle tests and the GPU tests.

The short-picket frames are the benchmark recipe (ten 3 mm pickets, 20 mm apart, offset errors from default_rng(10_000)) with
picket 0 shorter than the others: the leaf rows beyond its ends kiss one picket fewer, and the median kiss count decides whether
they are dropped (median 10), whether picket 0 is dropped from every row (median 9) or whether every row is (median 9.5)."""
from __future__ import annotations

import numpy as np

from oracle import synth


def short_picket_frame(full_h, short_h, short_off=0.0, orientation="up_down"):
    """Ten 3 mm pickets at -90..90 mm (+ the offset errors of bench_pf_frame(0)), picket 0 ``short_h`` mm long centred at
    ``short_off`` mm along the leaf stack, the others ``full_h`` mm long; Gaussian 1 mm, noise 0.002 seeded 0."""
    fr = synth.epid1024()
    err = np.random.default_rng(10_000).uniform(-0.5, 0.5, 10)
    for k, pos in enumerate(range(-90, 91, 20)):
        pos = pos + err[k]
        h, off = (short_h, short_off) if k == 0 else (full_h, 0)
        if orientation == "up_down":
            fr.add_filtered_field((h, 3), (off, pos))
        else:
            fr.add_filtered_field((3, h), (pos, off))
    fr.gaussian(1.0)
    fr.noise(0.002, seed=0)
    return fr.image


def _pickets(n, spacing_mm, width_mm):
    return synth.picketfence_frame(synth.epid1024(), pickets=n, picket_spacing_mm=spacing_mm, picket_width_mm=width_mm, seed=7,
                                   picket_offset_error=np.random.default_rng(3).uniform(-.3, .3, n))


def case_frame(name):
    """-> (frame uint16, pixel_spacing_mm, sid, ctor_kwargs, analyze_kwargs)"""
    ps, sid = 0.390625, 1000.0
    ht = {"height_threshold": 0.3}
    if name == "rows_removed":                 # median 10: the 20 rows beyond picket 0 are dropped
        return short_picket_frame(300, 150), ps, sid, {}, {}
    if name == "rows_removed_offset":          # the short picket off-centre: a different set of rows is dropped
        return short_picket_frame(300, 150, 7.5), ps, sid, {}, {}
    if name == "rows_removed_ht03":            # rows with 9 and with 10 kisses, median 10
        return short_picket_frame(200, 110), ps, sid, {}, ht
    if name == "median_half":                  # as many rows with 9 kisses as with 10: median 9.5 keeps no row
        return short_picket_frame(200, 100), ps, sid, {}, ht
    if name == "median_nine":                  # median 9: every row keeps only the rows without picket 0, which has no fit
        return short_picket_frame(300, 120), ps, sid, {}, ht
    if name == "rows_removed_separate":
        return short_picket_frame(300, 150), ps, sid, {}, {"separate_leaves": True, "nominal_gap_mm": 3}
    if name == "rows_removed_left_right":      # picket 0 peaks at half height: just under the default threshold here
        return short_picket_frame(300, 150, orientation="left_right"), ps, sid, {}, ht
    if name == "rows_removed_hdmlc":
        return short_picket_frame(300, 150), ps, sid, {"mlc": "HD"}, {}
    if name == "pickets32":                    # 1600 measurements: more than the default table of 1024 rows
        return _pickets(32, 10, 3), ps, sid, {}, {}
    if name == "pickets32_separate":           # 3200 |errors| for the median
        return _pickets(32, 10, 3), ps, sid, {}, {"separate_leaves": True, "nominal_gap_mm": 3}
    if name == "pickets2":
        return _pickets(2, 40, 4), ps, sid, {}, {}
    if name == "picket1":                      # np.median(np.diff([i])) is nan: the window bounds cannot be computed
        return _pickets(1, 40, 4), ps, sid, {}, {}
    if name == "picket1_spacing50":
        return _pickets(1, 40, 4), ps, sid, {}, {"picket_spacing": 50}
    raise KeyError(name)


CASES = ["rows_removed", "rows_removed_offset", "rows_removed_ht03", "median_half", "median_nine", "rows_removed_separate",
         "rows_removed_left_right", "rows_removed_hdmlc", "pickets32", "pickets32_separate", "pickets2", "picket1",
         "picket1_spacing50"]
