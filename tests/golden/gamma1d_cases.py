"""Seeded profile pairs for core.gamma.gamma_geometric and gamma_1d (reference core/gamma.py:105-226, 333-460), the profile gamma
methods, and the argument errors the reference raises.  The goldens are the unmodified reference's results
(tests/golden/make_gamma1d_golden.py)."""
from __future__ import annotations

import numpy as np


def field(x, centre=0.0, width=40.0, penumbra=2.0, scale=1000.0):
    """a flat field with sigmoid edges, 20 % tails"""
    inner = 1 / (1 + np.exp(-(x - centre + width / 2) / penumbra)) / (1 + np.exp((x - centre - width / 2) / penumbra))
    return scale * (0.8 * inner + 0.2 * np.exp(-((x - centre) / (2 * width)) ** 2))


# name: (function, n_ref, ref pitch, n_eval, eval pitch, eval shift, eval dose scale, dtype, coordinates kind, kwargs)
#   coordinates: "none" (element indices), "x" (both given), "dec_eval" / "dec_both" (decreasing), "int" (integer grids)
CASES = {}
for fn in ("geometric", "1d"):
    CASES.update({
        f"{fn}_identical": (fn, 201, 0.5, 201, 0.5, 0.0, 1.0, np.float64, "x", {}),
        f"{fn}_dose_3pct": (fn, 201, 0.5, 201, 0.5, 0.0, 1.03, np.float64, "x", dict(dose_to_agreement=3, distance_to_agreement=3)),
        f"{fn}_shift_dta2": (fn, 241, 0.25, 241, 0.25, 0.7, 1.0, np.float64, "x", dict(dose_to_agreement=2, distance_to_agreement=2)),
        f"{fn}_as1000_as1200": (fn, 256, 0.392, 320, 0.336, 0.2, 1.01, np.float64, "x", dict(distance_to_agreement=1)),
        f"{fn}_dec_eval": (fn, 161, 0.5, 161, 0.5, 0.3, 1.0, np.float64, "dec_eval", dict(distance_to_agreement=2)),
        f"{fn}_dec_both": (fn, 161, 0.5, 161, 0.5, -0.3, 0.99, np.float64, "dec_both", dict(distance_to_agreement=3)),
        f"{fn}_coarse_spacing": (fn, 60, 2.5, 60, 2.5, 0.5, 1.0, np.float64, "x", dict(distance_to_agreement=0.5)),
        f"{fn}_ref_inside_eval": (fn, 101, 0.5, 181, 0.5, 0.0, 1.02, np.float64, "x", {}),
        f"{fn}_int_grid_ties": (fn, 80, 1.0, 80, 1.0, 0.0, 1.01, np.int32, "int", dict(distance_to_agreement=2)),
        f"{fn}_none_coords": (fn, 90, 1.0, 90, 1.0, 1.0, 1.0, np.uint16, "none", dict(distance_to_agreement=1)),
        f"{fn}_thr0_cap1": (fn, 151, 0.5, 151, 0.5, 0.4, 1.02, np.float64, "x", dict(dose_threshold=0, gamma_cap_value=1)),
        f"{fn}_thr50_fill0": (fn, 151, 0.5, 151, 0.5, 0.4, 1.0, np.float64, "x", dict(dose_threshold=50, fill_value=0)),
        f"{fn}_fill_neg1": (fn, 151, 0.5, 151, 0.5, 0.4, 1.0, np.float32, "x", dict(fill_value=-1.0, distance_to_agreement=3)),
        f"{fn}_u16": (fn, 181, 0.5, 181, 0.5, 0.2, 1.01, np.uint16, "x", dict(distance_to_agreement=2)),
        f"{fn}_i32": (fn, 181, 0.5, 181, 0.5, -0.2, 0.99, np.int32, "x", dict(dose_to_agreement=2)),
        f"{fn}_f32": (fn, 181, 0.5, 181, 0.5, 0.2, 1.0, np.float32, "x", dict(dose_to_agreement=3, distance_to_agreement=3)),
        f"{fn}_4096": (fn, 4096, 0.1, 4096, 0.1, 0.15, 1.005, np.float64, "x", dict(distance_to_agreement=1)),
        f"{fn}_edges_clamp": (fn, 41, 1.0, 41, 1.0, 0.0, 1.0, np.float64, "x", dict(dose_threshold=0, distance_to_agreement=3)),
    })
for dta in (0.5, 1, 2, 3):
    CASES[f"1d_local_dta{dta}"] = ("1d", 161, 0.5, 161, 0.5, 0.3, 1.01, np.float64, "x", dict(global_dose=False, distance_to_agreement=dta))
CASES.update({
    "1d_local_f32": ("1d", 161, 0.5, 161, 0.5, 0.3, 1.01, np.float32, "x", dict(global_dose=False, distance_to_agreement=2)),
    "1d_local_u16": ("1d", 161, 0.5, 161, 0.5, 0.3, 1.01, np.uint16, "x", dict(global_dose=False)),
    "1d_rf1": ("1d", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(resolution_factor=1, distance_to_agreement=2)),
    "1d_rf5": ("1d", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(resolution_factor=5)),
    "1d_num_truncates_to_1": ("1d", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(distance_to_agreement=0.1)),
    "1d_nan_eval": ("1d", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(distance_to_agreement=2)),
    "1d_nan_ref": ("1d", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(distance_to_agreement=2, global_dose=False)),
    "1d_one_sample_eval": ("1d", 1, 0.5, 1, 0.5, 0.0, 1.0, np.float64, "x", {}),
    "geometric_dta_half": ("geometric", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(distance_to_agreement=0.5)),
    "geometric_nan_eval_outside": ("geometric", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(dose_threshold=50)),
    "geometric_nan_eval_raises": ("geometric", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", {}),
    "geometric_nan_ref_raises": ("geometric", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", {}),
    "geometric_fill0_int_nan_free": ("geometric", 121, 0.5, 121, 0.5, 0.3, 1.0, np.float64, "x", dict(fill_value=0, gamma_cap_value=1)),
})

# (function, kwargs, builder name) -> (exception type name, message)
ERROR_CASES = {
    "geometric_not_1d": ("geometric", {}, "2d"),
    "geometric_dta_zero": ("geometric", dict(distance_to_agreement=0), "ok"),
    "geometric_dose_zero": ("geometric", dict(dose_to_agreement=0), "ok"),
    "geometric_non_monotonic": ("geometric", {}, "non_monotonic"),
    "geometric_ref_length": ("geometric", {}, "ref_length"),
    "geometric_eval_length": ("geometric", {}, "eval_length"),
    "geometric_one_sample_eval": ("geometric", {}, "one_sample"),
    "geometric_empty": ("geometric", {}, "empty"),
    "1d_not_1d": ("1d", {}, "2d"),
    "1d_ref_length": ("1d", {}, "ref_length"),
    "1d_eval_length": ("1d", {}, "eval_length"),
    "1d_range": ("1d", {}, "range"),
    "1d_rf0": ("1d", dict(resolution_factor=0), "ok"),
    "1d_rf_2_5": ("1d", dict(resolution_factor=2.5), "ok"),
    "1d_empty": ("1d", {}, "empty"),
    "1d_negative_num": ("1d", dict(distance_to_agreement=-1), "ok"),
}


def _cast(a, dtype):
    if np.issubdtype(dtype, np.integer):
        return np.round(a).astype(dtype)
    return a.astype(dtype)


def case_args(name):
    """-> (function name, reference, evaluation, reference_coordinates, evaluation_coordinates, kwargs)"""
    fn, nr, pr, ne, pe, shift, scale, dtype, coords, kw = CASES[name]
    rng = np.random.default_rng(3000 + sorted(CASES).index(name))
    rx = (np.arange(nr) - (nr - 1) / 2) * pr
    ex = (np.arange(ne) - (ne - 1) / 2) * pe
    width = min(rx.max() - rx.min(), 40.0) * 0.6
    ref = field(rx, width=width) + rng.normal(0, 2, nr)
    ev = field(ex, centre=shift, width=width, scale=1000.0 * scale) + rng.normal(0, 2, ne)
    if name == "1d_nan_eval" or name.startswith("geometric_nan_eval"):
        ev[ne // 2 if name != "geometric_nan_eval_outside" else 2] = np.nan
    if name in ("1d_nan_ref", "geometric_nan_ref_raises"):
        ref[nr // 3] = np.nan
    if name.endswith("edges_clamp"):
        ref[:] = 500 + rng.normal(0, 5, nr)
    ref, ev = _cast(ref, dtype), _cast(ev, dtype)
    if coords == "none":
        return fn, ref, ev, None, None, dict(kw)
    if coords == "int":
        return fn, ref, ev, np.arange(nr) * 3, np.arange(ne) * 3, dict(kw)
    if coords == "dec_eval":
        return fn, ref, ev[::-1].copy(), rx, ex[::-1].copy(), dict(kw)
    if coords == "dec_both":
        return fn, ref[::-1].copy(), ev[::-1].copy(), rx[::-1].copy(), ex[::-1].copy(), dict(kw)
    return fn, ref, ev, rx, ex, dict(kw)


def error_args(name):
    fn, kw, kind = ERROR_CASES[name]
    x = np.arange(20, dtype=float)
    ref, ev, rc, ec = np.linspace(1, 2, 20), np.linspace(1, 2, 20), x, x.copy()
    if kind == "2d":
        ref = np.ones((4, 5))
    elif kind == "non_monotonic":
        rc = x.copy()
        rc[5] = 2
    elif kind == "ref_length":
        rc = x[:-1]
    elif kind == "eval_length":
        ec = x[:-1]
    elif kind == "one_sample":
        ev, ec = np.ones(1), np.zeros(1)
    elif kind == "empty":
        ref, ev, rc, ec = np.ones(0), np.ones(0), np.ones(0), np.ones(0)
    elif kind == "range":
        ec = x[5:]
        ev = ev[5:]
    return fn, ref, ev, rc, ec, dict(kw)


def profile_signal(n, rng, centre=0.0):
    x = np.arange(n) - (n - 1) / 2
    return field(x, centre=centre, width=n * 0.5, penumbra=n / 60) + rng.normal(0, 2, n)


# (method, reference length, reference dpmm, evaluation length, evaluation dpmm, kwargs)
PROFILE_CASES = {
    "fwxm_physical_same_pitch": ("physical", 301, 2.5, 301, 2.5, {}),
    "fwxm_physical_different_pitch": ("physical", 256, 2.55, 320, 2.976, dict(dose_to_agreement=2, distance_to_agreement=1)),
    "fwxm_physical_no_dpmm": ("physical", 201, None, 201, None, dict(distance_to_agreement=2)),
    "fwxm_physical_return_profiles": ("physical", 201, 2.0, 221, 2.2, dict(return_profiles=True)),
    "single_profile": ("single", 201, 2.0, 221, 2.2, {}),
    "single_profile_local": ("single", 201, 2.0, 201, 2.0, dict(global_dose=False, distance_to_agreement=2, dose_to_agreement=2)),
}
