"""Seeded (reference, evaluation) pairs for core.gamma.gamma_2d (reference core/gamma.py:229-330), and the argument errors the
reference raises.  The goldens are the unmodified reference's maps (tests/golden/make_gamma2d_golden.py)."""
from __future__ import annotations

import numpy as np

# name: (shape of the reference, shape of the evaluation or None (same), dtype of the pair (or reference, evaluation), kwargs)
CASES = {
    "defaults_u16": ((41, 37), None, np.uint16, {}),
    "dta0_u16": ((23, 29), None, np.uint16, dict(distance_to_agreement=0)),
    "dta2_cap1_thr0_f64": ((31, 33), None, np.float64, dict(distance_to_agreement=2, gamma_cap_value=1, dose_threshold=0)),
    "dta3_f32": ((37, 41), None, np.float32, dict(distance_to_agreement=3, dose_to_agreement=2)),
    "dta7_fill0_i32": ((29, 43), None, np.int32, dict(distance_to_agreement=7, fill_value=0)),
    "dta20_thr50_f64": ((31, 37), None, np.float64, dict(distance_to_agreement=20, dose_threshold=50, dose_to_agreement=0.5)),
    "dta40_f32": ((47, 53), None, np.float32, dict(distance_to_agreement=40, dose_to_agreement=0.3)),
    "dta40_boundary_f64": ((50, 50), None, np.float64, dict(distance_to_agreement=40)),
    "local_dta1_f64": ((33, 31), None, np.float64, dict(global_dose=False)),
    "local_dta3_u16": ((37, 29), None, np.uint16, dict(global_dose=False, distance_to_agreement=3, dose_to_agreement=3)),
    "local_f32_cap1": ((29, 31), None, np.float32, dict(global_dose=False, distance_to_agreement=2, gamma_cap_value=1)),
    "local_zeros_f64": ((31, 29), None, np.float64, dict(global_dose=False, distance_to_agreement=2, dose_threshold=0)),
    "local_zeros_i32": ((23, 27), None, np.int32, dict(global_dose=False, distance_to_agreement=1, dose_threshold=0)),
    "nan_inf_eval_f64": ((37, 31), None, np.float64, dict(distance_to_agreement=2)),
    "nan_inf_eval_f32": ((29, 37), None, np.float32, dict(distance_to_agreement=3, dose_threshold=0, fill_value=0)),
    "nan_ref_global_f64": ((19, 23), None, np.float64, {}),
    "nan_ref_local_f64": ((31, 29), None, np.float64, dict(global_dose=False, distance_to_agreement=2)),
    "all_zero_ref_f64": ((17, 19), None, np.float64, dict(dose_threshold=0)),
    "all_nan_disk_f64": ((31, 31), None, np.float64, dict(distance_to_agreement=2, dose_threshold=0)),
    "negative_f64": ((29, 31), None, np.float64, dict(distance_to_agreement=3, dose_threshold=0)),
    "negative_local_f32": ((23, 29), None, np.float32, dict(global_dose=False, distance_to_agreement=2, dose_threshold=0)),
    "eval_larger_f64": ((37, 41), (45, 50), np.float64, dict(distance_to_agreement=3)),
    "eval_larger_u16": ((29, 31), (30, 40), np.uint16, dict(distance_to_agreement=7, dose_threshold=0)),
    "row_1xN_u16": ((1, 53), None, np.uint16, dict(distance_to_agreement=3)),
    "col_Nx1_f64": ((47, 1), None, np.float64, dict(distance_to_agreement=2, global_dose=False)),
    "prime_53x59_f64": ((53, 59), None, np.float64, dict(distance_to_agreement=3, dose_threshold=50)),
    "mixed_f32_i32": ((31, 29), None, (np.float32, np.int32), dict(distance_to_agreement=2)),
    "mixed_f32_u16": ((29, 31), None, (np.float32, np.uint16), dict(distance_to_agreement=2, global_dose=False)),
    "mixed_u16_f32": ((27, 33), None, (np.uint16, np.float32), dict(distance_to_agreement=3)),
}

# (reference shape, evaluation shape, kwargs) -> (exception type name, message) as the reference raises them
ERROR_CASES = {
    "ndim_1d": ((7,), (5, 6), {}),
    "dta_negative": ((5, 6), (5, 6), dict(distance_to_agreement=-1)),
    "dta_float": ((5, 6), (5, 6), dict(distance_to_agreement=1.5)),
    "dta_float_integral": ((5, 6), (5, 6), dict(distance_to_agreement=2.0)),
    "dta_bool": ((5, 6), (5, 6), dict(distance_to_agreement=True)),
    "local_shapes": ((5, 6), (6, 6), dict(global_dose=False)),
}


def _field(shape, rng, shift=(0.0, 0.0), scale=1.0):
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cy, cx = (h - 1) / 2 + shift[0], (w - 1) / 2 + shift[1]
    sy, sx = max(h / 3, 1.0), max(w / 3, 1.0)
    return scale * 1000.0 * np.exp(-(((yy - cy) / sy) ** 2 + ((xx - cx) / sx) ** 2)) + rng.normal(0, 4, shape) + 20


def _cast(a, dtype):
    if np.issubdtype(dtype, np.integer):
        return np.round(a).clip(np.iinfo(dtype).min, np.iinfo(dtype).max).astype(dtype)
    return a.astype(dtype)


def case_pair(name):
    """-> (reference, evaluation, kwargs)"""
    rshape, eshape, dtypes, kw = CASES[name]
    rdt, edt = dtypes if isinstance(dtypes, tuple) else (dtypes, dtypes)
    rng = np.random.default_rng(2000 + sorted(CASES).index(name))
    eshape = eshape or rshape
    ref = _field(rshape, rng)
    ev = _field(eshape, rng, shift=(rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5)), scale=rng.uniform(0.97, 1.03))
    ev = ev[:eshape[0], :eshape[1]]
    if name == "dta40_boundary_f64":
        # every evaluation pixel is far off in dose but one, which the reference pixel (5, 3) reaches only through the disk's
        # boundary point (40, 9), a point of the circle r**2 + c**2 == 41**2
        ref = np.full(rshape, 100.0)
        ev = np.full(rshape, 130.0)
        ev[45, 12] = 100.0
    elif name.startswith("local_zeros"):
        ref[rng.random(rshape) < 0.15] = 0
        ev[rng.random(eshape) < 0.05] = 0
    elif name.startswith("nan_inf_eval"):
        ev[rng.random(eshape) < 0.05] = np.nan
        ev[rng.random(eshape) < 0.03] = np.inf
        ev[rng.random(eshape) < 0.02] = -np.inf
    elif name == "nan_ref_global_f64":
        ref[3, 4] = np.nan
    elif name == "nan_ref_local_f64":
        ref[rng.random(rshape) < 0.1] = np.nan
    elif name == "all_zero_ref_f64":
        ref[:] = 0
    elif name == "all_nan_disk_f64":
        ev[8:20, 10:25] = np.nan
    elif name.startswith("negative"):
        ref = ref - 300
        ev = ev - 300
    return _cast(ref, rdt), _cast(ev, edt), dict(kw)
