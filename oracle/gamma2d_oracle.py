"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

Vectorised numpy restatement of ``pylinac.core.gamma.gamma_2d`` (reference core/gamma.py:229-330, Low et al. 2004, Table I).  The
reference loops over the reference pixels and takes an ``np.nanmin`` over the disk of evaluation samples around each; here the loop
runs over the disk offsets instead and every pixel is updated at once, with the same expressions on the same dtypes (numpy 2
promotion: a float32 reference keeps the normalised doses, the dose difference and its square in float32, the sum with the fp64
distance term is fp64).  ``np.fmin`` is ``nanmin`` taken one offset at a time: the minimum is exact, so the order does not matter.

``offsets_visited`` counts the terms the device kernel evaluates per pixel with its exact early exit (offsets sorted by distance,
stop once the next distance alone reaches min(best, cap**2)), so that the saving of the early exit is a computed number.
"""
from __future__ import annotations

import numpy as np

from oracle.skimage_draw import disk


def _normalised(reference, evaluation, dose_to_agreement, global_dose):
    if global_dose:
        dose_ta = dose_to_agreement / 100 * reference.max()
    else:
        dose_ta = dose_to_agreement / 100 * reference
    return evaluation / dose_ta, reference / dose_ta


def _terms(reference, evaluation, dose_to_agreement, distance_to_agreement, global_dose, dose_threshold):
    """(ref_n, skip mask, padded eval_n, disk rows, disk cols, dist_r_2)"""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        eval_n, ref_n = _normalised(reference, evaluation, dose_to_agreement, global_dose)
        skip = np.isnan(ref_n) | (ref_n < dose_threshold / 100)
        dta = distance_to_agreement
        pad = np.pad(eval_n, dta, mode="edge")
        rr, cc = disk((0, 0), dta + 1)
        d2 = (rr / dta) ** 2 + (cc / dta) ** 2
    return ref_n, skip, pad, rr, cc, d2


def gamma_2d(reference, evaluation, dose_to_agreement=1, distance_to_agreement=1, gamma_cap_value=2, global_dose=True,
             dose_threshold=5, fill_value=np.nan):
    ref_n, skip, pad, rr, cc, d2 = _terms(reference, evaluation, dose_to_agreement, distance_to_agreement, global_dose,
                                          dose_threshold)
    h, w = reference.shape
    dta = distance_to_agreement
    best = np.full((h, w), np.nan)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(len(rr)):
            roi = pad[dta + rr[k]:dta + rr[k] + h, dta + cc[k]:dta + cc[k] + w]
            d = roi - ref_n
            best = np.fmin(best, d2[k] + d * d)
        out = np.full((h, w), float(gamma_cap_value))
        calc = ~skip & ~(best >= gamma_cap_value ** 2)
        out[calc] = np.sqrt(best[calc])
    out[skip] = fill_value
    return out


def offsets_visited(reference, evaluation, dose_to_agreement=1, distance_to_agreement=1, gamma_cap_value=2, global_dose=True,
                    dose_threshold=5):
    """-> (int64 [h, w] terms evaluated per pixel with the early exit (0 below the threshold), disk size)"""
    ref_n, skip, pad, rr, cc, d2 = _terms(reference, evaluation, dose_to_agreement, distance_to_agreement, global_dose,
                                          dose_threshold)
    order = np.argsort(d2, kind="stable")
    h, w = reference.shape
    dta = distance_to_agreement
    cap2 = gamma_cap_value ** 2
    best = np.full((h, w), np.nan)
    active = ~skip
    visited = np.zeros((h, w), np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in order:
            active &= ~(~np.isnan(best) & (d2[k] >= np.fmin(best, cap2)))
            if not active.any():
                break
            visited += active
            roi = pad[dta + rr[k]:dta + rr[k] + h, dta + cc[k]:dta + cc[k] + w]
            d = roi - ref_n
            best = np.where(active, np.fmin(best, d2[k] + d * d), best)
    return visited, len(rr)
