"""numpy restatement of pylinac.core.gamma.gamma_geometric and gamma_1d (reference core/gamma.py:16-226, 333-460) with no BLAS in
the segment distance: the 2-element dot products are an emulated fma(x1, y1, x0 * y0), math.dist is CPython 3.12's vector_norm
restated, and the window search is a bisection.  gamma_1d squares by multiplying (the reference's ``**2`` is libm pow)."""
from __future__ import annotations

import numpy as np

_DBL_MIN = np.finfo(np.float64).tiny


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a                      # 2**27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma(a, b, c):
    """correctly rounded a * b + c (Boldo and Melquiond, "Emulation of FMA and correctly rounded sums", 2008: the low parts are
    added with rounding to odd); finite operands whose product does not underflow"""
    a, b, c = (np.asarray(v, dtype=np.float64) for v in (a, b, c))
    with np.errstate(all="ignore"):
        ph, pl = _two_prod(a, b)
        uh, ul = _two_sum(c, ph)
        v, err = _two_sum(ul, pl)
        bits = v.view(np.int64)
        odd = (bits & 1) == 1
        fix = (err != 0) & ~odd & np.isfinite(v)
        v = np.where(fix, np.nextafter(v, np.where(err > 0, np.inf, -np.inf)), v)
        r = uh + v
        exact = a * b + c
        return np.where(np.isfinite(r) & np.isfinite(ph) & (ph != 0), r, exact)


def py_dist(px, py, qx, qy):
    """math.dist((px, py), (qx, qy)) of CPython 3.12, elementwise"""
    a, b = np.abs(np.asarray(px, np.float64) - qx), np.abs(np.asarray(py, np.float64) - qy)
    with np.errstate(all="ignore"):
        mx = np.maximum(np.where(a > 0, a, 0.0), np.where(b > 0, b, 0.0))
        mx = np.where(np.isnan(mx), 0.0, mx)
        sub = mx < _DBL_MIN
        unscale = np.where(sub & (mx > 0), _DBL_MIN, 1.0)
        a, b, m = a / unscale, b / unscale, mx / unscale
        _, e = np.frexp(np.where(m > 0, m, 1.0))
        scale = np.ldexp(1.0, -e)
        csum, frac1, frac2 = np.ones_like(a), np.zeros_like(a), np.zeros_like(a)

        def add(x, y, csum, frac1, frac2):
            hi, lo = _two_prod(x, y)
            s = csum + hi
            return s, frac1 + lo, frac2 + ((csum - s) + hi)

        csum, frac1, frac2 = add(a * scale, a * scale, csum, frac1, frac2)
        csum, frac1, frac2 = add(b * scale, b * scale, csum, frac1, frac2)
        h = np.sqrt(csum - 1.0 + (frac1 + frac2))
        csum, frac1, frac2 = add(-h, h, csum, frac1, frac2)
        x = csum - 1.0 + (frac1 + frac2)
        h = h + x / (2.0 * h)
        r = unscale * (h / scale)
        r = np.where(mx == 0, 0.0, r)
        r = np.where(np.isnan(a) | np.isnan(b), np.nan, r)
        return np.where(np.isinf(mx), mx, r)


def segment_distance(px, py, v1x, v1y, v2x, v2y):
    """_compute_distance(p, [v1, v2]) elementwise -> (distance, vtv is nan: the reference's pinv raises)"""
    with np.errstate(all="ignore"):
        a0, a1, p0, p1 = v1x - v2x, v1y - v2y, px - v2x, py - v2y
        vtv = fma(a1, a1, a0 * a0)
        inv = np.where(vtv == 0, 0.0, 1.0 / np.where(vtv == 0, 1.0, vtv))
        w0 = inv * fma(a1, p1, a0 * p0)
        w1 = 1.0 - w0
        d1, d2 = py_dist(px, py, v1x, v1y), py_dist(px, py, v2x, v2y)
        outside = np.where(d2 < d1, d2, d1)
        q0, q1 = w0 * v1x + w1 * v2x, w0 * v1y + w1 * v2y
        e0, e1 = px - q0, py - q1
        inside = np.sqrt(fma(e1, e1, e0 * e0))
        return np.where((w0 < 0) | (w1 < 0), outside, inside), np.isnan(vtv)


def argmin_abs(x: np.ndarray, t: float, dec: bool) -> int:
    """np.argmin(np.abs(x - t)) over a strictly monotonic x by two bisections (the device's search)"""
    if np.isnan(t):
        return 0
    m = len(x)
    lo, hi = 0, m
    while lo < hi:
        mid = (lo + hi) // 2
        if (x[mid] <= t) if dec else (x[mid] >= t):
            hi = mid
        else:
            lo = mid + 1
    p = lo
    best = np.inf
    if p < m:
        best = abs(x[p] - t)
    if p > 0 and abs(x[p - 1] - t) < best:
        best = abs(x[p - 1] - t)
    lo, hi = 0, p
    while lo < hi:
        mid = (lo + hi) // 2
        if abs(x[mid] - t) <= best:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _py_min(v: np.ndarray) -> float:
    """Python's min() of a sequence: nan iff the first item is nan, else the least non-nan item"""
    return np.nan if np.isnan(v[0]) else np.nanmin(v)


def gamma_geometric(reference, evaluation, reference_coordinates=None, evaluation_coordinates=None, dose_to_agreement=1,
                    distance_to_agreement=1, gamma_cap_value=2, dose_threshold=5, fill_value=np.nan):
    rc = np.arange(len(reference), dtype=float) if reference_coordinates is None else reference_coordinates
    ec = np.arange(len(evaluation), dtype=float) if evaluation_coordinates is None else evaluation_coordinates
    threshold = float(dose_threshold) / float(dose_to_agreement)
    nr = reference.astype(float) * 100 / (reference.max() * dose_to_agreement)
    ne = evaluation.astype(float) * 100 / (reference.max() * dose_to_agreement)
    nrx, nex = rc / distance_to_agreement, ec / distance_to_agreement
    dec = bool(np.all(np.diff(nex) < 0))
    gamma = np.full(len(reference), fill_value)
    for i in range(len(reference)):
        rx, rp = float(nrx[i]), float(nr[i])
        if rp < threshold:
            continue
        tl, tr = rx - distance_to_agreement, rx + distance_to_agreement
        if dec:
            tl, tr = tr, tl
        left = max(argmin_abs(nex, tl, dec) - 1, 0)
        right = min(argmin_abs(nex, tr, dec) + 1, len(ne) - 1)
        j = np.arange(left, right)
        d, bad = segment_distance(rx, rp, nex[j], ne[j], nex[j + 1], ne[j + 1])
        if bad.any():
            raise np.linalg.LinAlgError("SVD did not converge")
        g = _py_min(d)
        gamma[i] = gamma_cap_value if gamma_cap_value < g else g
    return gamma


def gamma_1d(reference, evaluation, reference_coordinates=None, evaluation_coordinates=None, dose_to_agreement=1,
             distance_to_agreement=1, gamma_cap_value=2, global_dose=True, dose_threshold=5, resolution_factor=3, fill_value=np.nan):
    rc = np.arange(len(reference), dtype=float) if reference_coordinates is None else reference_coordinates
    ec = np.arange(len(evaluation), dtype=float) if evaluation_coordinates is None else evaluation_coordinates
    threshold = reference.max() / 100 * dose_threshold
    dose_ta = dose_to_agreement / 100 * reference.max()
    order = np.argsort(ec, kind="mergesort")
    x, y = ec[order].astype(np.float64), evaluation[order].astype(np.float64)
    m = len(x)
    num = int(distance_to_agreement * resolution_factor * 2 + 1)
    dta2 = float(distance_to_agreement ** 2)
    single = np.result_type(dose_ta) == np.float32
    gamma, samples, xs = [], [], []
    with np.errstate(all="ignore"):
        for rx, rp in zip(rc, reference):
            if rp < threshold:
                gamma.append(fill_value)
                continue
            s = np.linspace(rx - distance_to_agreement, rx + distance_to_agreement, num=num)
            i = np.clip(np.searchsorted(x, s), 1, m - 1)
            lo, hi = i - 1, i
            v = ((s - x[lo]) / (x[hi] - x[lo])) * y[hi] + ((x[hi] - s) / (x[hi] - x[lo])) * y[lo]
            samples.extend(v)
            xs.extend(s)
            dist, dose = np.abs(float(rx) - s), float(rp) - v
            if global_dose:
                dd2 = dose_ta ** 2
            else:
                dd2 = (dose_to_agreement / 100 * rp) ** 2
            t2 = (dose * dose).astype(np.float32) / np.float32(dd2) if single else dose * dose / float(dd2)
            cg = np.sqrt(dist * dist / dta2 + t2.astype(np.float64))
            g = _py_min(cg)
            gamma.append(gamma_cap_value if gamma_cap_value < g else float(g))
    return np.asarray(gamma), np.asarray(samples, dtype=np.float64), np.asarray(xs, dtype=np.float64)
