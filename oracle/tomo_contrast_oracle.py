"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

A numpy restatement of pylinac.nuclear.TomographicContrast (nuclear.py:1553-1856): the slice stage (slice_data), the host selection
and the sphere search.  The search restates scipy 1.18.1's _minimize_neldermead with minimize()'s defaults and bounds, sorting the
simplex with the pinned 4-key argsort of numpy on an AVX-512 host (:func:`argsort4`) instead of np.argsort, so it gives the same answer
on any CPU.  Each objective evaluation sums the sphere over its bounding box only, as the device does.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

# np.argsort of 4 keys on an AVX-512 host differs from a stable sort on these weak orderings (each key's count of smaller keys)
ARGSORT4_EXCEPTIONS = {(2, 2, 0, 0): (3, 2, 1, 0), (2, 3, 0, 0): (3, 2, 0, 1), (3, 2, 0, 0): (3, 2, 1, 0), (2, 2, 0, 1): (2, 3, 1, 0),
                       (2, 2, 1, 0): (3, 2, 1, 0)}


def argsort4(f) -> list[int]:
    """np.argsort of 4 float64 keys as numpy 2.3 sorts them on an AVX512_SKX host: stable with nans last, except the weak
    orderings of ARGSORT4_EXCEPTIONS"""
    f = [float(v) for v in f]
    if not any(math.isnan(v) for v in f):
        key = tuple(sum(b < a for b in f) for a in f)
        if key in ARGSORT4_EXCEPTIONS:
            return list(ARGSORT4_EXCEPTIONS[key])
    return sorted(range(4), key=lambda i: (math.isnan(f[i]), 0.0 if math.isnan(f[i]) else f[i]))


def michelson(a, b) -> float:
    """pylinac.core.contrast.michelson(np.asarray([a, b])) without its warnings: nan for two nans"""
    v = [x for x in (a, b) if not math.isnan(x)]
    if not v:
        return math.nan
    mx, mn = np.float64(max(v)), np.float64(min(v))
    with np.errstate(invalid="ignore", divide="ignore"):
        return float((mx - mn) / (mx + mn))


def slice_rows(volume: np.ndarray, ufov_ratio: float = 0.8) -> list[dict]:
    """the per-slice quantities of slice_data before the area filter; None for a slice with no component"""
    gmax = volume.max()
    thr = float(gmax) * 0.10
    rows = []
    for frame in volume:
        arr = np.where(frame.astype(np.float64) < thr, 0, frame).astype(np.int64)
        binary = arr > 0
        lab, num = ndimage.label(binary, ndimage.generate_binary_structure(2, 1))
        if num < 1:
            rows.append(None)
            continue
        areas = np.bincount(lab.ravel())[1:]
        big = int(np.argmax(areas)) + 1                      # the first label of the largest area
        rr, cc = np.nonzero(lab == big)
        longest = max(int(rr.max() - rr.min() + 1), int(cc.max() - cc.min() + 1))
        erosion = int(round((1 - ufov_ratio) * longest))
        d2 = ndimage.distance_transform_edt(binary, return_distances=False, return_indices=True)
        d2 = (d2[0] - np.arange(binary.shape[0])[:, None]) ** 2 + (d2[1] - np.arange(binary.shape[1])[None, :]) ** 2
        eroded = np.ones_like(binary) if erosion < 0 else 4 * d2 > erosion * erosion
        vals = arr[eroded]
        n = int(vals.size)
        row = {"longest": longest, "erosion": erosion, "area": n, "centroid_row": float(np.float64(rr.sum()) / np.float64(rr.size)),
               "centroid_col": float(np.float64(cc.sum()) / np.float64(cc.size)), "sum": int(vals.sum()), "count": n}
        if n:
            mx, mn = int(vals.max()), int(vals.min())
            row.update(uniformity=float(np.float64(mx - mn) / np.float64(mx + mn)), value=float(np.float64(row["sum"]) / np.float64(n)),
                       max=mx, min=mn)
        else:
            row.update(uniformity=math.nan, value=math.nan, max=0, min=0)
        rows.append(row)
    return rows


def sphere_stats(volume: np.ndarray, col: float, row: float, zed: float, r2: float) -> tuple[int, int, int]:
    """(sum, count, min) of the voxels with ((x - col)**2 + (y - row)**2) + (z - zed)**2 <= r2, enumerated over the sphere's
    bounding box clipped to the volume"""
    nz, h, w = volume.shape
    r = math.sqrt(r2) + 1
    lo = [max(int(math.floor(c - r)), 0) for c in (zed, row, col)]
    hi = [min(int(math.ceil(c + r)), s - 1) for c, s in zip((zed, row, col), (nz, h, w))]
    if any(a > b for a, b in zip(lo, hi)):
        return 0, 0, 0
    z, y, x = np.ogrid[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1]
    mask = ((x - col) ** 2 + (y - row) ** 2) + (z - zed) ** 2 <= r2
    v = volume[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1][mask].astype(np.int64)
    return (int(v.sum()), int(v.size), int(v.min())) if v.size else (0, 0, 0)


def objective(volume, x, r2, baseline) -> tuple[float, bool]:
    """(contrast_f, whether the sphere was empty)"""
    s, n, _ = sphere_stats(volume, x[0], x[1], x[2], r2)
    mean = float(np.float64(s) / np.float64(n)) if n else math.nan
    return -michelson(mean, baseline) * 100, n == 0


def nelder_mead(func, x0, lb, ub, maxfun=600, maxiter=600) -> dict:
    """scipy's _minimize_neldermead (N = 3, default options, bounds) with the pinned argsort4"""
    xatol = fatol = 1e-4
    lb, ub = np.asarray(lb, float), np.asarray(ub, float)
    x0 = np.clip(np.asarray(x0, float), lb, ub)
    sim = np.empty((4, 3))
    sim[0] = x0
    for k in range(3):
        y = x0.copy()
        y[k] = (1 + 0.05) * y[k] if y[k] != 0 else 0.00025
        sim[k + 1] = y
    sim = np.clip(np.where(sim > ub, 2 * ub - sim, sim), lb, ub)
    fsim = np.full(4, np.inf)
    fcalls = [0]

    class MaxCalls(Exception):
        pass

    def f(x):
        if fcalls[0] >= maxfun:
            raise MaxCalls
        fcalls[0] += 1
        return func(np.copy(x))

    def order():
        nonlocal sim, fsim
        ind = argsort4(fsim)
        sim, fsim = sim[ind], fsim[ind]

    try:
        for k in range(4):
            fsim[k] = f(sim[k])
    except MaxCalls:
        pass
    order()
    order()
    iterations = 1
    while fcalls[0] < maxfun and iterations < maxiter:
        try:
            if np.max(np.abs(sim[1:] - sim[0])) <= xatol and np.max(np.abs(fsim[0] - fsim[1:])) <= fatol:
                break
            xbar = np.add.reduce(sim[:-1], 0) / 3
            xr = np.clip(2 * xbar - sim[-1], lb, ub)
            fxr = f(xr)
            if fxr < fsim[0]:
                xe = np.clip(3 * xbar - 2 * sim[-1], lb, ub)
                fxe = f(xe)
                sim[-1], fsim[-1] = (xe, fxe) if fxe < fxr else (xr, fxr)
            elif fxr < fsim[-2]:
                sim[-1], fsim[-1] = xr, fxr
            else:
                if fxr < fsim[-1]:
                    xc = np.clip(1.5 * xbar - 0.5 * sim[-1], lb, ub)
                    fxc = f(xc)
                    shrink = not fxc <= fxr
                else:
                    xc = np.clip(0.5 * xbar + 0.5 * sim[-1], lb, ub)
                    fxc = f(xc)
                    shrink = not fxc < fsim[-1]
                if not shrink:
                    sim[-1], fsim[-1] = xc, fxc
                else:
                    for j in range(1, 4):
                        sim[j] = np.clip(sim[0] + 0.5 * (sim[j] - sim[0]), lb, ub)
                        fsim[j] = f(sim[j])
            iterations += 1
        except MaxCalls:
            pass
        order()
    status = 1 if fcalls[0] >= maxfun else (2 if iterations >= maxiter else 0)
    return {"x": sim[0].copy(), "fun": float(np.min(fsim)), "nfev": fcalls[0], "nit": iterations, "status": status}


def analyze(volume: np.ndarray, pixel_size: float, sphere_diameters_mm=(38, 31.8, 25.4, 19.1, 15.9, 12.7),
            sphere_angles=(-10, -70, -130, -190, 110, 50), ufov_ratio=0.8, search_window_px=5, search_slices=3, maxfun=600,
            maxiter=600) -> dict:
    """TomographicContrast.analyze on one [z, h, w] volume: {"rows", "slice_data", "uniformity_frame", "baseline", "spheres"}; each
    sphere {"x", "nfev", "nit", "status", "n_empty", "sum", "count", "min", "radius"}.  Raises the reference's ValueErrors."""
    rows = slice_rows(volume, ufov_ratio)
    unif = {str(i + 1): r for i, r in enumerate(rows) if r is not None}
    areas = [v["area"] for v in unif.values()]
    with np.errstate(all="ignore"):
        import warnings

        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            median_area, std_area = np.median(areas), np.std(areas)
    data = {k: v for k, v in unif.items() if v["area"] > median_area - std_area}
    if len(sphere_diameters_mm) != len(sphere_angles):
        raise ValueError("The number of sphere diameters and angles must be the same.")
    start = max(data, key=lambda k: data[k]["uniformity"])
    frame = min(data, key=lambda k: data[k]["uniformity"])
    baseline = data[frame]["value"]
    u = data[start]
    unif_z = int(start) - 1
    spheres = []
    for angle, diameter in zip(sphere_angles, sphere_diameters_mm):
        distance = math.sqrt(u["area"] / math.pi) * 0.65
        radius = diameter / (2 * pixel_size)
        a = math.radians(angle)
        col_x = u["centroid_col"] + distance * math.cos(a)
        row_y = u["centroid_row"] + distance * math.sin(a)
        r2 = radius ** 2
        empty = [0]

        def func(x, r2=r2, empty=empty):
            v, e = objective(volume, x, r2, baseline)
            empty[0] += e
            return v

        res = nelder_mead(func, (col_x, row_y, unif_z), (col_x - search_window_px, row_y - search_window_px, unif_z - search_slices),
                          (col_x + search_window_px, row_y + search_window_px, unif_z + search_slices), maxfun, maxiter)
        s, n, mn = sphere_stats(volume, *res["x"], r2)
        spheres.append({**res, "n_empty": empty[0], "sum": s, "count": n, "min": mn, "radius": radius})
    return {"rows": rows, "slice_data": data, "uniformity_frame": frame, "baseline": baseline, "spheres": spheres}
