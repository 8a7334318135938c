"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

numpy restatement of pylinac.nuclear.TomographicUniformity (nuclear.py:1370-1551 on top of PlanarUniformity, nuclear.py:274-500)
with its intermediates, for the golden checks and the seeded stage fuzz of tests/test_gpu_tomo_uniformity.py.  The slab mean is a
float64 frame, so every sum after it rounds: this oracle writes each one in the summation order numpy and scipy use, which the device
reproduces (DESIGN.md section 4.16):

- :func:`pw` is numpy's pairwise sum (``pairwise_sum`` of numpy's loops); ``np.sum`` of a C-contiguous array is ``0 + pw(flat)``.
- :func:`block_sum` is skimage's ``block_reduce(func=np.sum)``: per block, ``acc = 0; acc += pw(row)`` for each of its rows.
- :func:`nema_filter` is ``convolve2d(a, kernel / 16, "same")``: the flipped kernel in raster order from 0.

Everything after the threshold is decided on ``array > 0``, so the FOV stages are oracle/nuclear_oracle.py's.
"""
from __future__ import annotations

import numpy as np

from oracle import nuclear_oracle as nm


def slab(n: int, first: int, last: int) -> tuple[int, int]:
    """analyze()'s frame checks in the reference's order: (first, last) of the slab [first, last), which may be empty"""
    if first < 0:
        raise ValueError("The first frame index is outside the array bounds. Increase the first frame index.")
    if last < 0:
        last += n
    if last >= n:
        raise ValueError("The last frame index is outside the array bounds. Decrease the last frame index.")
    if 0 < last <= first:
        raise ValueError("The first frame index must be less than the last frame index.")
    return first, last


def pw(x: np.ndarray) -> np.ndarray:
    """numpy's pairwise sum along the last axis, vectorised over the others"""
    x = np.asarray(x, np.float64)
    n = x.shape[-1]
    if n < 8:
        res = np.full(x.shape[:-1], -0.0)
        for i in range(n):
            res = res + x[..., i]
        return res
    if n <= 128:
        r = x[..., 0:8].copy()
        i = 8
        while i < n - n % 8:
            r = r + x[..., i:i + 8]
            i += 8
        res = ((r[..., 0] + r[..., 1]) + (r[..., 2] + r[..., 3])) + ((r[..., 4] + r[..., 5]) + (r[..., 6] + r[..., 7]))
        for k in range(i, n):
            res = res + x[..., k]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pw(x[..., :n2]) + pw(x[..., n2:])


def np_sum(a: np.ndarray) -> np.float64:
    """np.sum of a C-contiguous array: 0 + pw(the flattened array)"""
    return np.float64(0.0) + pw(np.ascontiguousarray(a).ravel())


def slab_mean(volume: np.ndarray, first: int, last: int) -> np.ndarray:
    """array[first:last].mean(axis=0): the exact integer sum over the slab, divided once"""
    t = volume[first:last].astype(np.int64).sum(axis=0)
    return t.astype(np.float64) / np.float64(last - first)


def block_sum(m: np.ndarray, b: int) -> np.ndarray:
    """block_reduce(m, (b, b), np.sum) with the bottom / right edges zero-padded"""
    h, w = m.shape
    hb, wb = -(-h // b), -(-w // b)
    p = np.zeros((hb * b, wb * b))
    p[:h, :w] = m
    blocks = p.reshape(hb, b, wb, b)
    acc = np.zeros((hb, wb))
    for r in range(b):
        acc = acc + pw(blocks[:, r, :, :])
    return acc


def nema_filter(binned: np.ndarray) -> np.ndarray:
    """convolve2d(binned, [[1,2,1],[2,4,2],[1,2,1]] / 16, "same") in scipy's order, then the outer rows and columns zeroed"""
    hb, wb = binned.shape
    out = np.zeros((hb, wb))
    if hb >= 3 and wb >= 3:
        acc = np.zeros((hb - 2, wb - 2))
        for di in (1, 0, -1):
            for dj in (1, 0, -1):
                k = (2.0 - abs(di)) * (2.0 - abs(dj)) / 16.0
                acc = acc + binned[1 + di:hb - 1 + di, 1 + dj:wb - 1 + dj] * k
        out[1:-1, 1:-1] = acc
    return out


def clean(filtered: np.ndarray, threshold: float) -> tuple[np.ndarray, float]:
    """the threshold at `threshold` x the mean of the values above 10 % of the max, then remove_small_objects(min_size=2)"""
    a = filtered.copy()
    t10 = np.max(a) * 0.10
    sel = a[a > t10]
    thr = np.float64(pw(sel) + 0.0) / np.float64(sel.size) * threshold if sel.size else np.nan
    a[a < thr] = 0
    b = a > 0
    nb = np.zeros_like(b)
    nb[1:] |= b[:-1]
    nb[:-1] |= b[1:]
    nb[:, 1:] |= b[:, :-1]
    nb[:, :-1] |= b[:, 1:]
    a[~(b & nb)] = 0
    return a, thr


def nanmean_zero_outside(values: np.ndarray, keep: np.ndarray) -> tuple[float, int]:
    """(sum, count) of np.nanmean over `values` with nan outside `keep`: the sum is pw over the whole frame, zeros outside"""
    return float(np_sum(np.where(keep, values, 0.0))), int(keep.sum())


def analyze(volume: np.ndarray, pixel_size: float, first: int, last: int, ufov_ratio=0.8, cfov_ratio=0.75, center_ratio=0.4,
            threshold=0.75, window_size=5) -> dict:
    """The slab [first, last) of `volume` (first / last already checked, the slab not empty): the stage planes and, when the frame
    has a component, the three FOVs (nuclear_oracle.fov + uniformity) and the center / ring sums."""
    b = nm.determine_binning(pixel_size)
    out = {"bin": b, "mean": slab_mean(volume, first, last)}
    out["binned"] = block_sum(out["mean"], b)
    out["filtered"] = nema_filter(out["binned"])
    out["cleaned"], out["threshold"] = clean(out["filtered"], threshold)
    binary = out["cleaned"] > 0
    out["edt2"] = nm.squared_edt(binary)
    if not binary.any():
        out["status"] = "no_component"
        return out
    out["status"] = "ok"
    sizes = {"ufov": ufov_ratio, "cfov": cfov_ratio * ufov_ratio, "center_fov": center_ratio * ufov_ratio}
    for name, size in sizes.items():
        f = nm.fov(out["cleaned"], size)
        f.update(nm.uniformity(f["fov"], window_size))
        out[name] = f
    c = out["cleaned"]
    out["center"] = nanmean_zero_outside(c, out["center_fov"]["mask"] & (c > 0))
    out["ring"] = nanmean_zero_outside(c, out["ufov"]["mask"] & (c > 0) & ~(out["cfov"]["mask"] & (c > 0)))
    cs, cn = out["center"]
    rs, rn = out["ring"]
    cm = np.float64(cs) / np.float64(cn) if cn else np.nan
    rm = np.float64(rs) / np.float64(rn) if rn else np.nan
    out["center_border_ratio"] = float(cm / rm)
    return out
