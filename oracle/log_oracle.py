"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

A numpy statement of ``FluenceBase.calc_map`` (log_analyzer.py:478-612) and of the fluence gamma statistics (:736-748), written
from the arrays a parsed log exposes.  Pinned bit for bit to the goldens of the unmodified reference (tests/golden/log_golden.npz)
on the CPU; the GPU tests run seeded fuzz against it, since the reference does not exist there.
"""
from __future__ import annotations

import numpy as np

WIDTH_MM, HEIGHT_MM, HD_HEIGHT_MM = 400, 400, 220


def leaf_rows(hdmlc: bool, resolution: float) -> np.ndarray:
    large, small = (5 / resolution, 2.5 / resolution) if hdmlc else (10 / resolution, 5 / resolution)
    nl, ns = (14, 32) if hdmlc else (10, 40)
    return np.cumsum([0] + [large] * nl + [small] * ns + [large] * nl).astype(int)


def under_y_jaw(pair: int, hdmlc: bool, y1_max: float, y2_max: float) -> bool:
    outer, inner, pos = (5.0, 2.5, 100) if hdmlc else (10, 5, 0)
    th = outer
    for leaf in range(1, pair + 1):
        th = outer if (leaf <= 10 or leaf >= 110) else (inner if (leaf <= 50 or leaf >= 70) else outer)
        pos += th
    return pos < 200 - y1_max * 10 or pos - th > y2_max * 10 + 200


def fluence(mu: np.ndarray, x1: np.ndarray, x2: np.ndarray, right: np.ndarray, left: np.ndarray, snapshot_idx, moved: np.ndarray,
            under_jaw: np.ndarray, hdmlc: bool, resolution: float, equal_aspect: bool) -> np.ndarray:
    """mu [nsnap]; x1 / x2 jaw actual [nsnap]; right / left leaf positions [nsnap, pairs] (bank A / bank B of the kind);
    moved / under_jaw [pairs] bool -> the float64 map"""
    npairs = right.shape[1]
    W = int(WIDTH_MM / resolution)
    R = int((HD_HEIGHT_MM if hdmlc else HEIGHT_MM) / resolution) if equal_aspect else npairs
    out = np.zeros((R, W))
    sidx = np.asarray(snapshot_idx, dtype=np.int64).reshape(-1)
    if len(sidx) < 1 or np.max(mu) < 0.5:
        return out
    rows = leaf_rows(hdmlc, resolution)
    dmu = np.concatenate([[mu[0]], np.diff(mu)])
    total = mu[-1]
    off = int(np.round(200 / resolution))
    ljaw = np.round((200 / resolution) - (x1 * 10 / resolution))
    rjaw = np.round((x2 * 10 / resolution) + (200 / resolution))
    line = np.zeros(W, np.float32)
    for p in range(npairs):
        if under_jaw[p]:
            continue
        line[:] = 0
        rt = np.round(right[:, p] * 10 / resolution) + off
        lt = -np.round(left[:, p] * 10 / resolution) + off
        if moved[p]:
            a = np.maximum(lt[sidx], ljaw[sidx])
            b = np.minimum(rt[sidx], rjaw[sidx])
            for s, lo, hi in zip(sidx, a, b):
                line[int(lo) : int(hi)] += dmu[s]
        else:
            s0 = sidx[0]
            lo, hi = max(lt[s0], ljaw.min()), min(rt[s0], rjaw.max())
            line[int(lo) : int(hi)] = total
        if equal_aspect:
            out[rows[p] : rows[p + 1], :] = line
        else:
            out[p, :] = line
    if total == 25000:
        out /= total
    return out


def fluence_of(fl, resolution: float, equal_aspect: bool = False) -> np.ndarray:
    """the map of a fluence object (ActualFluence / ExpectedFluence of pylinac_b200.log_analyzer or of the reference)"""
    mlc, kind = fl._mlc, fl.FLUENCE_TYPE
    n = mlc.num_pairs
    right = np.stack([getattr(mlc.leaf_axes[p], kind) for p in range(1, n + 1)], axis=1)
    left = np.stack([getattr(mlc.leaf_axes[p + n], kind) for p in range(1, n + 1)], axis=1)
    moved = np.array([mlc.pair_moved(p) for p in range(1, n + 1)], bool)
    y1m, y2m = fl._jaws.y1.actual.max(), fl._jaws.y2.actual.max()
    under = np.array([under_y_jaw(p, mlc.hdmlc, y1m, y2m) for p in range(1, n + 1)], bool)
    return fluence(getattr(fl._mu, kind), fl._jaws.x1.actual, fl._jaws.x2.actual, right, left, mlc.snapshot_idx, moved, under, mlc.hdmlc,
                   resolution, equal_aspect)


def gamma_stats(gamma_map: np.ndarray):
    """(avg_gamma, pass_prcnt) of a gamma map with nan below the threshold (log_analyzer.py:743-748)"""
    with np.errstate(invalid="ignore", divide="ignore"):
        ok = gamma_map[~np.isnan(gamma_map)]
        avg = np.sum(ok) / ok.size if ok.size else 0
        return avg, np.sum(ok < 1) / np.sum(ok >= 0) * 100
