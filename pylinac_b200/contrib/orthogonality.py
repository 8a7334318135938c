"""Jaw orthogonality of a square field -- drop-in for ``pylinac.contrib.orthogonality.JawOrthogonality`` (contrib/orthogonality.py:14-86).

``analyze()`` = Canny edges of the stretched image, straight-line Hough transform at 0.05 degree steps, the four most prominent
lines, the corner angles between them.  Edge detection, the Hough accumulator and its maximum filter / thresholding run on the
device (``epid_canny``, ``epid_hough_line``, ``epid_hough_candidates``, csrc/edges.cu); grouping the few surviving accumulator cells
into peaks (scikit-image's ``_prominent_peaks`` bookkeeping) is scalar work here.

scikit-image is not available where this was built and the reference holds no test vectors for this class: the three skimage
functions are restated from their published algorithms (parity unpinned; see oracle/edges_oracle.py).  Not here: plotting.
"""
from __future__ import annotations

import numpy as np

from .. import _native as nat
from ..core.array_utils import stretch
from ..core.image import load


def _prominent_peaks(ctx, accum, rows: int, cols: int, min_xdistance: int, min_ydistance: int, threshold=None, num_peaks=np.inf):
    """skimage's _prominent_peaks on a device accumulator: -> (values, column indices, row indices)"""
    cand, gmax, filtered = nat.hough_candidates(ctx, accum, min_xdistance, min_ydistance, threshold)
    with filtered:
        if threshold is None:
            threshold = 0.5 * gmax
        # 8-connected components of the candidate cells (sparse), numbered in raster order of their first cell like skimage.label
        order = np.lexsort((cand[:, 1], cand[:, 0]))
        cand = cand[order]
        index = {(int(y), int(x)): k for k, (y, x, _) in enumerate(cand)}
        parent = list(range(len(cand)))

        def find(a):
            while parent[a] != a:
                parent[a] = parent[parent[a]]
                a = parent[a]
            return a

        for k, (y, x, _) in enumerate(cand):
            for dy, dx in ((0, -1), (-1, -1), (-1, 0), (-1, 1)):
                j = index.get((int(y) + dy, int(x) + dx))
                if j is not None:
                    a, b = find(k), find(j)
                    if a != b:
                        parent[max(a, b)] = min(a, b)
        groups: dict[int, list[int]] = {}
        for k in range(len(cand)):
            groups.setdefault(find(k), []).append(k)
        props = []
        for label, (root, members) in enumerate(sorted(groups.items())):
            cells = cand[members]
            props.append((int(cells[:, 2].max()), float(cells[:, 0].mean()), float(cells[:, 1].mean()), label))
        # sorted(props, key=intensity_max)[::-1]: a stable ascending sort, reversed (ties come out in descending label order)
        props = sorted(props, key=lambda p: p[0])[::-1]
        centers = np.array([[int(np.round(p[1])), int(np.round(p[2]))] for p in props], dtype=np.int32).reshape(-1, 2)
        values = nat.gather_i32(ctx, filtered, centers) if len(centers) else np.zeros(0, np.int32)
    peaks, ys, xs = [], [], []
    zeroed: set[tuple[int, int]] = set()      # accumulator cells an accepted peak has zeroed in the reference's img_max
    yext, xext = np.mgrid[-min_ydistance: min_ydistance + 1, -min_xdistance: min_xdistance + 1]
    for (yi, xi), accum_v in zip(centers, values):
        yi, xi = int(yi), int(xi)
        v = 0 if (yi, xi) in zeroed else int(accum_v)
        if v > threshold:
            # neighbourhood suppression: rows strictly inside (0, rows) without reflection; columns are periodic (angles
            # ..., 89.95, -90, -89.95, ...) with the distance axis mirrored when they wrap
            ynh, xnh = yi + yext, xi + xext
            inside = np.logical_and(ynh > 0, ynh < rows)
            ynh, xnh = ynh[inside], xnh[inside]
            low = xnh < 0
            ynh[low] = rows - ynh[low]
            xnh[low] += cols
            high = xnh >= cols
            ynh[high] = rows - ynh[high]
            xnh[high] -= cols
            zeroed.update(zip(ynh.tolist(), xnh.tolist()))
            peaks.append(v)
            ys.append(yi)
            xs.append(xi)
    peaks, ys, xs = np.array(peaks), np.array(ys, dtype=int), np.array(xs, dtype=int)
    if num_peaks < len(peaks):
        keep = np.argsort(peaks)[::-1][: int(num_peaks)]
        peaks, ys, xs = peaks[keep], ys[keep], xs[keep]
    return peaks, xs, ys


def hough_line_peaks(ctx, accum, angles, dists, min_distance: int = 9, min_angle: int = 10, threshold=None, num_peaks=np.inf):
    """skimage.transform.hough_line_peaks on a device accumulator"""
    (_, rows, cols), _ = accum.shape_dtype
    min_angle = min(min_angle, cols)
    h, a, d = _prominent_peaks(ctx, accum, rows, cols, min_xdistance=min_angle, min_ydistance=min_distance, threshold=threshold, num_peaks=num_peaks)
    if a.size > 0:
        return h, angles[a], dists[d]
    return h, np.array([]), np.array([])


class JawOrthogonality:
    """contrib/orthogonality.py:14-86"""

    line_angles: dict
    result: dict

    def __init__(self, path):
        self.image = load(path)

    def analyze(self):
        ctx = nat.Context.default()
        edge_image = nat.canny(ctx, stretch(np.asarray(self.image.array)))
        self.edge_image = edge_image
        # classic straight-line Hough transform at a precision of 0.05 degree
        tested_angles = np.linspace(-np.pi / 2, np.pi / 2, num=360 * 10, endpoint=False)
        accum, offset = nat.hough_line(ctx, edge_image, tested_angles)
        with accum:
            d = np.linspace(-offset, offset, 2 * offset + 1)
            _, angles, dists = hough_line_peaks(ctx, accum, tested_angles, d)
        if len(angles) < 4:
            raise IndexError(f"only {len(angles)} lines were found; a square field has four")      # the reference fails indexing [2] / [3]
        sorted_idx = np.argsort(np.abs(angles))
        sorted_angles, sorted_dists = angles[sorted_idx], dists[sorted_idx]
        # the two (near-)vertical lines come first, the two horizontal ones last; the smaller distance is left / bottom
        line_angles = {}
        lo, hi = (0, 1) if sorted_dists[0] < sorted_dists[1] else (1, 0)
        line_angles["left"] = {"angle": sorted_angles[lo], "dist": sorted_dists[lo]}
        line_angles["right"] = {"angle": sorted_angles[hi], "dist": sorted_dists[hi]}
        lo, hi = (2, 3) if sorted_dists[2] < sorted_dists[3] else (3, 2)
        line_angles["bottom"] = {"angle": sorted_angles[lo], "dist": sorted_dists[lo]}
        line_angles["top"] = {"angle": sorted_angles[hi], "dist": sorted_dists[hi]}
        ang = lambda a, b: float(np.abs(np.rad2deg(line_angles[a]["angle"] - line_angles[b]["angle"])))      # noqa: E731
        self.line_angles = line_angles
        self.result = {"top_left": ang("left", "top"), "top_right": ang("right", "top"), "bottom_left": ang("left", "bottom"),
                       "bottom_right": ang("right", "bottom")}

    def results(self) -> dict:
        return self.result
