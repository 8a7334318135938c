"""numpy restatement of the frames WinstonLutz.from_cbct analyses (winston_lutz.py:1465-1505), the semantics csrc/stack.cu and
epid_zoom implement on the device:

* np.stack(slices, axis=-1).max(axis=0) / .max(axis=1) of a volume [N, H, W] -> colmax (W, N), rowmax (H, N);
* scipy.ndimage.zoom(p, (1, ratio), grid_mode=True, mode='nearest', order=1) with an integer output: N' = round(N * ratio)
  (Python round), sample o reads position (o + 0.5) * (N / N') - 0.5 clamped to [0, N - 1], weights w0 = 1 - frac, w1 = 1 - w0,
  value = w0 * p[i] + w1 * p[i + 1] (the tap past the end is the edge sample, weight 0), then t + 0.5 (t - 0.5 below zero for a
  signed dtype) clamped to the dtype and truncated toward zero;
* np.rot90(k=1) -> left (from colmax) / top (from rowmax), np.fliplr -> right / bottom;
* array_to_dicom writes the integer bytes with PixelRepresentation 0: the uint16 view of those bits is what is read back.
"""
from __future__ import annotations

import numpy as np


def projections(volume: np.ndarray):
    """-> (colmax (W, N), rowmax (H, N)) in the volume's dtype"""
    np_stack = np.moveaxis(np.asarray(volume), 0, -1)
    return np_stack.max(axis=0), np_stack.max(axis=1)


def zoom_rows(p: np.ndarray, ratio: float) -> np.ndarray:
    """zoom along axis 1 only (axis 0 has factor 1: its taps carry weights 1 and 0 exactly), integer output in p's dtype"""
    n = p.shape[1]
    n_out = int(round(n * ratio))
    z = np.float64(n) / np.float64(n_out)
    cc = (np.arange(n_out, dtype=np.float64) + 0.5) * z - 0.5
    cc = np.clip(cc, 0.0, float(n - 1))
    fl = np.floor(cc)
    t = cc - fl
    w0 = 1.0 - t
    w1 = 1.0 - w0
    i0 = fl.astype(np.int64)
    i1 = np.minimum(i0 + 1, n - 1)
    v = p.astype(np.float64)
    val = w0 * v[:, i0] + w1 * v[:, i1]
    info = np.iinfo(p.dtype)
    if info.min < 0:
        val = np.where(val > 0, val + 0.5, val - 0.5)
    else:
        val = np.where(val > 0, val + 0.5, 0.0)
    val = np.clip(val, info.min, info.max)
    return np.trunc(val).astype(p.dtype)


def cbct_frames(volume: np.ndarray, slice_thickness: float, pixel_spacing: float) -> dict:
    """-> {gantry: uint16 frame} for gantry 270 (left), 0 (top), 90 (right), 180 (bottom)"""
    colmax, rowmax = projections(volume)
    ratio = slice_thickness / pixel_spacing
    left = np.rot90(zoom_rows(colmax, ratio), k=1)
    top = np.rot90(zoom_rows(rowmax, ratio), k=1)
    frames = {270: left, 0: top, 90: np.fliplr(left), 180: np.fliplr(top)}
    return {g: np.ascontiguousarray(a).view(np.uint16) for g, a in frames.items()}
