"""TEST INFRASTRUCTURE ONLY -- never imported by the product (pylinac_b200/).

numpy / scipy restatement of pylinac.nuclear's PlanarUniformity frame pipeline (preprocess + get_fov + FOV properties,
nuclear.py:151-500) with its intermediates, for the golden checks and the seeded fuzz of tests/test_gpu_nuclear.py.  It follows the
reference line for line in float64 (skimage calls as restated in oracle/skimage_nuclear.py) and reports the integer stage planes the
device computes: S = 16 x the filtered value, and the exact squared EDT.
"""
from __future__ import annotations

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view
from scipy import ndimage
from scipy.signal import convolve2d

from oracle import skimage_nuclear as sk


def determine_binning(pixel_size: float) -> int:
    binning = 1
    while pixel_size < 4.48:
        pixel_size *= 2
        binning *= 2
    return binning


def preprocess(frame: np.ndarray, bin_size: int, threshold: float) -> dict:
    array = sk.block_reduce(np.copy(frame), block_size=(bin_size, bin_size), func=np.sum)
    kernel = np.array([[1, 2, 1], [2, 4, 2], [1, 2, 1]], dtype=float)
    kernel /= kernel.sum()
    array = convolve2d(array, kernel, mode="same")
    array[0, :] = 0
    array[-1, :] = 0
    array[:, 0] = 0
    array[:, -1] = 0
    filtered = array.copy()
    with np.errstate(invalid="ignore", divide="ignore"):
        sel = array[array > np.max(array) * 0.10]
        thr = sel.mean() * threshold if sel.size else np.nan
    array[array < thr] = 0
    binary_frame = array > 0
    sk.remove_small_objects(binary_frame, min_size=2, out=binary_frame)
    sk.remove_small_holes(binary_frame, area_threshold=2, out=binary_frame)
    array[binary_frame == 0] = 0
    return {"filtered_s": (filtered * 16).astype(np.int64), "cleaned": array, "cleaned_s": (array * 16).astype(np.int64), "threshold": thr}


def squared_edt(binary: np.ndarray) -> np.ndarray:
    """exact integer squared distance to the nearest background pixel (0 on the background), from scipy's feature transform"""
    if not binary.any():
        return np.zeros(binary.shape, np.int64)
    idx = ndimage.distance_transform_edt(binary, return_distances=False, return_indices=True)
    rr, cc = np.indices(binary.shape)
    return ((idx[0] - rr).astype(np.int64) ** 2 + (idx[1] - cc).astype(np.int64) ** 2) * binary


def fov(cleaned: np.ndarray, size: float) -> dict:
    """get_fov(cleaned, size): raises get_fov's ValueError for a frame without a component"""
    binary_frame = cleaned > 0
    labeled, _ = sk.label(binary_frame, connectivity=1, return_num=True)
    rois = sk.regionprops(labeled, intensity_image=cleaned)
    largest = max(rois, key=lambda x: x.area)
    longest = max(largest.image.shape)
    erosion = int(round((1 - size) * longest))
    eroded = sk.isotropic_erosion(binary_frame, radius=erosion / 2)
    boundary = sk.find_boundaries(eroded, connectivity=1, mode="inner")
    by, bx = np.nonzero(boundary)
    return {"longest": longest, "erosion": erosion, "mask": eroded, "fov": np.where(eroded, cleaned, 0), "boundary_x": bx, "boundary_y": by}


def _michelson_x100(mx, mn):
    return (mx - mn) / (mx + mn) * 100


def uniformity(fov_array: np.ndarray, window_size: int) -> dict:
    """IU, max / min points and, per axis, the max window value, its first (i, j) and the number of windows holding a FOV pixel
    (none along an axis shorter than the window); None where the reference raises."""
    out = {"n_fov": int((fov_array > 0).sum())}
    nz = fov_array[fov_array > 0]
    if nz.size:
        out["iu"] = _michelson_x100(nz.max(), nz.min())
        nan_array = np.where(fov_array == 0, np.nan, fov_array)
        out["max_point"] = tuple(int(v) for v in np.unravel_index(np.nanargmax(nan_array), fov_array.shape))
        out["min_point"] = tuple(int(v) for v in np.unravel_index(np.nanargmin(nan_array), fov_array.shape))
    else:
        out["iu"] = out["max_point"] = out["min_point"] = None
    out["window_too_large"] = window_size > fov_array.shape[0] or window_size > fov_array.shape[1]
    for axis in (0, 1):
        out[f"du_{axis}"] = None
        out[f"du_count_{axis}"] = 0
        if window_size > fov_array.shape[axis]:
            continue
        hi = sliding_window_view(np.where(fov_array > 0, fov_array, -np.inf), window_size, axis=axis).max(axis=-1)
        lo = sliding_window_view(np.where(fov_array > 0, fov_array, np.inf), window_size, axis=axis).min(axis=-1)
        valid = np.isfinite(hi)
        out[f"du_count_{axis}"] = int(valid.sum())
        if valid.any():
            with np.errstate(invalid="ignore"):
                v = np.where(valid, _michelson_x100(hi, lo), -1.0)
            k = int(np.argmax(v))
            out[f"du_{axis}"] = (float(v.flat[k]), tuple(int(t) for t in np.unravel_index(k, v.shape)))
    out["du"] = None if out["window_too_large"] or out["du_0"] is None or out["du_1"] is None else max(out["du_1"][0], out["du_0"][0])
    return out


def analyze_frame(frame: np.ndarray, pixel_size: float, ufov_ratio=0.95, cfov_ratio=0.75, window_size=5, threshold=0.75) -> dict:
    """The whole frame: {"bin", preprocess's planes, "edt2", "status" ("ok" / "no_component"), "ufov" / "cfov": fov() + uniformity()}"""
    b = determine_binning(pixel_size)
    out = {"bin": b}
    out.update(preprocess(frame, b, threshold))
    binary = out["cleaned"] > 0
    out["edt2"] = squared_edt(binary)
    if not binary.any():
        out["status"] = "no_component"
        return out
    out["status"] = "ok"
    for name, size in (("ufov", ufov_ratio), ("cfov", cfov_ratio * ufov_ratio)):
        f = fov(out["cleaned"], size)
        f.update(uniformity(f["fov"], window_size))
        out[name] = f
    return out
