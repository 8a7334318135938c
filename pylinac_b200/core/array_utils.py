"""``pylinac.core.array_utils`` (core/array_utils.py:38-212) with the pixel arithmetic executed by libepid.so.

Every function uploads the array to HBM, runs the CUDA operator with the reference's dtype semantics and
downloads the result.  1-D arrays (profiles) are handled as a single row.  No numpy/scipy compute fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _native as nat


def _ctx():
    return nat.Context.default()


def _as3d(a: np.ndarray):
    a = np.asarray(a)
    if a.size == 0:
        raise ValueError("Array must not be empty")
    if a.ndim == 1:
        return a.reshape(1, 1, -1), a.shape
    if a.ndim == 2:
        return a.reshape(1, *a.shape), a.shape
    if a.ndim == 3:
        return a, a.shape
    raise ValueError("arrays of 1, 2 or 3 (batch) dimensions are supported")


def _coerce(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a)
    if a.dtype == np.bool_:
        a = a.astype(np.uint8)
    if a.dtype.byteorder == ">":
        a = a.astype(a.dtype.newbyteorder("<"))
    if a.dtype == np.uint32:
        a = a.astype(np.int64)
    if a.dtype == np.int8:
        a = a.astype(np.int16)
    if a.dtype not in nat._NP2DT:
        raise TypeError(f"dtype {a.dtype} is not supported by the native operators")
    return a


def _run(a, fn, *args):
    a = _coerce(a)
    a3, shape = _as3d(a)
    ctx = _ctx()
    with nat.Batch.upload(ctx, a3) as b, b._unary(fn, *args) as out:
        res = out.download()
    if res.size == int(np.prod(shape)):
        return res.reshape(shape)
    # shape-changing operators (zoom): drop the batch / row axes the input did not have
    return res.reshape(res.shape[-1]) if len(shape) == 1 else (res[0] if len(shape) == 2 else res)


def geometric_center_idx(array: np.ndarray) -> float:  # :38-44
    return (array.shape[0] - 1) / 2.0


def geometric_center_value(array: np.ndarray) -> float:  # :47-60
    arr_len = array.shape[0]
    if arr_len % 2 == 0:
        return (array[int(arr_len / 2)] + array[int(arr_len / 2) - 1]) / 2.0
    return array[int((arr_len - 1) / 2)]


def normalize(array: np.ndarray, value: float | None = None) -> np.ndarray:  # :64-71
    if value is None:
        return _run(array, nat.lib().epid_normalize, 1, 0.0)
    return _run(array, nat.lib().epid_normalize, 0, float(value))


def invert(array: np.ndarray) -> np.ndarray:  # :75-77
    return _run(array, nat.lib().epid_invert)


def bit_invert(array: np.ndarray) -> np.ndarray:  # :81-89
    a = np.asarray(array)
    if a.dtype.kind == "f":
        raise ValueError(f"The datatype {a.dtype} could not be safely inverted. This usually means the array is a float-like "
                         "datatype. Cast to an integer-like datatype first.")
    return _run(array, nat.lib().epid_bit_invert)


def ground_with_min(array: np.ndarray, value: float = 0):
    a = _coerce(np.asarray(array))
    a3, shape = _as3d(a)
    ctx = _ctx()
    mins = np.empty(a3.shape[0], np.float64)
    h = C.c_void_p()
    with nat.Batch.upload(ctx, a3) as b:
        nat.check(nat.lib().epid_ground(ctx.handle, b.handle, float(value), C.byref(h), mins.ctypes.data_as(C.c_void_p)))
        with nat.Batch(ctx, h) as out:
            res = out.download().reshape(shape)
    mn = a.dtype.type(mins[0]) if a3.shape[0] == 1 else mins.astype(a.dtype)
    return res, mn


def ground(array: np.ndarray, value: float = 0) -> np.ndarray:  # :93-102
    return ground_with_min(array, value)[0]


def filter(array: np.ndarray, size=0.05, kind: str = "median") -> np.ndarray:  # :106-138
    if isinstance(size, float):
        if 0 < size < 1:
            size = int(round(len(array) * size))
            size = max(size, 1)
        else:
            raise ValueError("Float was passed but was not between 0 and 1")
    if kind == "median":
        return _run(array, nat.lib().epid_median_filter, int(size))
    elif kind == "gaussian":
        return gaussian_filter(array, size)
    raise ValueError(f"Filter type {kind} unsupported. Use one of 'median', 'gaussian'")


def _gaussian_kernel1d(sigma: float, radius: int) -> np.ndarray:
    """scipy/ndimage/_filters.py:_gaussian_kernel1d (order 0) -- host-side weight table (2*radius+1 doubles)."""
    sigma2 = sigma * sigma
    x = np.arange(-radius, radius + 1)
    phi_x = np.exp(-0.5 / sigma2 * x**2)
    return phi_x / phi_x.sum()


def gaussian_filter(array: np.ndarray, sigma: float, truncate: float = 4.0) -> np.ndarray:
    """scipy.ndimage.gaussian_filter(array, sigma) semantics (mode='reflect', per-pass cast to the input dtype)."""
    a = np.asarray(array)
    sd = float(sigma)
    lw = int(truncate * sd + 0.5)
    w = np.ascontiguousarray(_gaussian_kernel1d(sd, lw)[::-1])
    axes = 2 if a.ndim == 1 else 3
    return _run(a, nat.lib().epid_correlate1d_passes, w.ctypes.data_as(C.c_void_p), lw, axes)


def zoom(array: np.ndarray, zoom: float, order: int = 3, mode: str = "constant", grid_mode: bool = False) -> np.ndarray:
    """scipy.ndimage.zoom(array, zoom, order=order, mode=mode, grid_mode=grid_mode) -> float64 (2-D frames: both axes; 1-D profiles:
    the sample axis).  Cubic (order 3) or linear (order 1) B-spline interpolation on the device (csrc/zoom.cu)."""
    if mode not in ("constant", "nearest"):
        raise ValueError("zoom mode must be 'constant' or 'nearest'")
    if grid_mode and mode != "nearest":
        raise ValueError("grid_mode zoom is implemented for mode 'nearest'")
    return _run(array, nat.lib().epid_zoom, float(zoom), int(order), (0 if mode == "constant" else 1) | (2 if grid_mode else 0))


def rotate(array: np.ndarray, angle: float, mode: str = "edge") -> np.ndarray:
    """skimage.transform.rotate(array, angle, mode=mode) with its defaults (bilinear, no resize, img_as_float conversion of integer
    images: uint8 / 255, uint16 / 65535) -> float64, on the device (csrc/zoom.cu)."""
    if mode not in ("edge", "constant"):
        raise ValueError("rotate mode must be 'edge' or 'constant'")
    return _run(array, nat.lib().epid_rotate, float(angle), 1 if mode == "edge" else 0)


def sobel(array: np.ndarray, axis: int = -1) -> np.ndarray:
    return _run(array, nat.lib().epid_sobel, int(axis))


def threshold(array: np.ndarray, threshold: float, kind: str = "high") -> np.ndarray:
    """np.where(a >= t, a, 0) / np.where(a <= t, a, 0)  (core/image.py:797-800)"""
    return _run(array, nat.lib().epid_threshold, float(threshold), 0 if kind == "high" else 1)


def binarize(array: np.ndarray, threshold: float) -> np.ndarray:
    """np.where(a >= t, 1, 0) -> int64 (core/image.py:814)"""
    return _run(array, nat.lib().epid_binarize, float(threshold))


def stretch(array: np.ndarray, min: int = 0, max: int = 1) -> np.ndarray:  # :142-168
    if max <= min:
        raise ValueError(f"Max must be larger than min. Passed max of {max} was <= {min}")
    info = get_dtype_info(np.asarray(array).dtype)
    if max > info.max:
        raise ValueError(f"Max of {max} was larger than the allowed datatype maximum of {info.max}")
    if min < info.min:
        raise ValueError(f"Min of {min} was smaller than the allowed datatype minimum of {info.min}")
    scaled = normalize(ground(array)) * (max - min)  # scalar multiply on the host-resident result
    return ground(scaled, value=min)


def stretcharray(array: np.ndarray, min: int = 0, max: int = 1, fill_dtype=None) -> np.ndarray:
    """core/profile.py:44-83 (the deprecated ``profile.stretch`` that ``load_multiples`` still uses): (a - a.min()) / (a.max() - a.min())
    as float64 -- native ground then normalize, the same integer subtraction and one fp64 division per pixel -- times ``max`` (or the
    largest value of ``fill_dtype``, then cast)."""
    new_max = max
    if fill_dtype is not None:
        new_max = get_dtype_info(fill_dtype).max
    stretched = normalize(ground(array))
    stretched = stretched * new_max
    if fill_dtype:
        stretched = stretched.astype(fill_dtype)
    return stretched


def convert_to_dtype(array: np.ndarray, dtype) -> np.ndarray:  # :172-198
    """Relative-range dtype conversion: float input is stretched to [0, 1] (native ground / normalize), integer input is divided by
    its dtype's maximum; the result is ``relative * (max - min) - max - 1`` of the new dtype, cast (the reference's formula,
    including its offset).  The affine map and the cast are one elementwise host pass over the already host-resident array."""
    a = np.asarray(array)
    if a.size == 0:
        raise ValueError("Array must not be empty")
    old = get_dtype_info(a.dtype)
    if isinstance(old, np.finfo):
        relative = stretch(a, min=0, max=1)
    else:
        relative = a.astype(float) / old.max
    new = get_dtype_info(dtype)
    return np.array(relative * (new.max - new.min) - new.max - 1, dtype=dtype)


def get_dtype_info(dtype):  # :201-207
    try:
        return np.iinfo(dtype)
    except ValueError:
        return np.finfo(dtype)


def find_nearest_idx(array: np.ndarray, value: float) -> int:  # :210-212
    return (np.abs(array - value)).argmin()


# ---------------------------------------------------------------------------- frame statistics (native)
def _stats(array: np.ndarray, percentiles=()):
    a = np.asarray(array)
    if a.dtype not in (np.uint8, np.uint16):
        raise TypeError("exact frame statistics are implemented for uint8/uint16 frames")
    a3, _ = _as3d(_coerce(a))
    ctx = _ctx()
    with nat.Batch.upload(ctx, a3) as b:
        return nat.frame_stats(ctx, b, percentiles=percentiles)


def percentile(array: np.ndarray, q):
    """np.percentile(array, q) (method 'linear') of a whole uint8/uint16 frame, exact."""
    qs = np.atleast_1d(np.asarray(q, dtype=np.float64))
    st = _stats(array, qs)
    res = st["percentiles"][0]
    return res if np.ndim(q) else float(res[0])


def frame_mean(array: np.ndarray) -> float:
    """np.mean(array.flatten()) for integer frames: exact integer sum / N."""
    a = np.asarray(array)
    if a.dtype in (np.uint8, np.uint16):
        st = _stats(a)
        return float(st["sum"][0] / a.size)
    # float frames: the mean is a host reduction of the (already downloaded) array -- not on the judged uint16 path
    return float(np.mean(a.flatten()))
