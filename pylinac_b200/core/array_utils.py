"""``pylinac.core.array_utils`` (core/array_utils.py:38-212) with the pixel arithmetic executed by libepid.so.

Every function uploads the array to HBM, runs the CUDA operator with the reference's dtype semantics and
downloads the result.  1-D arrays (profiles) are handled as a single row; a 3-D array is a batch of frames, each
processed as the 2-D call would process it alone.  No numpy/scipy compute fallback.

Dtypes follow numpy 2: bool, int8 and uint32 give numpy's results and exceptions (int8 and uint32 compute in int16 /
int64 and cast back modularly, which is exact for every operator here), and a scalar argument takes part in type
promotion as numpy's weak Python scalars or strong numpy scalars do.  uint64 and float16 raise TypeError.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _native as nat

# dtypes the device computes in for the ones it has no kernels for (exact: modular for int8 / uint32, 0 / 1 for bool)
_WIDEN = {np.dtype(np.bool_): np.dtype(np.uint8), np.dtype(np.int8): np.dtype(np.int16), np.dtype(np.uint32): np.dtype(np.int64)}


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
    if a.dtype.byteorder == ">":
        a = a.astype(a.dtype.newbyteorder("<"))
    if a.dtype in _WIDEN:
        a = a.astype(_WIDEN[a.dtype])
    if a.dtype not in nat._NP2DT:
        raise TypeError(f"dtype {a.dtype} is not supported by the native operators")
    return a


def _run(a, fn, *args, same_dtype: bool = True):
    """Run the unary operator on the device; ``same_dtype``: the result has the input's dtype (cast back from the widened one)."""
    dt = np.asarray(a).dtype
    a = _coerce(a)
    a3, shape = _as3d(a)
    ctx = _ctx()
    with nat.Batch.upload(ctx, a3) as b, b._unary(fn, *args) as out:
        res = out.download()
    if same_dtype and res.dtype != dt:
        res = res.astype(dt.newbyteorder("="))
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
    """array / (value or array.max()) with numpy 2's result dtype: float32 for a float32 array over its own max or a Python
    scalar, float64 when either side is float64 (an ``np.float64`` value included)."""
    a = np.asarray(array)
    if value is None:
        return _run(a, nat.lib().epid_normalize, 1, 0.0, same_dtype=False)
    rt = np.result_type(a.dtype, value)
    if rt.kind in "f" and rt != a.dtype:
        a = a.astype(rt)       # exact: numpy converts the array to the result dtype before dividing
    return _run(a, nat.lib().epid_normalize, 0, float(value), same_dtype=False)


def invert(array: np.ndarray) -> np.ndarray:  # :75-77
    a = np.asarray(array)
    if a.dtype == np.bool_:
        raise TypeError("The numpy boolean negative, the `-` operator, is not supported, use the `~` operator or the logical_not "
                        "function instead.")
    return _run(a, nat.lib().epid_invert)


def bit_invert(array: np.ndarray) -> np.ndarray:  # :81-89
    a = np.asarray(array)
    if a.dtype.kind == "f":
        raise ValueError(f"The datatype {a.dtype} could not be safely inverted. This usually means the array is a float-like "
                         "datatype. Cast to an integer-like datatype first.")
    if a.dtype == np.bool_:
        return _run(a, nat.lib().epid_bit_invert, same_dtype=False) == 255      # ~0 = 255, ~1 = 254: np.invert is the logical not
    return _run(a, nat.lib().epid_bit_invert)


def ground_with_min(array: np.ndarray, value: float = 0):
    """(array - array.min() + value, array.min()); the minimum is a scalar of the array's dtype (one per frame for a batch).
    ``a - min`` is taken in the array's dtype (wrapping as numpy's does) and ``+ value`` in numpy 2's result dtype: the array's
    own for an in-range Python int (out of range: numpy's OverflowError), a wider one for a float or a wider numpy scalar."""
    a0 = np.asarray(array)
    if a0.dtype == np.bool_:
        raise TypeError("numpy boolean subtract, the `-` operator, is not supported, use the bitwise_xor, the `^` operator, or the "
                        "logical_xor function instead.")
    rt = np.result_type(a0.dtype, value)
    same = rt == a0.dtype
    if same and a0.dtype.kind in "iu":
        a0.dtype.type(value)       # OverflowError for a Python int outside the dtype, as numpy's `+ value` raises
    a = _coerce(a0)
    a3, shape = _as3d(a)
    ctx = _ctx()
    mins = np.empty(a3.shape[0], a.dtype)
    h = C.c_void_p()
    with nat.Batch.upload(ctx, a3) as b:
        nat.check(nat.lib().epid_ground(ctx.handle, b.handle, float(value) if same else 0.0, C.byref(h), mins.ctypes.data_as(C.c_void_p)))
        with nat.Batch(ctx, h) as out:
            res = out.download().reshape(shape)
    dt = a0.dtype.newbyteorder("=")
    res, mins = res.astype(dt, copy=False), mins.astype(dt)
    if not same:
        res = res + value          # numpy's promotion of the grounded array and the scalar (host-resident result)
    return res, (mins[0] if a3.shape[0] == 1 else mins)


def ground(array: np.ndarray, value: float = 0) -> np.ndarray:  # :93-102
    return ground_with_min(array, value)[0]


def filter(array: np.ndarray, size=0.05, kind: str = "median") -> np.ndarray:  # :106-138
    """ndimage.median_filter(array, size) / ndimage.gaussian_filter(array, sigma=size) of a profile or frame; a float size is
    that fraction of the rows (of each frame's rows for a batch)."""
    if isinstance(size, float):
        if 0 < size < 1:
            rows = len(array) if np.ndim(array) < 3 else np.shape(array)[1]
            size = int(round(rows * size))
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
    if a.dtype == np.bool_:
        raise TypeError("gaussian_filter of a bool array is not supported")
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
    return _run(array, nat.lib().epid_zoom, float(zoom), int(order), (0 if mode == "constant" else 1) | (2 if grid_mode else 0),
                same_dtype=False)


def rotate(array: np.ndarray, angle: float, mode: str = "edge") -> np.ndarray:
    """skimage.transform.rotate(array, angle, mode=mode) with its defaults (bilinear, no resize, img_as_float conversion of integer
    images: uint8 / 255, uint16 / 65535) -> float64, on the device (csrc/zoom.cu)."""
    if mode not in ("edge", "constant"):
        raise ValueError("rotate mode must be 'edge' or 'constant'")
    return _run(array, nat.lib().epid_rotate, float(angle), 1 if mode == "edge" else 0, same_dtype=False)


def sobel(array: np.ndarray, axis: int = -1) -> np.ndarray:
    """ndimage.sobel(array, axis): the [-1, 0, 1] derivative along ``axis``, then [1, 2, 1] along the other axis of a frame.
    A 1-D profile has no other axis: its result is the derivative alone."""
    a = np.asarray(array)
    if a.dtype == np.bool_:
        raise TypeError("sobel of a bool array is not supported")
    if a.ndim == 1:
        if axis not in (0, -1):
            raise ValueError("axis must be 0 or -1 for a 1-D array")
        d = np.array([-1.0, 0.0, 1.0])
        return _run(a, nat.lib().epid_correlate1d_passes, d.ctypes.data_as(C.c_void_p), 1, 2)
    return _run(a, nat.lib().epid_sobel, int(axis))


def _compare_threshold(a: np.ndarray, t) -> float:
    """The threshold as the double that compares with every pixel as numpy 2's ``a >= t`` does: numpy compares in
    np.result_type(a, t), which is float32 for a float32 array and a Python float, so t is rounded to float32 first (exact
    comparisons of float32 pixels in double).  A wider result type compares exactly in double already."""
    if np.result_type(a.dtype, t) == np.float32:
        return float(np.float32(t))
    return float(t)


def threshold(array: np.ndarray, threshold: float, kind: str = "high") -> np.ndarray:
    """np.where(a >= t, a, 0) / np.where(a <= t, a, 0)  (core/image.py:797-800); int64 for a bool array, as np.where gives"""
    a = np.asarray(array)
    res = _run(a, nat.lib().epid_threshold, _compare_threshold(a, threshold), 0 if kind == "high" else 1, same_dtype=a.dtype != np.bool_)
    return res.astype(np.int64) if a.dtype == np.bool_ else res


def binarize(array: np.ndarray, threshold: float) -> np.ndarray:
    """np.where(a >= t, 1, 0) -> int64 (core/image.py:814)"""
    a = np.asarray(array)
    return _run(a, nat.lib().epid_binarize, _compare_threshold(a, threshold), same_dtype=False)


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
