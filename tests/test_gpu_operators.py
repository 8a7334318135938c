"""The operator layer (core.array_utils, the core.image / core.profile methods on it, csrc/ops.cu and csrc/filters.cu) against
the numpy / scipy expression the reference evaluates, on the same input, at every dtype, filter size and frame shape it
accepts.  Results must be equal, with numpy's dtype and shape: the float gaussian and sobel reproduce scipy's summation order
(-fmad=false), so even one ulp is a defect."""
import numpy as np
import pytest
from scipy import ndimage

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64]
SHAPES_2D = [(1, 1), (1, 13), (11, 1), (8, 32), (9, 33), (37, 53)]
PROFILES = [1, 2, 7, 1000]


def au():
    from pylinac_b200.core import array_utils

    return array_utils


def rand(shape, dtype, seed=0):
    """Values spread over the dtype (integers: its whole range up to 32 bits; floats: signed, with repeats and fractions)."""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return rng.integers(0, 2, shape).astype(bool)
    if dt.kind in "iu":
        info = np.iinfo(dt)
        lo, hi = max(info.min, -(2**31)), min(info.max, 2**32 - 1)
        return rng.integers(lo, hi, shape, endpoint=True).astype(dt)
    return (np.round(rng.normal(0, 1000, shape), 1) * rng.random(shape)).astype(dt)


def same(got, want):
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(got, want)


def scipy_median(a, k):
    return ndimage.median_filter(a, size=k)


def skip_scipy_1d_quirk(a, k):
    """scipy 1.18's 1-D median path disagrees with its own 2-D path at exactly k = 2n + 2 (median_filter([1, 0], size=6) is
    [1, 1], median_filter([[1, 0]], size=6) is [[0, 1]]); the device answers as the 2-D path.  Only that one size is skipped."""
    return a.ndim == 1 and k == 2 * a.shape[0] + 2


# ---------------------------------------------------------------------------------------------------------------- median
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", SHAPES_2D + [(n,) for n in PROFILES])
def test_median_every_small_k(dtype, shape):
    a = rand(shape, dtype, seed=len(shape) * 100 + shape[0])
    for k in range(1, 13):
        if skip_scipy_1d_quirk(a, k):
            continue
        same(au().filter(a, size=k), scipy_median(a, k))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [31, 32, 51, 64])
def test_median_large_k_2d(dtype, k):
    a = rand((40, 48), dtype, seed=k)
    same(au().filter(a, size=k), scipy_median(a, k))


@pytest.mark.parametrize("k", [32, 51, 64])
def test_median_large_k_uint16_frame(k):
    a = rand((150, 120), np.uint16, seed=k)
    same(au().filter(a, size=k), scipy_median(a, k))


def test_median_k10_vmat_frame():
    """vmat._identify_images: Image.filter(size=10) on uint16 frames (even size, upper median, k_median_u16's bisection)"""
    from pylinac_b200.core import image

    a = rand((384, 512), np.uint16, seed=10) // 4 + 1000
    img = image.ArrayImage(a.copy())
    img.filter(size=10, kind="median")
    same(img.array, scipy_median(a, 10))


@pytest.mark.parametrize("shape, k", [((640, 96), 32), ((1300, 16), 65)])
def test_image_filter_default_size(shape, k):
    from pylinac_b200.core import image

    a = rand(shape, np.uint16, seed=k)
    assert int(round(shape[0] * 0.05)) == k
    img = image.ArrayImage(a.copy())
    img.filter()
    same(img.array, scipy_median(a, k))


@pytest.mark.parametrize("dtype", [np.uint16, np.float64, np.int32])
@pytest.mark.parametrize("n", [1000, 4096])
def test_profile_median_default_size(dtype, n):
    """SingleProfile.filter() / array_utils.filter(profile) with size=0.05: k = 50 and 205"""
    a = rand((n,), dtype, seed=n)
    k = int(round(n * 0.05))
    same(au().filter(a), scipy_median(a, k))
    for kk in (k - 1, k + 1, 2 * n // 3):
        same(au().filter(a, size=kk), scipy_median(a, kk))


def test_single_profile_filter_default():
    from pylinac_b200.core.profile import SingleProfile

    x = np.arange(1000)
    v = (np.clip((300 - np.abs(x - 500)) / 20.0, 0, 1) * 40000 + 1000 + (x * 7919) % 97).astype(np.uint16)
    p = SingleProfile(v.copy())
    before = np.asarray(p.values).copy()
    p.filter()
    same(np.asarray(p.values), scipy_median(before, int(round(len(before) * 0.05))))


def test_median_refuses_only_what_no_tile_holds():
    from pylinac_b200 import _native as nat

    a = rand((20, 20), np.float64)
    same(au().filter(a, size=151), scipy_median(a, 151))
    with pytest.raises(nat.NativeError, match="shared-memory tile"):
        au().filter(a, size=152)


# ---------------------------------------------------------------------------------------------------------------- gaussian
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("sigma", [0.5, 1, 2.5, 4, 16])
def test_gaussian(dtype, sigma):
    for i, shape in enumerate(SHAPES_2D + [(n,) for n in PROFILES]):
        a = rand(shape, dtype, seed=i)
        same(au().gaussian_filter(a, sigma), ndimage.gaussian_filter(a, sigma))
        if float(sigma).is_integer():      # Image.filter(size=int, kind="gaussian"); a float size is a fraction of the rows
            same(au().filter(a, size=int(sigma), kind="gaussian"), ndimage.gaussian_filter(a, sigma))


@pytest.mark.parametrize("dtype", [np.uint16, np.float32, np.float64])
def test_gaussian_radius_above_256(dtype):
    a = rand((40, 50), dtype, seed=70)
    same(au().gaussian_filter(a, 70), ndimage.gaussian_filter(a, 70))
    p = rand((300,), dtype, seed=71)
    same(au().gaussian_filter(p, 100), ndimage.gaussian_filter(p, 100))


# ---------------------------------------------------------------------------------------------------------------- sobel
@pytest.mark.parametrize("dtype", DTYPES)
def test_sobel(dtype):
    for i, shape in enumerate(SHAPES_2D + [(n,) for n in PROFILES]):
        a = rand(shape, dtype, seed=i)
        for axis in ((0, 1, -1) if a.ndim == 2 else (0, -1)):
            with np.errstate(all="ignore"):
                want = ndimage.sobel(a, axis)
            same(au().sobel(a, axis), want)


def test_sobel_profile_is_the_derivative():
    p = np.array([1, 4, 9, 16, 25], np.float64)
    same(au().sobel(p), np.array([3, 8, 12, 16, 9], np.float64))
    same(au().sobel(p, 0), ndimage.sobel(p, 0))


# ---------------------------------------------------------------------------------------------------------------- batches
def test_batch_is_per_frame():
    frames = np.stack([rand((37, 53), np.int32, seed=1) // 1000, rand((37, 53), np.int32, seed=2) // 10 + 5000,
                       rand((37, 53), np.int32, seed=3) % 7 - 3])
    f64 = frames.astype(np.float64) / 3
    A = au()
    for i, f in enumerate(frames):
        same(A.filter(frames, size=5)[i], scipy_median(f, 5))
        same(A.gaussian_filter(frames, 2.5)[i], ndimage.gaussian_filter(f, 2.5))
        same(A.sobel(frames, 0)[i], ndimage.sobel(f, 0))
        same(A.invert(frames)[i], -f + f.max() + f.min())
        same(A.ground(frames, 3)[i], f - f.min() + 3)
        same(A.normalize(f64)[i], f64[i] / f64[i].max())
        same(A.threshold(frames, 0.5)[i], np.where(f >= 0.5, f, 0))
    _, mins = A.ground_with_min(frames)
    same(mins, frames.min(axis=(1, 2)))


# ---------------------------------------------------------------------------------------------------------------- maps
def test_float32_threshold_compares_in_float32():
    from pylinac_b200.core import image

    a = np.array([[1.0, 0.99999994, 1.0000001, 2.0]], np.float32)
    for t in (1.00000001, 0.99999997, 1.0000000596):
        same(au().threshold(a, t), np.where(a >= t, a, 0))
        same(au().threshold(a, t, kind="low"), np.where(a <= t, a, 0))
        same(au().binarize(a, t), np.where(a >= t, 1, 0))
        img = image.ArrayImage(a.copy())
        img.threshold(t)
        same(img.array, np.where(a >= t, a, 0))
        same(image.ArrayImage(a.copy()).as_binary(t).array, np.where(a >= t, 1, 0))
        # a strong float64 scalar compares in float64
        same(au().threshold(a, np.float64(t)), np.where(a >= np.float64(t), a, 0))
    u = np.array([[0, 1, 2, 65535]], np.uint16)
    same(au().threshold(u, 1.5), np.where(u >= 1.5, u, 0))
    same(au().binarize(u, np.float32(1.5)), np.where(u >= np.float32(1.5), 1, 0))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("where", ["first", "middle", "last", "second frame"])
def test_nan_propagates_through_min_max(dtype, where):
    a = rand((3, 9, 33), dtype, seed=5)
    idx = {"first": (0, 0, 0), "middle": (0, 4, 17), "last": (0, 8, 32), "second frame": (1, 3, 3)}[where]
    a[idx] = np.nan
    A = au()
    inputs = [a] if where == "second frame" else [a, a[0]]
    for x in inputs:
        frames = x if x.ndim == 3 else x[None]
        outs = [np.reshape(fn(x), frames.shape) for fn in (A.normalize, A.invert, A.ground)]
        for i, f in enumerate(frames):
            same(outs[0][i], f / f.max())
            same(outs[1][i], -f + f.max() + f.min())
            same(outs[2][i], f - f.min() + 0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_normalize_value_promotion(dtype):
    a = rand((9, 33), dtype, seed=9)
    for v in (3.0, np.float64(3.0), 7, np.float32(0.3)):
        same(au().normalize(a, value=v), a / v)
    same(au().normalize(a), a / a.max())


@pytest.mark.parametrize("dtype", DTYPES)
def test_ground_value_promotion(dtype):
    a = rand((9, 33), dtype, seed=11)
    for v in (0, 5, 2.5, np.float64(2.0), np.float32(1.5)):
        with np.errstate(over="ignore"):
            want = a - a.min() + v
        same(au().ground(a, value=v), want)


def test_ground_value_out_of_range():
    a = np.array([[5, 7, 9]], np.uint16)
    with pytest.raises(OverflowError):
        a - a.min() + (-5)
    with pytest.raises(OverflowError):
        au().ground(a, value=-5)
    with pytest.raises(OverflowError):
        au().ground(a.astype(np.int8), value=200)


def test_image_ground_int64_min():
    from pylinac_b200.core import image

    a = np.array([[2**62 + 1, 2**62 + 3], [2**62 + 7, 2**62 + 2]], np.int64)
    img = image.ArrayImage(a.copy())
    mn = img.ground()
    assert type(mn) is np.int64 and mn == 2**62 + 1
    same(img.array, a - a.min())


def test_int16_wraps():
    a = np.array([[-32768, 0, 32767, 100]], np.int16)
    with np.errstate(over="ignore"):
        same(au().invert(a), -a + a.max() + a.min())
        same(au().ground(a), a - a.min())
        same(au().ground(a, value=3), a - a.min() + 3)


# ---------------------------------------------------------------------------------------------------------------- int8 / uint32 / bool
@pytest.mark.parametrize("dtype", [np.int8, np.uint32])
def test_narrow_and_uint32_dtypes(dtype):
    a = rand((9, 33), dtype, seed=13)
    A = au()
    with np.errstate(over="ignore"):
        same(A.bit_invert(a), np.invert(a))
        same(A.invert(a), -a + a.max() + a.min())
        same(A.ground(a), a - a.min())
        same(A.ground(a, value=3), a - a.min() + 3)
    same(A.normalize(a), a / a.max())
    same(A.threshold(a, 10.5), np.where(a >= 10.5, a, 0))
    same(A.binarize(a, 10.5), np.where(a >= 10.5, 1, 0))
    for k in (1, 2, 3, 4, 7):
        same(A.filter(a, size=k), scipy_median(a, k))
    same(A.gaussian_filter(a, 1.5), ndimage.gaussian_filter(a, 1.5))
    for axis in (0, 1):
        with np.errstate(all="ignore"):
            same(A.sobel(a, axis), ndimage.sobel(a, axis))
    _, mn = A.ground_with_min(a)
    assert type(mn) is np.dtype(dtype).type and mn == a.min()


def test_uint32_bit_invert_extremes():
    a = np.array([0, 5, 2**32 - 1], np.uint32)
    same(au().bit_invert(a), np.array([2**32 - 1, 2**32 - 6, 0], np.uint32))


def test_bool():
    a = rand((9, 33), bool, seed=17)
    A = au()
    same(A.bit_invert(a), np.invert(a))
    same(A.normalize(a), a / a.max())
    same(A.threshold(a, 0.5), np.where(a >= 0.5, a, 0))
    same(A.binarize(a, 0.5), np.where(a >= 0.5, 1, 0))
    for k in (2, 3):
        same(A.filter(a, size=k), scipy_median(a, k))
    for ours, theirs in ((A.invert, lambda x: -x + x.max() + x.min()), (A.ground, lambda x: x - x.min() + 0)):
        with pytest.raises(TypeError) as want:
            theirs(a)
        with pytest.raises(TypeError, match="boolean") as got:
            ours(a)
        assert str(got.value) == str(want.value)


@pytest.mark.parametrize("dtype", [np.uint64, np.float16])
def test_unsupported_dtypes_raise(dtype):
    with pytest.raises(TypeError):
        au().filter(np.ones((4, 4), dtype), size=3)
