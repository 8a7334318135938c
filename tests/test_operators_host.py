"""The semantics the operator kernels restate (csrc/filters.cu, csrc/ops.cu), pinned against numpy / scipy without a device:
the median window and its rank, correlate1d's summation order and integer cast, the median's order-preserving keys, and the
comparison type array_utils picks for threshold / binarize."""
import numpy as np
import pytest
from scipy import ndimage


def reflect(i, n):
    """scipy mode='reflect' (d c b a | a b c d | d c b a), as filters.cu's reflect_idx loops it"""
    while i < 0 or i >= n:
        if i < 0:
            i = -i - 1
        if i >= n:
            i = 2 * n - 1 - i
    return i


def device_median(a, k):
    """k_median_u16 / k_median_key: k x k window at offsets -(k//2) .. k-1-k//2, element of rank k*k//2.  A frame of one row
    (a 1-D profile) is k_median_row: the k-wide window at rank k//2."""
    rows = a.reshape(1, -1) if a.ndim == 1 else a
    H, W = rows.shape
    out = np.empty_like(rows)
    for y in range(H):
        for x in range(W):
            cols = [reflect(x + i - k // 2, W) for i in range(k)]
            if H == 1:
                out[y, x] = np.sort(rows[0, cols])[k // 2]
            else:
                win = rows[np.ix_([reflect(y + j - k // 2, H) for j in range(k)], cols)]
                out[y, x] = np.sort(win.ravel())[(k * k) // 2]
    return out.reshape(a.shape)


def scipy_reflect_defect(shape, k):
    """scipy 1.18 reflects a window offset of two or more periods (k // 2 >= 4 L on an axis of length L >= 2) to the wrong
    sample, up to values that are not in the input at all (median_filter([13, 41], size=17)[0] is 33).  No device answer can
    match that, so those sizes are not compared."""
    return any(L >= 2 and k // 2 >= 4 * L for L in shape)


@pytest.mark.parametrize("shape", [(1,), (2,), (5,), (40,), (1, 1), (1, 7), (7, 1), (3, 2), (5, 5), (7, 13)])
def test_median_window_matches_scipy(shape):
    rng = np.random.default_rng(sum(shape))
    a = rng.integers(0, 50, shape).astype(np.int32)       # repeats, so ties are exercised
    for k in range(1, 17):
        if a.ndim == 1 and k == 2 * a.shape[0] + 2:
            # scipy 1.18's 1-D path disagrees with its own 2-D path (and the device) at exactly this size; pinned below
            continue
        if scipy_reflect_defect(a.shape, k):
            continue
        np.testing.assert_array_equal(device_median(a, k), ndimage.median_filter(a, size=k), err_msg=f"k={k}")


def test_row_rule_is_the_2d_rule():
    """k copies of each of k samples put rank k*k//2 on rank k//2: a 1-row frame's 2-D median is the row median"""
    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 8):
        a = rng.integers(0, 9, n)
        for k in range(1, 2 * n + 6):
            np.testing.assert_array_equal(device_median(a, k), ndimage.median_filter(a[None], size=k)[0])


def test_scipy_1d_quirk_is_only_k_2n_plus_2():
    """scipy's 1-D median path agrees with its 2-D path on a 1-row frame at every size but k = 2n + 2, where its answer
    depends on memory outside the input (median_filter([1, 0], size=6) has given [1, 1] where the 2-D path gives [0, 1])"""
    rng = np.random.default_rng(5)
    for n in range(2, 9):
        for _ in range(4):
            a = rng.integers(0, 20, n)
            for k in range(1, 2 * n + 8):
                if k != 2 * n + 2:
                    np.testing.assert_array_equal(ndimage.median_filter(a, size=k), ndimage.median_filter(a[None], size=k)[0])


# ------------------------------------------------------------------------------------------------------------- correlate1d
def _cast(v, dt):
    """cast_from_double: integers through long long (truncation, then modular), floats rounded"""
    if dt == np.int32 and not -(2**31) <= v < 2**31:
        return np.int32(-(2**31))          # x86's cvttsd2si, which scipy's (npy_int) cast compiles to
    if dt.kind in "iu":
        return np.array(int(np.trunc(v))).astype(np.int64).astype(dt)[()]
    return dt.type(v)


def device_correlate1d(a, w, axis):
    """k_correlate1d: scipy's NI_Correlate1D order (symmetric / anti-symmetric pairs summed first), fp64, reflect"""
    r = (len(w) - 1) // 2
    sym = 0
    if r > 0:
        if all(abs(w[r + i] - w[r - i]) <= 2.220446049250313e-16 for i in range(1, r + 1)):
            sym = 1
        elif all(abs(w[r + i] + w[r - i]) <= 2.220446049250313e-16 for i in range(1, r + 1)):
            sym = -1
    H, W = a.shape
    n = H if axis == 0 else W
    out = np.empty_like(a)
    for y in range(H):
        for x in range(W):
            line = a[:, x] if axis == 0 else a[y, :]
            l = y if axis == 0 else x
            at = lambda i: float(line[reflect(i, n)])    # noqa: E731
            if sym:
                t = at(l) * w[r]
                for ll in range(-r, 0):
                    t += ((at(l + ll) + at(l - ll)) if sym > 0 else (at(l + ll) - at(l - ll))) * w[ll + r]
            else:
                t = at(l - r) * w[0]
                for ll in range(-r + 1, r + 1):
                    t += at(l + ll) * w[ll + r]
            out[y, x] = _cast(t, a.dtype)
    return out


def gaussian_weights(sigma):
    """array_utils._gaussian_kernel1d reversed, as gaussian_filter hands it to the device"""
    from pylinac_b200.core import array_utils as au

    r = int(4.0 * sigma + 0.5)
    return np.ascontiguousarray(au._gaussian_kernel1d(sigma, r)[::-1])


CORR_DTYPES = [np.uint8, np.uint16, np.int16, np.int32, np.float32, np.float64]


def _corr_input(shape, dtype, seed):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt.kind == "u":
        return rng.integers(0, 250 if dt.itemsize == 1 else 3000, shape).astype(dt)
    return (rng.random(shape) * 3000 - 1000).astype(dt)


@pytest.mark.parametrize("dtype", CORR_DTYPES)
@pytest.mark.parametrize("shape", [(1, 1), (1, 6), (3, 2), (5, 7), (2, 9)])
def test_correlate1d_gaussian_bit_exact(dtype, shape):
    a = _corr_input(shape, dtype, seed=shape[0] * 10 + shape[1])
    for sigma in (0.5, 1, 2.5, 4):     # radius 2..16: larger than every frame here
        w = gaussian_weights(sigma)
        got = device_correlate1d(device_correlate1d(a, w, 0), w, 1)
        want = ndimage.gaussian_filter(a, sigma)
        assert got.dtype == want.dtype
        np.testing.assert_array_equal(got, want, err_msg=f"sigma={sigma}")
        np.testing.assert_array_equal(device_correlate1d(a, w, 1), ndimage.gaussian_filter1d(a, sigma, axis=1))


@pytest.mark.parametrize("dtype", CORR_DTYPES)
@pytest.mark.parametrize("shape", [(1, 1), (1, 6), (3, 2), (5, 7), (2, 9)])
def test_correlate1d_sobel_bit_exact(dtype, shape):
    a = _corr_input(shape, dtype, seed=shape[0] * 7 + shape[1])
    d, s = np.array([-1.0, 0.0, 1.0]), np.array([1.0, 2.0, 1.0])
    for axis in (0, 1):
        got = device_correlate1d(device_correlate1d(a, d, axis), s, 1 - axis)
        with np.errstate(all="ignore"):
            want = ndimage.sobel(a, axis)
        np.testing.assert_array_equal(got, want, err_msg=f"axis={axis}")
    if np.dtype(dtype).kind in "iu":      # results beyond the dtype: wrap, or INT32_MIN for int32
        info = np.iinfo(dtype)
        e = np.array([[info.max, info.min, info.max, info.min], [info.min, info.max, info.max, 0]], dtype)
        with np.errstate(all="ignore"):
            for axis in (0, 1):
                np.testing.assert_array_equal(device_correlate1d(device_correlate1d(e, d, axis), s, 1 - axis), ndimage.sobel(e, axis))
    # a 1-D profile: the derivative pass alone
    p = a.reshape(1, -1)
    np.testing.assert_array_equal(device_correlate1d(p, d, 1)[0], ndimage.sobel(p[0]))


# ------------------------------------------------------------------------------------------------------------- median keys
def med_key(a):
    """MedKey<T>::key: integers flip the sign bit; floats flip all bits of negatives and set the sign bit of the rest"""
    a = np.asarray(a)
    if a.dtype.kind == "u":
        return a.astype(np.uint64)
    if a.dtype.kind == "i":
        ui = np.dtype(f"u{a.dtype.itemsize}")
        return a.view(ui) ^ ui.type(1 << (a.dtype.itemsize * 8 - 1))
    ui = np.uint32 if a.dtype == np.float32 else np.uint64
    b = a.view(ui)
    sign = ui(1 << (a.dtype.itemsize * 8 - 1))
    return np.where(b & sign, ~b, b | sign)


def med_val(k, dtype):
    """MedKey<T>::val, the inverse"""
    dt = np.dtype(dtype)
    if dt.kind == "u":
        return k.astype(dt)
    if dt.kind == "i":
        ui = np.dtype(f"u{dt.itemsize}")
        return (k.astype(ui) ^ ui.type(1 << (dt.itemsize * 8 - 1))).view(dt)
    ui = np.uint32 if dt == np.float32 else np.uint64
    k = k.astype(ui)
    sign = ui(1 << (dt.itemsize * 8 - 1))
    return np.where(k & sign, k & ~sign, ~k).view(dt)


KEY_CASES = {
    np.uint8: [0, 1, 127, 128, 255],
    np.uint16: [0, 1, 32767, 32768, 65534, 65535],
    np.int16: [-32768, -1, 0, 1, 32767],
    np.int32: [-(2**31), -1, 0, 1, 2**31 - 1],
    np.int64: [-(2**63), -(2**62) - 1, -1, 0, 1, 2**62 + 1, 2**63 - 1],
    np.float32: [-np.inf, -3.4e38, -1.0, -1.4e-45, -0.0, 0.0, 1.4e-45, 1.17e-38, 1.0, 3.4e38, np.inf],
    np.float64: [-np.inf, -1.7e308, -1.0, -5e-324, -2.2e-308, -0.0, 0.0, 5e-324, 2.2e-308, 1.0, 1.7e308, np.inf],
}


@pytest.mark.parametrize("dtype", list(KEY_CASES))
def test_median_key_preserves_order(dtype):
    rng = np.random.default_rng(1)
    v = np.array(KEY_CASES[dtype], dtype)
    v = np.concatenate([v, rng.permutation(v)])
    k = med_key(v)
    order = np.argsort(k, kind="stable")
    np.testing.assert_array_equal(v[order], np.sort(v))
    # -0 sorts before +0 with its own key; every other pair keeps numpy's order strictly
    for x, y, kx, ky in zip(v[order][:-1], v[order][1:], k[order][:-1], k[order][1:]):
        assert (kx < ky) == (x < y or (x == y and np.signbit(x) and not np.signbit(y))) or x == y
    back = med_val(k, dtype)
    np.testing.assert_array_equal(back.view(np.uint8), v.view(np.uint8))


# ------------------------------------------------------------------------------------------------------------- comparison type
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64, np.bool_])
def test_threshold_compares_as_numpy(dtype):
    from pylinac_b200.core import array_utils as au

    a = np.array([0, 1, 2, 3], dtype) if dtype != np.bool_ else np.array([False, True])
    if np.dtype(dtype).kind == "f":
        a = np.array([1.0, np.nextafter(np.float32(1), np.float32(0)), np.nextafter(np.float32(1), np.float32(2)), 2.0], dtype)
    for t in (1.00000001, 0.99999997, 1.0000000596, 1.5, 2, np.float64(1.00000001), np.float32(1.5), np.float32(1.0000001)):
        c = au._compare_threshold(a, t)
        # what the device computes, (double)pixel >= c, is numpy's comparison in np.result_type(a, t)
        np.testing.assert_array_equal(a.astype(np.float64) >= c, a >= t, err_msg=repr(t))
        np.testing.assert_array_equal(a.astype(np.float64) <= c, a <= t, err_msg=repr(t))


def test_largest_median_sizes():
    """DESIGN.md 4.7: the largest k whose (32 + k - 1) x (8 + k - 1) tile of keys fits 227 KB of shared memory per block"""
    def largest(key_bytes):
        return max(k for k in range(1, 400) if key_bytes * (31 + k) * (7 + k) <= 227 * 1024)

    assert (largest(2), largest(4), largest(8)) == (322, 222, 151)
