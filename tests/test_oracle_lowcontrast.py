"""CPU: the LowContrastDiskROI goldens against numpy on the restated skimage.draw.disk, and a numpy model of epid_disk_percentiles'
plan and lerp (csrc/roi.cu k_disk_percentiles) against np.percentile for every dtype, at the ranks and weights where the plan's type
and numpy's index past the end matter."""
import json

import numpy as np
import pytest

from oracle.skimage_draw import disk
from tests.golden.lowcontrast_cases import Q, ROI_CASES

GOLDEN = np.load("tests/golden/lowcontrast_golden.npz")


@pytest.mark.parametrize("name", sorted(ROI_CASES))
def test_golden_is_numpy_on_the_restated_disk(name):
    build, specs = ROI_CASES[name]
    arr = build()
    for (cy, cx, r, _), rec in zip(specs, json.loads(str(GOLDEN["roi:" + name]))):
        rr, cc = disk((cy, cx), r)
        try:
            vals = arr[rr, cc]
        except IndexError as e:
            assert rec["percentile"][0]["error"] == [type(e).__name__, str(e)]
            continue
        for q, got in zip(Q, rec["percentile"]):
            try:
                want = np.percentile(vals, q)
            except Exception as e:  # noqa: BLE001 -- compared with the golden's exception
                assert got["error"] == [type(e).__name__, str(e)], q
                continue
            assert got["value"] == ["float", float(want)] or (np.isnan(want) and np.isnan(got["value"][1])), q
        if vals.size:
            assert rec["pixel_value"]["value"][1] == float(np.median(vals)) or np.isnan(np.median(vals))
            assert rec["std"]["value"][1] == float(np.std(vals)) or np.isnan(np.std(vals))


def pct_plan(n, q, F):
    """stats.cuh pct_plan in the type F: ranks (prev, next), clamped past either end"""
    vi = F(n - 1) * (F(q) / F(100))
    if vi >= F(n - 1):
        return n - 1, n - 1, vi
    if vi < 0:
        return 0, 0, vi
    return int(np.floor(vi)), int(np.floor(vi)) + 1, vi


def percentile_model(vals, q):
    """k_disk_percentiles' result for Python number q: order statistics at pct_plan's ranks, numpy's weight (vi less the previous
    index, -1 past the end) and np_lerp_d with b - a formed in the pixels' own type"""
    F = np.float32 if vals.dtype == np.float32 else np.float64
    n = vals.size
    if np.issubdtype(vals.dtype, np.floating) and np.isnan(vals).any():
        return F(np.nan)
    prev, nxt, vi = pct_plan(n, q, F)
    srt = np.sort(vals)
    a, b = srt[prev], srt[nxt]
    t = F(np.float64(vi) - (-1.0 if vi >= F(n - 1) else float(prev)))
    with np.errstate(over="ignore"):
        d = F(b - a) if np.issubdtype(vals.dtype, np.integer) else F(b) - F(a)   # integers subtract in their own type, wrapping
    r = F(F(a) + d * t)
    if t >= F(0.5):
        r = F(F(b) - d * (F(1) - t))
    return r


def _values(rng, dtype, n):
    if np.issubdtype(dtype, np.integer):
        info = np.iinfo(dtype)
        return rng.integers(info.min, int(info.max) + 1, n).astype(dtype)
    return (rng.standard_normal(n) * 1e4).astype(dtype)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64])
def test_percentile_model_is_numpy(dtype):
    rng = np.random.default_rng(11)
    qs = [0, 1, 2.5, 50, 99, 99.5, 100, 99.99999999, 33.333333333333336, 12.5, 87.5]
    for n in (1, 2, 3, 7, 8, 100, 101, 1000, 4097, 70001):
        vals = _values(rng, dtype, n)
        for q in qs + [float(x) for x in rng.uniform(0, 100, 6)]:
            want = np.percentile(vals, q)
            got = percentile_model(vals, q)
            assert got.dtype == want.dtype and (got == want or (np.isnan(got) and np.isnan(want))), (n, q, got, want)


def test_float32_plans_in_float32():
    """np.percentile of a float32 array is float32: q / float32(100), the index and the lerp are float32, so the ranks and weights
    differ from a float64 plan for some (n, q), and q = 99.99999999 is 100 in float32"""
    rng = np.random.default_rng(12)
    differ = 0
    for n in range(2, 400):
        v = rng.standard_normal(n).astype(np.float32)
        for q in (0.1, 1.3, 33.3, 66.7, 99.9):
            p32, p64 = pct_plan(n, q, np.float32), pct_plan(n, q, np.float64)
            differ += (p32[0], np.float32(p32[2] - p32[0])) != (p64[0], np.float32(p64[2] - p64[0]))
            assert percentile_model(v, q) == np.percentile(v, q)
    assert differ > 0
    assert np.percentile(np.float32([1, 2]), 99.99999999) == np.float32(2)
    with pytest.raises(ValueError, match=r"Percentiles must be in the range \[0, 100\]"):
        np.percentile(np.float64([1, 2]), 99.99999999 + 1e-6)


def test_integer_difference_wraps_as_numpy():
    v = np.array([-30000, 30000], np.int16)
    assert percentile_model(v, 50) == np.percentile(v, 50) == 32768.0       # b - a wrapped to -5536
    v = np.array([-2**31, 2**31 - 1], np.int32)
    assert percentile_model(v, 25) == np.percentile(v, 25)


def test_signed_zero_at_the_end():
    """one pixel of -0.0: numpy's weight there is 1, and b - (b - a) * 0 keeps the sign"""
    v = np.array([-0.0])
    assert np.signbit(np.percentile(v, 0)) and np.signbit(percentile_model(v, 0))
    v = np.array([-0.0, -0.0])
    assert np.signbit(np.percentile(v, 100)) == np.signbit(percentile_model(v, 100))
