"""CPU: the QuadrantResolution / DiskROI goldens against numpy on the restated skimage.draw.disk, the product's host restatement of
disk() and of numpy's IndexError against the oracle's, and a numpy model of epid_disk_stats' summation orders against numpy itself."""
import json

import numpy as np
import pytest

from oracle.skimage_draw import disk as oracle_disk
from pylinac_b200.core import roi as proi
from tests.golden.nuclear_cases import digest
from tests.golden.quadrant_cases import CASES, DISK_CASES

GOLDEN = np.load("tests/golden/quadrant_golden.npz")


def golden(name):
    return json.loads(str(GOLDEN[name]))


def _roi_checks(frame, rec):
    cx, cy = rec["center"]
    r = rec["radius"]
    rr, cc = oracle_disk((cy, cx), r)
    prr, pcc = proi.disk((cy, cx), r)
    assert np.array_equal(rr, prr) and np.array_equal(cc, pcc)
    if "error" in rec["circle_mask"]:
        with pytest.raises(IndexError) as e:
            frame[rr, cc]
        assert [type(e.value).__name__, str(e.value)] == rec["circle_mask"]["error"]
        with pytest.raises(IndexError) as e:
            proi.check_disk_bounds(frame.shape, cy, cx, r)
        assert [type(e.value).__name__, str(e.value)] == rec["circle_mask"]["error"]
        return
    proi.check_disk_bounds(frame.shape, cy, cx, r)
    vals = frame[rr, cc]
    assert digest(vals) == rec["circle_mask"] and vals.size == rec["count"]
    if vals.size == 0:
        assert np.isnan(rec["mean"]["value"]) and rec["min"]["error"][0] == "ValueError"
        return
    for name, fn in (("mean", np.mean), ("std", np.std), ("pixel_value", np.median), ("min", np.min), ("max", np.max)):
        assert float(fn(vals)) == rec[name]["value"], name


@pytest.mark.parametrize("name", sorted(CASES))
def test_quadrant_golden_is_numpy_on_the_restated_disk(name):
    rec = golden(name)
    frame = CASES[name][0]()[0]
    for _, roi in rec.get("rois", []):
        _roi_checks(frame, roi)


@pytest.mark.parametrize("name", sorted(DISK_CASES))
def test_disk_golden_is_numpy_on_the_restated_disk(name):
    build, disks = DISK_CASES[name]
    arr = build()
    for (cy, cx, r), rec in zip(disks, golden("disk:" + name)):
        assert rec["center"] == [cx, cy]
        _roi_checks(arr, rec)


def test_host_disk_matches_the_oracle_on_random_disks():
    rng = np.random.default_rng(5)
    for _ in range(400):
        cy, cx = rng.uniform(-40, 40, 2)
        r = rng.choice([rng.uniform(0.05, 3), rng.uniform(3, 60)])
        a, b = oracle_disk((cy, cx), r), proi.disk((cy, cx), r)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_check_disk_bounds_is_numpy_indexing():
    """negative indices down to -size wrap; anything beyond raises numpy's IndexError, whichever axis and side it is on"""
    rng = np.random.default_rng(6)
    shape = (37, 53)
    arr = np.zeros(shape, np.uint8)
    raised = 0
    for _ in range(600):
        cy, cx = rng.uniform(-60, 80, 2)
        r = rng.uniform(0.2, 20)
        rr, cc = proi.disk((cy, cx), r)
        try:
            arr[rr, cc]
            expect = None
        except IndexError as e:
            expect = str(e)
        try:
            proi.check_disk_bounds(shape, cy, cx, r)
            got = None
        except IndexError as e:
            got = str(e)
        assert got == expect, (cy, cx, r)
        raised += expect is not None
    assert 100 < raised < 500


# ---------------------------------------------------------------------------------------- the summation orders of epid_disk_stats
def _leaf(x, A):
    n = len(x)
    if n < 8:
        res = A(-0.0)
        for v in x:
            res = A(res + v)
        return res
    r = [A(v) for v in x[:8]]
    i = 8
    while i < n - n % 8:
        for k in range(8):
            r[k] = A(r[k] + x[i + k])
        i += 8
    res = A(A(A(r[0] + r[1]) + A(r[2] + r[3])) + A(A(r[4] + r[5]) + A(r[6] + r[7])))
    for v in x[i:]:
        res = A(res + v)
    return res


def _pw(x, A):
    if len(x) <= 128:
        return _leaf(x, A)
    n2 = len(x) // 2
    n2 -= n2 % 8
    return A(_pw(x[:n2], A) + _pw(x[n2:], A))


def disk_stats_model(vals):
    """mean / std / median of the kernel's expressions (csrc/roi.cu k_disk_stats) in numpy scalars"""
    A = np.float32 if vals.dtype == np.float32 else np.float64
    x = vals.astype(A)
    n = len(x)
    step = 8192 if np.issubdtype(vals.dtype, np.integer) else n
    s = A(0.0)
    for c in range(0, n, step):
        s = A(s + _pw(x[c:c + step], A))
    mean = A(np.float64(s) / n)
    d = x - mean
    ss = A(A(0.0) + _pw(d * d, A))
    std = np.sqrt(A(np.float64(ss) / n))
    srt = np.sort(vals)
    a = A(srt[(n - 1) // 2])
    if n % 2:
        med = A(np.float64(A(A(0.0) + A(A(-0.0) + a))) / 1.0)
    else:
        b = A(srt[n // 2])
        med = A(np.float64(A(A(0.0) + A(A(A(-0.0) + a) + b))) / 2.0)
    return float(mean), float(std), float(med)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64])
def test_summation_model_is_numpy(dtype):
    """numpy's mean (float64 chunks of 8192 for integers, float32 sums for float32), std and median of a raster-ordered gather"""
    rng = np.random.default_rng(7)
    for n in (1, 2, 7, 8, 127, 129, 1000, 8193, 20001):
        if dtype == np.int64:
            v = rng.integers(-2**62, 2**62, n)
        elif np.issubdtype(dtype, np.integer):
            info = np.iinfo(dtype)
            v = rng.integers(info.min, int(info.max) + 1, n)
        else:
            v = rng.standard_normal(n) * 1e4
        v = v.astype(dtype)
        assert disk_stats_model(v) == (float(np.mean(v)), float(np.std(v)), float(np.median(v))), n
