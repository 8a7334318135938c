"""GPU: QuadrantResolution and DiskROI against the goldens of the unmodified reference, bit for bit through NM files (results strings,
captured warnings, exception types and messages included); a seeded fuzz of epid_disk_stats against numpy on arr[disk(...)] compared
with ==; and the batch entry point against frame-by-frame calls and device-resident input."""
import contextlib
import json

import numpy as np
import pytest

from oracle.skimage_draw import disk
from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from pylinac_b200.core import roi as proi
from tests.golden.make_quadrant_golden import disk_record, record
from tests.golden.quadrant_cases import CASES, DISK_CASES, WIDTHS, bars

pytestmark = pytest.mark.gpu
GOLDEN = np.load("tests/golden/quadrant_golden.npz")


@pytest.mark.parametrize("name", sorted(CASES))
def test_quadrant_resolution_matches_the_reference(name, tmp_path):
    assert json.dumps(record(nuclear, name, tmp_path, opener=contextlib.nullcontext), sort_keys=True) == str(GOLDEN[name])


@pytest.mark.parametrize("name", sorted(DISK_CASES))
def test_disk_roi_matches_the_reference(name):
    assert json.dumps(disk_record(name, proi), sort_keys=True) == str(GOLDEN["disk:" + name])


def _frame(rng, dtype, shape):
    if dtype == np.int64:
        return rng.integers(-2**62, 2**62, shape).astype(np.int64)
    if np.issubdtype(dtype, np.integer):
        info = np.iinfo(dtype)
        return rng.integers(info.min, int(info.max) + 1, shape).astype(dtype)
    return (rng.standard_normal(shape) * 1e4 + 3).astype(dtype)


def _disks(rng, h, w):
    """fractional centres and radii from 0.3 to 150 px inside the frame, disks across the top and left edges (negative indices
    wrap), one-pixel disks, empty disks and disks of up to 70 k pixels"""
    out = []
    for _ in range(24):
        r = float(rng.choice([rng.uniform(0.3, 3), rng.uniform(3, 40), rng.uniform(40, 150)]))
        out.append((float(rng.uniform(r, h - r)), float(rng.uniform(r, w - r)), r))
    out += [(float(rng.uniform(-8, 3)), float(rng.uniform(20, w - 20)), float(rng.uniform(5, 15))),      # across the top edge
            (float(rng.uniform(20, h - 20)), float(rng.uniform(-8, 3)), float(rng.uniform(5, 15))),      # across the left edge
            (-2.5, -3.25, 9.5),                                                                          # across the corner
            (17.0, 23.0, 1.0), (5.0, 6.0, 0.7),                                                          # one pixel
            (12.5, 40.5, 0.3), (30.5, 7.5, 0.5),                                                         # empty
            (h / 2, w / 2, 150.0)]                                                                       # ~70 k pixels
    return out


def _expect(a, cy, cx, r):
    v = a[disk((cy, cx), r)]
    if v.size == 0:
        return {"count": 0}
    return {"count": v.size, "mean": float(np.mean(v)), "std": float(np.std(v)), "median": float(np.median(v)),
            "min": float(np.min(v)), "max": float(np.max(v))}


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64])
def test_disk_stats_fuzz_matches_numpy(dtype):
    rng = np.random.default_rng(1000 + np.dtype(dtype).num)
    ctx = nat.Context.default()
    mismatches = []
    for trial in range(3):
        h, w = 320 + trial * 7, 330 + trial * 11
        frames = np.stack([_frame(rng, dtype, (h, w)) for _ in range(2)])
        disks = [(f, *d) for f in range(2) for d in _disks(rng, h, w)]
        got = nat.disk_stats(ctx, frames, disks)
        for i, (f, cy, cx, r) in enumerate(disks):
            exp = _expect(frames[f], cy, cx, r)
            if got["count"][i] != exp["count"]:
                mismatches.append((trial, i, "count", got["count"][i], exp["count"]))
                continue
            if exp["count"] == 0:
                if not all(np.isnan(got[k][i]) for k in ("mean", "std", "median", "min", "max")):
                    mismatches.append((trial, i, "empty"))
                continue
            mismatches += [(trial, i, k, got[k][i], exp[k]) for k in ("mean", "std", "median", "min", "max") if got[k][i] != exp[k]]
    assert not mismatches, mismatches[:10]


def test_disk_stats_nan_pixels():
    a = np.random.default_rng(3).standard_normal((64, 64))
    a[30, 30] = np.nan
    got = nat.disk_stats(nat.Context.default(), a, [(0, 30.2, 29.8, 6.5), (0, 10.0, 10.0, 4.0)])
    for i, (cy, cx, r) in enumerate([(30.2, 29.8, 6.5), (10.0, 10.0, 4.0)]):
        v = a[disk((cy, cx), r)]
        for k, fn in (("mean", np.mean), ("std", np.std), ("median", np.median), ("min", np.min), ("max", np.max)):
            assert np.array_equal(got[k][i], fn(v), equal_nan=True), (i, k)


def test_disk_stats_rejects_a_disk_beyond_the_frame():
    with pytest.raises(ValueError, match="beyond"):
        nat.disk_stats(nat.Context.default(), np.zeros((32, 32), np.uint16), [(0, 30.0, 10.0, 5.0)])


def test_batch_matches_frame_by_frame_and_device_input():
    frames = np.concatenate([bars(s)[:1] for s in (31, 32, 33)] + [np.zeros((1, 512, 512), np.uint16)])
    batch = nuclear.analyze_quadrant_resolution_batch(frames, WIDTHS)
    with nat.Batch.upload(nat.Context.default(), frames) as b:
        device = nuclear.analyze_quadrant_resolution_batch(b, WIDTHS)
    for f, (one, dev) in enumerate(zip(batch, device)):
        single = nuclear.analyze_quadrant_resolution_batch(frames[f], WIDTHS)[0]
        for k in ("counts", "means", "stds", "medians", "mins", "maxs"):
            assert getattr(one, k) == getattr(single, k) == getattr(dev, k), (f, k)
        roi = proi.DiskROI(frames[f], radius=70, center=one.centers[0])
        assert (roi.mean, roi.std, roi.pixel_value, roi.min, roi.max) == (one.means[0], one.stds[0], one.medians[0], one.mins[0],
                                                                          one.maxs[0])
    assert batch[0].quadrants == nuclear.analyze_quadrant_resolution_batch(frames[:1], WIDTHS)[0].quadrants
    with pytest.raises(ZeroDivisionError):
        batch[3].mtf
    with pytest.raises(IndexError, match="out of bounds for axis 0 with size 256"):
        nuclear.analyze_quadrant_resolution_batch(frames[:, :256, :256], WIDTHS)


def test_batch_matches_the_golden_case():
    rec = json.loads(str(GOLDEN["u16_512"]))
    res = nuclear.analyze_quadrant_resolution_batch(CASES["u16_512"][0](), WIDTHS)[0]
    assert json.dumps([[float(k), float(v)] for k, v in res.mtf.mtfs.items()]) == json.dumps(rec["mtfs"])
    assert json.dumps([[float(k), float(v)] for k, v in res.mtf.fwhms.items()]) == json.dumps(rec["fwhms"])
    assert res.quadrants == rec["results_dict"]["value"]["quadrants"]
