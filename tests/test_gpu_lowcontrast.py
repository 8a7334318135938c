"""GPU: LowContrastDiskROI, core.contrast and the low-contrast batch against the goldens of the unmodified reference, bit for bit
(values with their types, warnings, exception types and messages); a seeded fuzz of epid_disk_percentiles against
np.percentile(arr[disk(...)], q) compared with == for every dtype; and the batch against ROI-by-ROI calls and device-resident input."""
import json

import numpy as np
import pytest

from oracle.skimage_draw import disk
from pylinac_b200 import _native as nat
from pylinac_b200.core import roi as proi
from tests.golden.lowcontrast_cases import BATCH_CASES, LEEDS_BG, LEEDS_LIKE, ROI_CASES
from tests.golden.make_lowcontrast_golden import roi_records
from tests.test_lowcontrast_host import batch_as_record, run_batch

pytestmark = pytest.mark.gpu
GOLDEN = np.load("tests/golden/lowcontrast_golden.npz")


@pytest.mark.parametrize("name", sorted(ROI_CASES))
def test_low_contrast_roi_matches_the_reference(name):
    assert json.dumps(roi_records(name, proi), sort_keys=True) == str(GOLDEN["roi:" + name])


@pytest.mark.parametrize("name", sorted(BATCH_CASES))
def test_batch_matches_the_reference(name):
    assert json.dumps(batch_as_record(run_batch(name)), sort_keys=True) == str(GOLDEN["batch:" + name])


def _frame(rng, dtype, shape):
    if np.issubdtype(dtype, np.integer):
        info = np.iinfo(dtype)
        a = rng.integers(info.min, int(info.max) + 1, shape)
        if rng.uniform() < 0.5:                      # a narrow band too: many repeated values, so ranks share keys
            a = rng.integers(info.min // 2 + 100, info.min // 2 + 140, shape) if info.min < 0 else rng.integers(100, 140, shape)
        return a.astype(dtype)
    a = (rng.standard_normal(shape) * 1e4 + 3).astype(dtype)
    if rng.uniform() < 0.3:
        a[rng.integers(0, shape[0]), rng.integers(0, shape[1])] = np.nan
    return a


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.int16, np.int32, np.int64, np.float32, np.float64])
def test_disk_percentiles_fuzz_matches_numpy(dtype):
    rng = np.random.default_rng(2000 + np.dtype(dtype).num)
    ctx = nat.Context.default()
    mismatches = []
    for trial in range(4):
        h, w = 200 + trial * 7, 230 + trial * 11
        frames = np.stack([_frame(rng, dtype, (h, w)) for _ in range(3)])
        disks = []
        for f in range(3):
            for _ in range(20):
                r = float(rng.choice([rng.uniform(0.3, 3), rng.uniform(3, 30), rng.uniform(30, 90)]))
                disks.append((f, float(rng.uniform(-5, h - r)), float(rng.uniform(-5, w - r)), r))
        q = [float(x) for x in rng.uniform(0, 100, 5)] + [0, 1, 99, 100, 50.0, 2.5]
        got = nat.disk_percentiles(ctx, frames, disks, q)
        for i, (f, cy, cx, r) in enumerate(disks):
            v = frames[f][disk((cy, cx), r)]
            for k, x in enumerate(q):
                want = float(np.percentile(v, x)) if v.size else np.nan
                if not (got[i, k] == want or (np.isnan(got[i, k]) and np.isnan(want))):
                    mismatches.append((trial, i, x, got[i, k], want))
    assert not mismatches, mismatches[:10]


def test_float32_result_is_numpy_s_float32():
    a = np.random.default_rng(5).standard_normal((64, 64)).astype(np.float32)
    got = nat.disk_percentiles(nat.Context.default(), a, [(0, 30.2, 29.8, 20.5)], [33.3, 99.99999999])
    v = a[disk((30.2, 29.8), 20.5)]
    assert [float(np.percentile(v, 33.3)), float(np.percentile(v, 99.99999999))] == got[0].tolist()
    assert np.float32(got[0, 0]) == got[0, 0]                 # a float32 value, widened


def test_disk_percentiles_reject_bad_input():
    ctx = nat.Context.default()
    with pytest.raises(ValueError, match=r"Percentiles must be in the range \[0, 100\]"):
        nat.disk_percentiles(ctx, np.zeros((32, 32), np.uint16), [(0, 10.0, 10.0, 5.0)], [101])
    with pytest.raises(ValueError, match="beyond"):
        nat.disk_percentiles(ctx, np.zeros((32, 32), np.uint16), [(0, 30.0, 10.0, 5.0)], [50])


def test_batch_matches_roi_by_roi_and_device_input():
    build, geom, kw = BATCH_CASES["leeds_u16"]
    frames = build()
    batch = run_batch("leeds_u16", frames)
    with nat.Batch.upload(nat.Context.default(), frames) as b:
        device = run_batch("leeds_u16", b)
    assert batch_as_record(batch) == batch_as_record(device)
    for f, res in enumerate(batch):
        bg = [proi.LowContrastDiskROI.from_phantom_center(frames[f], geom["angle"] + s["angle"], geom["radius"] * s["roi radius"],
                                                          geom["radius"] * s["distance from center"], proi.Point(*geom["center"]))
              for s in LEEDS_BG.values()]
        background = np.mean([r.pixel_value for r in bg])
        rois = [proi.LowContrastDiskROI.from_phantom_center(frames[f], geom["angle"] + s["angle"], geom["radius"] * s["roi radius"],
                                                            geom["radius"] * s["distance from center"], proi.Point(*geom["center"]),
                                                            None, background)
                for s in LEEDS_LIKE.values()]
        proi.fill_disk_percentiles(rois, (1, 99))
        assert res.background == background
        assert res.medians == [r.pixel_value for r in rois] and res.stds == [r.std for r in rois]
        assert res.contrasts == [r.contrast for r in rois] and res.visibilities == [r.visibility for r in rois]
        assert res.cnrs == [r.contrast_to_noise for r in rois] and res.snrs == [r.signal_to_noise for r in rois]
        assert res.percentiles == [[r.percentile(1), r.percentile(99)] for r in rois]


def test_fill_disk_percentiles_is_one_call():
    a = np.random.default_rng(6).integers(0, 4000, (128, 128)).astype(np.uint16)
    rois = [proi.LowContrastDiskROI(a, radius=7.5, center=proi.Point(20 + 10 * i, 64)) for i in range(9)]
    ctx = nat.Context.default()
    proi.fill_disk_stats(rois)
    before = ctx.launches()
    proi.fill_disk_percentiles(rois, (1, 99))
    assert ctx.launches() == before + 1
    assert [r.percentile(99) for r in rois] == [float(np.percentile(r.circle_mask(), 99)) for r in rois]
    assert ctx.launches() == before + 1
