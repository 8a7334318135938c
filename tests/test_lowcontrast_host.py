"""CPU: core.contrast, LowContrastDiskROI, planar_imaging.percent_integral_uniformity and the host arithmetic of
analyze_low_contrast_batch against the goldens of the unmodified reference, with the device's disk statistics and percentiles replaced
by numpy's over the same pixels."""
import json

import numpy as np
import pytest

from oracle.skimage_draw import disk
from pylinac_b200 import _native as nat
from pylinac_b200 import planar_imaging
from pylinac_b200.core import contrast as pcontrast
from pylinac_b200.core import roi as proi
from tests.golden.lowcontrast_cases import BATCH_CASES, LEEDS_BG, LEEDS_LIKE, ROI_CASES
from tests.golden.make_lowcontrast_golden import contrast_records, roi_records

GOLDEN = np.load("tests/golden/lowcontrast_golden.npz")


def _frames(frames):
    a = np.asarray(frames)
    return a[None] if a.ndim == 2 else a


def numpy_disk_stats(ctx, frames, disks):
    a = _frames(frames)
    out = {k: np.full(len(disks), np.nan) for k in nat.DISK_STATS}
    for i, (f, cy, cx, r) in enumerate(disks):
        v = a[int(f)][disk((cy, cx), r)]
        out["count"][i] = v.size
        if v.size:
            for k, fn in (("mean", np.mean), ("std", np.std), ("min", np.min), ("max", np.max), ("median", np.median)):
                out[k][i] = fn(v)
    return out


def numpy_disk_percentiles(ctx, frames, disks, q):
    a = _frames(frames)
    out = np.full((len(disks), len(q)), np.nan)
    for i, (f, cy, cx, r) in enumerate(disks):
        v = a[int(f)][disk((cy, cx), r)]
        if v.size:
            out[i] = [float(np.percentile(v, x)) for x in q]
    return out


@pytest.fixture
def numpy_device(monkeypatch):
    monkeypatch.setattr(nat, "disk_stats", numpy_disk_stats)
    monkeypatch.setattr(nat, "disk_percentiles", numpy_disk_percentiles)
    monkeypatch.setattr(nat.Context, "default", classmethod(lambda cls, device=None: None))


def test_contrast_functions_match_the_reference():
    assert json.dumps(contrast_records(pcontrast), sort_keys=True) == str(GOLDEN["contrast"])


@pytest.mark.parametrize("name", sorted(ROI_CASES))
def test_low_contrast_roi_matches_the_reference(name, numpy_device):
    assert json.dumps(roi_records(name, proi), sort_keys=True) == str(GOLDEN["roi:" + name])


def batch_as_record(res) -> list:
    return [{"background": f.background, "piu": f.piu,
             "rois": [{"median": m, "std": s, "contrast": c, "cnr": cn, "snr": sn, "visibility": v, "passed_visibility": pv,
                       "percentiles": p}
                      for m, s, c, cn, sn, v, pv, p in zip(f.medians, f.stds, f.contrasts, f.cnrs, f.snrs, f.visibilities,
                                                           f.passed_visibility, f.percentiles)]} for f in res]


def run_batch(name, frames=None):
    build, geom, kw = BATCH_CASES[name]
    return proi.analyze_low_contrast_batch(build() if frames is None else frames, geom["center"], geom["angle"], geom["radius"],
                                           LEEDS_LIKE, LEEDS_BG, **kw)


@pytest.mark.parametrize("name", sorted(BATCH_CASES))
def test_batch_arithmetic_matches_the_reference(name, numpy_device):
    assert json.dumps(batch_as_record(run_batch(name)), sort_keys=True) == str(GOLDEN["batch:" + name])


def test_batch_geometry_per_frame(numpy_device):
    """per-frame geometry arrays give each frame the result of its own scalar geometry"""
    build, geom, kw = BATCH_CASES["leeds_u16"]
    frames = build()
    n = len(frames)
    per = proi.analyze_low_contrast_batch(frames, [geom["center"]] * n, [geom["angle"], 2.0, -1.0], np.full(n, geom["radius"]),
                                          LEEDS_LIKE, LEEDS_BG)
    for f, a in enumerate([geom["angle"], 2.0, -1.0]):
        one = proi.analyze_low_contrast_batch(frames[f], geom["center"], a, geom["radius"], LEEDS_LIKE, LEEDS_BG)[0]
        assert batch_as_record([per[f]]) == batch_as_record([one])
    with pytest.raises(ValueError, match="phantom_angle has 2 entries for 3 frames"):
        proi.analyze_low_contrast_batch(frames, geom["center"], [0.0, 1.0], geom["radius"], LEEDS_LIKE, LEEDS_BG)


def test_batch_takes_the_phantom_centre_as_a_point(numpy_device):
    """ImagePhantomBase.phantom_center is a Point: a Point, n Points and a mix give the result of the (x, y) form"""
    build, geom, kw = BATCH_CASES["leeds_rotated_weber"]
    frames = build()
    n = len(frames)
    want = batch_as_record(run_batch("leeds_rotated_weber", frames))
    p = proi.Point(*geom["center"])
    for center in (p, [p] * n, [p, geom["center"], p], np.array([geom["center"]] * n)):
        got = proi.analyze_low_contrast_batch(frames, center, geom["angle"], geom["radius"], LEEDS_LIKE, LEEDS_BG, **kw)
        assert batch_as_record(got) == want
    with pytest.raises(ValueError, match="phantom_center has 2 entries for 3 frames"):
        proi.analyze_low_contrast_batch(frames, [p, p], geom["angle"], geom["radius"], LEEDS_LIKE, LEEDS_BG)


def test_batch_raises_the_reference_s_errors(numpy_device):
    build, geom, _ = BATCH_CASES["leeds_u16"]
    frames = build()
    with pytest.raises(ValueError, match="did not match any valid options"):
        proi.analyze_low_contrast_batch(frames, geom["center"], 0.0, geom["radius"], LEEDS_LIKE, LEEDS_BG, contrast_method="x")
    with pytest.raises(ValueError, match="^RMS calculations require"):
        proi.analyze_low_contrast_batch(frames, geom["center"], 0.0, geom["radius"], LEEDS_LIKE, LEEDS_BG,
                                        contrast_method="Root Mean Square")
    with pytest.raises(ValueError, match=r"^Percentiles must be in the range \[0, 100\]$"):
        proi.analyze_low_contrast_batch(frames, geom["center"], 0.0, geom["radius"], LEEDS_LIKE, LEEDS_BG, percentiles=(1, 101))
    with pytest.raises(IndexError, match="out of bounds"):
        proi.analyze_low_contrast_batch(frames, geom["center"], 0.0, 200.0, LEEDS_LIKE, LEEDS_BG)
    with pytest.raises(TypeError):
        run_batch("leeds_u16")[0].passed                 # no contrast threshold, as in the reference
    assert run_batch("leeds_int16_difference")[0].passed == [c > 10.0 for c in run_batch("leeds_int16_difference")[0].contrasts]


def test_percent_integral_uniformity():
    assert planar_imaging.percent_integral_uniformity(max=1100.0, min=900.0) == 100 * (1 - (200.0 + 1e-6) / (2000.0 + 1e-6))
    assert planar_imaging.percent_integral_uniformity(max=0.0, min=0.0) == 0.0


def test_unsupported_percentile_dtypes():
    a = np.zeros((16, 16), np.int8)
    roi = proi.LowContrastDiskROI(a, radius=3, center=proi.Point(8, 8))
    with pytest.raises(NotImplementedError, match="int8"):
        roi.percentile(50)
