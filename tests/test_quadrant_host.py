"""CPU: QuadrantResolution's host geometry (the ROI centres, the rows-as-x centre, bar widths as dict keys) and core.mtf's moments
MTF against the goldens of the unmodified reference."""
import json
import math

import numpy as np
import pytest

from pylinac_b200 import nuclear
from pylinac_b200.core.geometry import Point
from pylinac_b200.core.mtf import MomentMTF, moments_fwhm, moments_mtf
from pylinac_b200.core.roi import DiskROI
from tests.golden.quadrant_cases import CASES

GOLDEN = np.load("tests/golden/quadrant_golden.npz")
WITH_ROIS = sorted(n for n in CASES if "rois" in json.loads(str(GOLDEN[n])))


@pytest.mark.parametrize("name", WITH_ROIS)
def test_roi_centres_are_the_reference_s(name):
    rec = json.loads(str(GOLDEN[name]))
    build, kw = CASES[name]
    _, h, w = build().shape
    centers = nuclear._quadrant_centers(h, w, kw["bar_widths"], kw.get("distance_from_center_mm", 130))
    assert [[float(k), [c.x, c.y]] for k, c in centers.items()] == [[k, r["center"]] for k, r in rec["rois"]]
    assert all(r["radius"] == kw.get("roi_diameter_mm", 70) for _, r in rec["rois"])


@pytest.mark.parametrize("name", WITH_ROIS)
def test_moment_mtf_from_the_golden_statistics(name):
    rec = json.loads(str(GOLDEN[name]))
    if any("error" in r["circle_mask"] for _, r in rec["rois"]):
        return
    lpmm = 1 / (2 * np.asarray(CASES[name][1]["bar_widths"]))
    means = [r["mean"]["value"] for _, r in rec["rois"]]
    stds = [r["std"]["value"] for _, r in rec["rois"]]
    try:
        mtf = MomentMTF(lpmm, means, stds)
    except Exception as e:  # noqa: BLE001 -- compared with the reference's exception
        assert [type(e).__name__, str(e)] == rec["analyze_error"]
        return
    assert "analyze_error" not in rec
    assert json.dumps([[float(k), float(v)] for k, v in mtf.mtfs.items()]) == json.dumps(rec["mtfs"])
    assert json.dumps([[float(k), float(v)] for k, v in mtf.fwhms.items()]) == json.dumps(rec["fwhms"])


def test_moments_raise_as_the_reference():
    with pytest.raises(ValueError, match="math domain error"):
        moments_mtf(100.0, 9.0)            # std**2 < mean
    with pytest.raises(ZeroDivisionError):
        moments_mtf(0.0, 0.0)              # a blank ROI
    with pytest.raises(ValueError, match="math domain error"):
        moments_fwhm(1.0, 10.0, 20.0)      # MTF above 1: the log is negative
    assert moments_mtf(100.0, 30.0) == math.sqrt(2 * (30.0**2 - 100.0)) / 100.0


def test_bar_width_count_and_centre_quirks():
    for widths in ([1, 2, 3], [1, 2, 3, 4, 5], []):
        with pytest.raises(ValueError, match="Must have 4 bar widths"):
            nuclear.analyze_quadrant_resolution_batch(np.zeros((1, 8, 8), np.uint16), widths)
    # rows give x: on a 300 x 600 frame the centre is (x 150, y 300)
    c = nuclear._quadrant_centers(300, 600, [1, 2, 3, 4], 0)
    assert [(p.x, p.y) for p in c.values()] == [(150.0, 300.0)] * 4
    # a repeated width keeps its first position and its last centre
    c = nuclear._quadrant_centers(512, 512, [3, 2, 3, 1], 100)
    assert list(c) == [3, 2, 1]
    assert c[3].x < 256 and c[3].y < 256             # the -135 degree disk replaced the 45 degree one


def test_shifted_center_expressions():
    p = DiskROI._get_shifted_center(-135, 130, Point(256, 256))
    assert (p.x, p.y) == (256 + np.cos(np.deg2rad(-135)) * 130, 256 + np.sin(np.deg2rad(-135)) * 130)


def test_masked_array_keeps_the_disk_and_clips_to_the_frame():
    a = np.arange(20 * 30, dtype=np.float64).reshape(20, 30)
    m = DiskROI(a, radius=6.5, center=Point(3.2, 4.7)).masked_array()      # the disk crosses the top-left corner: clipped, no wrap
    inside = ~np.isnan(m)
    yy, xx = np.mgrid[0:20, 0:30]
    want = ((yy - 4.7) / 6.5) ** 2 + ((xx - 3.2) / 6.5) ** 2 < 1
    assert np.array_equal(inside, want) and np.array_equal(m[inside], a[inside])
    assert DiskROI(a.astype(np.uint16), radius=3, center=Point(10, 10)).masked_array().dtype == np.uint16   # the image's dtype
