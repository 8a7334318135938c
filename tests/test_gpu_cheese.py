"""GPU: TomoCheese / CIRS062M on the seeded series of tests/golden/cheese_cases.py, written as DICOM and read back, equal (==) to the
unmodified reference's results in tests/golden/cheese_golden.npz: every slice's localization row, origin slice, roll, ROI dicts,
results(), results_data(), printed messages and exceptions.  A seeded fuzz compares each stage of epid_ct_localize with
oracle/ct_oracle.py bit for bit, and its Gaussian (mode 'nearest') with ndimage.gaussian_filter."""
import contextlib
import io
import json

import numpy as np
import pytest
from scipy import ndimage

from oracle import ct_oracle
from pylinac_b200 import _native as nat
from pylinac_b200 import cheese
from tests.ct_writer import write_ct_slice
from tests.golden.cheese_cases import ANALYZE, CASES, case_series
from tests.golden.make_cheese_golden import ROW_KEYS

pytestmark = pytest.mark.gpu
GOLDEN = np.load("tests/golden/cheese_golden.npz")


def write_case(name, directory):
    raw, slopes, intercepts, px, thk = case_series(name)
    order = np.random.default_rng(5).permutation(len(raw))
    for k, z in enumerate(order):
        write_ct_slice(directory / f"CT{k:04d}.dcm", raw[z], series_uid="1.2.826.0.1.3680043.2.7", z=z * thk, slice_thickness=thk,
                       pixel_spacing=px, slope=slopes[z], intercept=intercepts[z])


def _jsonable(x):
    return json.loads(json.dumps(x))


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_matches_reference(name, tmp_path):
    write_case(name, tmp_path)
    ph = getattr(cheese, CASES[name]["phantom"])(str(tmp_path))
    rows = ph.localization(ph.clear_borders)
    got = np.array([[r[k] for k in ROW_KEYS] for r in rows], dtype=np.float64)
    gold = GOLDEN[f"{name}/rows"]
    np.testing.assert_array_equal(got[:, :4], gold[:, :4])
    np.testing.assert_array_equal(got[:, 4:6], gold[:, 4:6])
    ok = gold[:, 0] != ct_oracle.NO_EDGES
    np.testing.assert_array_equal(got[:, 6], gold[:, 6])
    np.testing.assert_array_equal(got[ok, 7], gold[ok, 7])
    for rec in json.loads(str(GOLDEN[f"{name}/reference"])):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            if "error" in rec:
                with pytest.raises(Exception) as ei:
                    ph.analyze(**rec["kwargs"])
                assert (type(ei.value).__name__, str(ei.value)) == (rec["error"], rec["message"])
            else:
                ph.analyze(**rec["kwargs"])
                assert ph.origin_slice == rec["origin_slice"]
                assert float(ph.catphan_roll) == rec["catphan_roll"]
                assert _jsonable({k: r.as_dict() for k, r in ph.module.rois.items()}) == rec["rois"]
                assert ph.results() == rec["results"]
                assert ph.results(as_list=True) == rec["results_list"]
                rd, gold_rd = _jsonable(ph.results_data(as_dict=True)), dict(rec["results_data"])
                for k in ("pylinac_version", "date_of_analysis"):      # which package made the result, and when
                    rd.pop(k), gold_rd.pop(k)
                assert rd == gold_rd
        assert buf.getvalue() == rec["stdout"]


@pytest.mark.parametrize("seed", range(6))
def test_stages_match_oracle(seed):
    rng = np.random.default_rng(100 + seed)
    h, w = [(37, 53), (64, 64), (100, 131), (257, 129), (33, 300), (200, 200)][seed]
    n = 3
    yy, xx = np.mgrid[0:h, 0:w]
    vol = np.empty((n, h, w), np.int16)
    for z in range(n):
        r = np.hypot(yy - h / 2 - rng.normal(0, 3), xx - w / 2 - rng.normal(0, 3))
        hu = np.where(r < min(h, w) * rng.uniform(0.2, 0.45), rng.normal(0, 40, (h, w)), -1000 + rng.normal(0, 15, (h, w)))
        if z == 1:
            hu[h // 3, w // 3] = 3000.0                      # metal: clipping matters
            hu[-3:, :] = 200.0                                # a couch on the border
        if z == 2 and seed % 2:
            hu[:] = -1000.0                                   # nothing in view
        vol[z] = np.rint(hu + 1024).astype(np.int16)
    slope, icpt = np.array([1.0, 0.5, 1.0]), np.array([-1024.0, -1000.0, -1024.0])
    vol[1] = np.rint((vol[1].astype(float) - 1024 + 1000) / 0.5).clip(-32768, 32767).astype(np.int16)
    size = np.pi * (min(h, w) * 0.35) ** 2
    for clear in (True, False):
        rows, st = nat.ct_localize(nat.Context.default(), vol, slope, icpt, [2, 0, 1], size, clear, stages=True)
        for k, z in enumerate([2, 0, 1]):
            o = ct_oracle.localize_slice(vol[z], slope[z], icpt[z], size, clear)
            r = rows[k]
            assert r["status"] == o["status"] and r["max_edge"] == o["max_edge"], (seed, z)
            if o["status"] == ct_oracle.NO_EDGES:
                continue
            assert np.array_equal(st["scharr"][k], o["scharr"])
            assert np.array_equal(st["smoothed"][k], o["smoothed"])
            assert np.array_equal(st["smoothed"][k], ndimage.gaussian_filter(st["scharr"][k], 1, mode="nearest", truncate=4.0))
            assert r["threshold"] == o["threshold"]
            assert np.array_equal(st["filled"][k], o["filled"])
            assert np.array_equal(st["labels"][k], o["labels"])
            assert (r["n_regions"], r["label"], r["area"]) == (o["n_regions"], o["label"], o["area"])
            if o["n_regions"]:
                assert (r["centroid_row"], r["centroid_col"]) == (o["centroid_row"], o["centroid_col"])


def test_rows_and_stages_across_chunks():
    """1024 x 1024 slices run 16 to a chunk: 18 listed slices take two chunks.  Every row equals the oracle's, and the stage planes
    of the slices on both sides of the chunk boundary equal the oracle's planes."""
    rng = np.random.default_rng(7)
    n, h, w = 18, 1024, 1024
    yy, xx = np.mgrid[0:h, 0:w]
    vol = np.empty((n, h, w), np.int16)
    for z in range(n):
        r = np.hypot(yy - 500 - z, xx - 520 + 2 * z)
        hu = np.where(r < 300 + 5 * z, rng.normal(0, 20, (h, w)), -1000.0)
        hu[np.hypot(yy - 500, xx - 700) < 20] = 2500.0 if z % 3 == 0 else 300.0
        if z == 5:
            hu[:] = -1000.0
        vol[z] = np.rint(hu + 1024).astype(np.int16)
    slope, icpt = np.ones(n), np.full(n, -1024.0)
    order = rng.permutation(n)
    size = np.pi * 330.0**2
    rows, st = nat.ct_localize(nat.Context.default(), vol, slope, icpt, order, size, True, stages=True)
    for k, z in enumerate(order):
        o = ct_oracle.localize_slice(vol[z], slope[z], icpt[z], size, True)
        got = [rows[k][key] for key in ROW_KEYS]
        want = [o.get(key, np.nan) for key in ROW_KEYS]
        if o["status"] == ct_oracle.NO_EDGES:
            got[7] = want[7] = np.nan          # the oracle stops at the edge check
        np.testing.assert_array_equal(np.array(got, float), np.array(want, float), err_msg=f"slice {z}")
        if k in (0, 15, 16, 17) and o["status"] != ct_oracle.NO_EDGES:
            for plane in ("scharr", "smoothed", "filled", "labels"):
                assert np.array_equal(st[plane][k], o[plane]), (plane, k, z)


def test_chunks_of_tiny_slices_stay_within_the_grid():
    """70 000 slices of 4 x 4: the chunk is capped at 65 535 slices (the grid's z limit), so two chunks run"""
    vol = np.full((70000, 4, 4), 24, np.int16)
    vol[69999, 1, 1] = 1024
    rows = nat.ct_localize(nat.Context.default(), vol, 1.0, -1024.0, np.arange(70000), 4.0, False)
    assert (rows["status"][:-1] == nat.CT_NO_EDGES).all() and (rows["n_regions"][:-1] == 0).all()
    assert rows["status"][-1] != nat.CT_NO_EDGES and rows["max_edge"][-1] > 0.1
