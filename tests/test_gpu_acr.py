"""GPU: ACRCT on the seeded series of tests/golden/acr_cases.py, written as DICOM and read back, equal (==) to the unmodified
reference's results in tests/golden/acr_golden.npz: every slice's localization row, the roll slice's region table, origin slice, roll,
every ROI value, results(), results_data() and the warnings.  Seeded fuzz compares the Slice branch of epid_ct_localize and the region
table of epid_ct_regions with oracle/acr_oracle.py bit for bit, on random slices and on crafted ones whose masks hold nested rings,
regions inside another's hole, holes open to the bbox edge, one-pixel spirals and a ring around the whole frame."""
import json
import warnings

import numpy as np
import pytest
from scipy import ndimage

from oracle import acr_oracle, ct_oracle
from pylinac_b200 import _native as nat
from pylinac_b200 import acr, cheese
from tests.ct_writer import write_ct_slice
from tests.golden.acr_cases import ANALYZE, CASES, case_series
from tests.golden.make_acr_golden import REGION_KEYS, ROW_KEYS

pytestmark = pytest.mark.gpu
GOLDEN = np.load("tests/golden/acr_golden.npz")


def write_case(name, directory):
    raw, slopes, intercepts, px, thk = case_series(name)
    order = np.random.default_rng(3).permutation(len(raw))
    for k, z in enumerate(order):
        write_ct_slice(directory / f"CT{k:04d}.dcm", raw[z], series_uid="1.2.826.0.1.3680043.2.9", z=z * thk, slice_thickness=thk,
                       pixel_spacing=px, slope=slopes[z], intercept=intercepts[z])


def _jsonable(x):
    return json.loads(json.dumps(x, default=str))


def module_rois(ph):
    out = {}
    for m in ("ct_calibration_module", "uniformity_module", "spatial_resolution_module", "low_contrast_module"):
        mod = getattr(ph, m)
        for group in ("rois", "background_rois"):
            for k, r in getattr(mod, group).items():
                out[f"{m}/{group}/{k}"] = [float(r.pixel_value), float(r.mean), float(r.std), float(r.min), float(r.max)]
    return out


def region_table(rows):
    return [{k: (tuple(int(v) for v in r[k]) if k == "bbox" else int(r[k])) for k in REGION_KEYS} for r in rows]


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_matches_reference(name, tmp_path):
    write_case(name, tmp_path)
    ph = acr.ACRCT(str(tmp_path))
    rows = ph.localization(ph.clear_borders)
    got = np.array([[r[k] for k in ROW_KEYS] for r in rows], dtype=np.float64)
    gold = GOLDEN[f"{name}/rows"]
    np.testing.assert_array_equal(got[:, :6], gold[:, :6])
    np.testing.assert_array_equal(got[:, 6], gold[:, 6])
    ok = gold[:, 0] != ct_oracle.NO_EDGES
    np.testing.assert_array_equal(got[ok, 7], gold[ok, 7])
    records = json.loads(str(GOLDEN[f"{name}/reference"]))
    second = acr.ACRCT(str(tmp_path))
    for rec in records:
        target = ph if rec["instance"] == 0 else second
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if "error" in rec:
                with pytest.raises(Exception) as ei:
                    target.analyze(**rec["kwargs"])
                assert (type(ei.value).__name__, str(ei.value)) == (rec["error"], rec["message"])
            else:
                target.analyze(**rec["kwargs"])
                assert target.origin_slice == rec["origin_slice"]
                assert float(target.catphan_roll) == rec["catphan_roll"]
                assert module_rois(target) == rec["rois"]
                assert target.results() == rec["results"]
                mtf50 = float(target.spatial_resolution_module.mtf.relative_resolution(50))
                assert mtf50 == rec["mtf50"] or (np.isnan(mtf50) and np.isnan(rec["mtf50"]))
                rd, gold_rd = _jsonable(target.results_data(as_dict=True)), dict(rec["results_data"])
                for k in ("pylinac_version", "date_of_analysis", "warnings"):      # which package made it, when, and where it warned
                    rd.pop(k), gold_rd.pop(k)
                assert rd == gold_rd
        assert [[str(w.message), w.category.__name__] for w in caught] == rec["warnings"]
    # the region table of the first analyze()'s roll slice
    if f"{name}/regions" in GOLDEN.files:
        raw, slopes, intercepts, px, thk = case_series(name)
        z = records[0]["origin_slice"]
        table, thres, max_edge = nat.ct_regions(nat.Context.default(), raw, slopes, intercepts, z, 110 / px, capacity=4)
        assert region_table(table) == [dict(r, bbox=tuple(r["bbox"])) for r in json.loads(str(GOLDEN[f"{name}/regions"]))]
        assert [thres, max_edge] == GOLDEN[f"{name}/region_threshold"].tolist()
        ecc = np.array([r.eccentricity for r in ph.get_regions(z)])
        gold_ecc = GOLDEN[f"{name}/eccentricity"]
        assert np.all(np.abs(ecc - gold_ecc) <= 1e-9) and np.array_equal(ecc < 0.5, gold_ecc < 0.5)


def _slices(seed, h, w):
    rng = np.random.default_rng(200 + seed)
    yy, xx = np.mgrid[0:h, 0:w]
    vol = np.empty((3, h, w), np.int16)
    for z in range(3):
        r = np.hypot(yy - h / 2 - rng.normal(0, 3), xx - w / 2 - rng.normal(0, 3))
        hu = np.where(r < min(h, w) * rng.uniform(0.2, 0.45), rng.normal(0, 40, (h, w)), -1000 + rng.normal(0, 15, (h, w)))
        for _ in range(6):                                   # bubbles and inserts
            cy, cx, rad = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, 9)
            hu[np.hypot(yy - cy, xx - cx) < rad] = rng.choice([-1000.0, 900.0, 3000.0])
        if z == 2 and seed % 2:
            hu[:] = 17.0                                      # constant: a constant disk
        vol[z] = np.rint(hu + 1024).clip(-32768, 32767).astype(np.int16)
    return vol


@pytest.mark.parametrize("seed", range(6))
def test_slice_branch_matches_oracle(seed):
    """Slice-branch rows and stages; the disk is larger than the slice for seeds 0 and 3 (it reaches past the image)"""
    h, w = [(37, 53), (64, 64), (100, 131), (257, 129), (33, 300), (200, 200)][seed]
    radius = [60.0, 20.0, 45.5, 200.0, 12.25, 90.0][seed]
    vol = _slices(seed, h, w)
    slope, icpt = np.array([1.0, 1.0, 1.0]), np.array([-1024.0, -1024.0, -1024.0])
    size = np.pi * (min(h, w) * 0.35) ** 2
    for clear in (True, False):
        rows, st = nat.ct_localize(nat.Context.default(), vol, slope, icpt, [2, 0, 1], size, clear, clip_in_localization=False,
                                   stages=True, otsu_disk_radius=radius)
        for k, z in enumerate([2, 0, 1]):
            o = acr_oracle.localize_slice(vol[z], slope[z], icpt[z], size, clear, radius)
            r = rows[k]
            assert r["status"] == o["status"] and r["max_edge"] == o["max_edge"], (seed, z)
            if o["status"] == ct_oracle.NO_EDGES:
                continue
            assert np.array_equal(st["scharr"][k], o["scharr"])
            assert np.array_equal(st["smoothed"][k], o["smoothed"])
            assert r["threshold"] == o["threshold"]
            assert np.array_equal(st["filled"][k], o["filled"])
            assert np.array_equal(st["labels"][k], o["labels"])
            assert (r["n_regions"], r["label"], r["area"]) == (o["n_regions"], o["label"], o["area"])
            if o["n_regions"]:
                assert (r["centroid_row"], r["centroid_col"]) == (o["centroid_row"], o["centroid_col"])


def test_disk_threshold_differs_from_whole_slice():
    """a slice whose disk Otsu threshold is not 0.8 x the whole-slice one: the disk changes which pixels Otsu sees"""
    vol = _slices(2, 100, 131)
    rows = nat.ct_localize(nat.Context.default(), vol, 1.0, -1024.0, [0], 10.0, False, clip_in_localization=False,
                           otsu_disk_radius=30.0)
    o = acr_oracle.localize_slice(vol[0], 1.0, -1024.0, 10.0, False, 30.0)
    whole = acr_oracle.skimage_ct.threshold_otsu(o["smoothed"]) * 0.8
    assert rows[0]["threshold"] == o["threshold"] != whole


def test_branch_arguments():
    vol = np.zeros((1, 8, 8), np.int16)
    ctx = nat.Context.default()
    with pytest.raises(NotImplementedError, match="without clipping"):
        nat.ct_localize(ctx, vol, 1.0, 0.0, [0], 10.0, True, clip_in_localization=False)
    with pytest.raises(ValueError, match="not clipped"):
        nat.ct_localize(ctx, vol, 1.0, 0.0, [0], 10.0, True, clip_in_localization=True, otsu_disk_radius=3.0)
    with pytest.raises(ValueError, match="below 1 pixel"):
        nat.ct_localize(ctx, vol, 1.0, 0.0, [0], 10.0, True, clip_in_localization=False, otsu_disk_radius=0.5)
    with pytest.raises(ValueError, match="otsu_disk_radius must be > 0"):
        nat.ct_regions(ctx, vol, 1.0, 0.0, 0, 0.0)


def _check_regions(raw, radius, capacity=3):
    table, thres, max_edge = nat.ct_regions(nat.Context.default(), raw[None], 1.0, -1024.0, 0, radius, capacity=capacity)
    regions, t, me, labels = acr_oracle.slice_regions(raw, 1.0, -1024.0, radius)
    assert (thres, max_edge) == (t, me)
    want = acr_oracle.region_rows(regions, raw.shape[1])
    assert region_table(table) == [dict(r, bbox=tuple(r["bbox"])) for r in want]
    for r in regions:      # the oracle's filled_area is ndimage.binary_fill_holes of each crop
        assert r.filled_area == int(ndimage.binary_fill_holes(r.image).sum())
    return table


@pytest.mark.parametrize("seed", range(6))
def test_region_table_matches_oracle(seed):
    h, w = [(37, 53), (64, 64), (100, 131), (257, 129), (33, 300), (200, 200)][seed]
    vol = _slices(seed, h, w)
    for z in range(3):
        _check_regions(vol[z], [60.0, 20.0, 45.5, 200.0, 12.25, 90.0][seed])


def _crafted(kind):
    """HU slices whose edge masks hold the shapes filled_area has to get right"""
    h = w = 160
    yy, xx = np.mgrid[0:h, 0:w]
    hu = np.full((h, w), -1000.0)
    r = np.hypot(yy - 80, xx - 80)
    if kind == "nested":
        for rad in (10, 22, 34, 46, 58):                      # rings of steps: nested edge rings
            hu[r < rad] += 600.0
    elif kind == "inside_hole":
        hu[(r > 40) & (r < 48)] = 800.0                        # a thick ring, and a blob in its hole
        hu[np.hypot(yy - 80, xx - 75) < 6] = 800.0
    elif kind == "open_hole":
        hu[(r > 30) & (r < 40)] = 800.0
        hu[(r > 30) & (r < 40) & (xx > 95) & (abs(yy - 80) < 5)] = -1000.0      # a gap: the hole opens to the bbox edge
    elif kind == "spiral":
        t = np.arctan2(yy - 80, xx - 80)
        arm = (r - 6 * (t + np.pi)) % 12
        hu[(arm < 3) & (r < 70) & (r > 4)] = 800.0
    elif kind == "frame_ring":
        hu[:] = 0.0
        hu[6:-6, 6:-6] = -1000.0
        hu[30:40, 30:130] = 900.0
    return np.rint(hu + 1024).astype(np.int16)


@pytest.mark.parametrize("kind", ["nested", "inside_hole", "open_hole", "spiral", "frame_ring"])
def test_filled_area_on_crafted_masks(kind):
    table = _check_regions(_crafted(kind), 200.0, capacity=1)
    assert len(table) >= 1


def test_cheese_rows_unchanged():
    """the ndarray branch (the cheese phantoms) still gives the golden rows of tests/golden/cheese_golden.npz"""
    from tests.golden.cheese_cases import CASES as CHEESE, case_series as cheese_series

    gold = np.load("tests/golden/cheese_golden.npz")
    for name in ("tomo_metal", "cirs_uint16"):
        raw, slopes, intercepts, px, _ = cheese_series(name)
        cls = getattr(cheese, CHEESE[name]["phantom"])
        size = np.pi * cls.catphan_radius_mm**2 / px**2
        rows = nat.ct_localize(nat.Context.default(), raw, slopes, intercepts, np.arange(len(raw)), size, cls.clear_borders)
        got = np.array([[r[k] for k in ROW_KEYS] for r in rows], dtype=np.float64)
        g = gold[f"{name}/rows"]
        ok = g[:, 0] != ct_oracle.NO_EDGES
        np.testing.assert_array_equal(got[:, :7], g[:, :7])
        np.testing.assert_array_equal(got[ok, 7], g[ok, 7])


def test_constant_disk():
    """the smoothed edges are 0.0 throughout the disk (a step far outside it): threshold_otsu's constant case, 0.0 x 0.8"""
    hu = np.full((96, 96), -1000.0)
    hu[:, 80:] = 300.0
    vol = np.rint(hu + 1024).astype(np.int16)[None]
    rows = nat.ct_localize(nat.Context.default(), vol, 1.0, -1024.0, [0], 100.0, False, clip_in_localization=False,
                           otsu_disk_radius=20.0)
    o = acr_oracle.localize_slice(vol[0], 1.0, -1024.0, 100.0, False, 20.0)
    assert rows[0]["threshold"] == o["threshold"] == 0.0 and rows[0]["status"] == o["status"]
    _check_regions(vol[0], 20.0)
