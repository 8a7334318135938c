"""Generate tests/golden/acr_golden.npz: the UNMODIFIED reference ``pylinac.acr.ACRCT`` (stub-imported; skimage served by
oracle/acr_oracle.py over oracle/skimage_ct.py) on the seeded series of acr_cases.py, with the per-slice localization and the roll
slice's region table of oracle/acr_oracle.py, checked against the reference's own Slice.phantom_roi and get_regions.

pydicom is not installed here, so the series reaches the reference through a fake ``DicomImageStack`` holding each slice's HU array
(raw * slope + intercept in float64, as pydicom's apply_rescale gives it), its ImagePositionPatient and the SliceThickness /
PixelSpacing tags.

Run here (the container that has the reference):  python -m tests.golden.make_acr_golden
"""
from __future__ import annotations

import json
import types
import warnings

import numpy as np

from tests.golden.acr_cases import ANALYZE, CASES, EXPECT, case_series

ROW_KEYS = ("status", "n_regions", "label", "area", "centroid_row", "centroid_col", "max_edge", "threshold")
REGION_KEYS = ("label", "first", "area", "filled_area", "bbox", "sum_r", "sum_c", "m_rr", "m_cc", "m_rc")


def fake_stack_class(hu, px, thk):
    from pylinac.core import image as rimage

    class Img(rimage.ArrayImage):
        z_position = 0.0

    class FakeStack:
        def __init__(self, folder, check_uid=True, min_number=39, **kwargs):
            self.images = []
            for z, a in enumerate(hu):
                im = Img(a)
                im.z_position = z * thk
                self.images.append(im)
            self.metadatas = [types.SimpleNamespace(ImagePositionPatient=[0.0, 0.0, z * thk]) for z in range(len(hu))]
            self.metadata = types.SimpleNamespace(SliceThickness=thk, PixelSpacing=[px, px])
            self.slice_spacing = thk

        def __getitem__(self, i):
            return self.images[i]

        def __len__(self):
            return len(self.images)

        def __iter__(self):
            return iter(self.images)

    return FakeStack


def module_rois(ph):
    """every ROI value results_data does not show: each module ROI's median, mean, std, min and max"""
    out = {}
    for m in ("ct_calibration_module", "uniformity_module", "spatial_resolution_module", "low_contrast_module"):
        mod = getattr(ph, m)
        for group in ("rois", "background_rois"):
            for k, r in getattr(mod, group).items():
                out[f"{m}/{group}/{k}"] = [float(r.pixel_value), float(r.mean), float(r.std), float(r.min), float(r.max)]
    return out


def run_reference(cls, kwargs_list):
    """-> list of records: per analyze() call its results or error, and the warnings it raised.  The first instance runs every
    kwargs set and then the first once more; a second instance then runs the first set."""
    out = []
    first = cls(["unused"])
    calls = [(first, kw) for kw in kwargs_list + kwargs_list[:1]] + [(cls(["unused"]), kwargs_list[0])]
    for ph, kw in calls:
        rec = {"kwargs": kw, "instance": 0 if ph is first else 1}
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            try:
                ph.analyze(**kw)
                rd = ph.results_data(as_dict=True)
                rec.update(origin_slice=ph.origin_slice, catphan_roll=float(ph.catphan_roll), results=ph.results(),
                           results_data=json.loads(json.dumps(rd, default=str)), rois=module_rois(ph),
                           mtf50=float(ph.spatial_resolution_module.mtf.relative_resolution(50)))
            except Exception as e:  # noqa: BLE001 -- the reference's exception is part of the golden
                rec.update(error=type(e).__name__, message=str(e))
        rec["warnings"] = [[str(w.message), w.category.__name__] for w in caught]
        out.append(rec)
    return out


def check_expectations(name, rows, res, size, px):
    e = EXPECT[name]
    statuses = set(rows[:, 0].astype(int).tolist())
    if "statuses" in e:
        assert e["statuses"] <= statuses, (name, statuses)
    if "error" in e:
        assert res[0].get("error") == e["error"], (name, res[0].get("error"), res[0].get("message"))
    else:
        assert "error" not in res[0], (name, res[0])
    for w in e.get("warnings", []):
        assert any(w in m for m, _ in res[0]["warnings"]), (name, res[0]["warnings"])
    if "roll" in e:
        lo, hi = e["roll"]
        assert lo <= res[0]["catphan_roll"] <= hi, (name, res[0]["catphan_roll"])
    if e.get("beyond"):
        assert 110 / px > size / 2, name


def main():
    from oracle import acr_oracle, skimage_draw
    from oracle.refstub import import_reference

    import_reference()
    from pylinac.core import roi as rroi

    rroi.draw = types.SimpleNamespace(disk=skimage_draw.disk)
    rct = acr_oracle.install()
    from pylinac import acr

    store = {}
    for name in CASES:
        raw, slopes, intercepts, px, thk = case_series(name)
        hu = raw.astype(np.float64) * slopes[:, None, None] + intercepts[:, None, None]
        rct.image.DicomImageStack = fake_stack_class(hu, px, thk)
        acr.CatPhanBase = rct.CatPhanBase
        cls = acr.ACRCT
        catphan_size = np.pi * cls.catphan_radius_mm**2 / px**2
        radius = 110 / px
        rows = []
        for z in range(len(raw)):
            o = acr_oracle.localize_slice(raw[z], slopes[z], intercepts[z], catphan_size, cls.clear_borders, radius)
            rows.append([o.get(k, np.nan) for k in ROW_KEYS])
        rows = np.array(rows, dtype=np.float64)
        # the oracle's rows are the reference's own Slice.phantom_roi
        ref = cls(["unused"])
        for z in range(len(raw)):
            s = rct.Slice(ref, z, clear_borders=cls.clear_borders, original_image=ref.dicom_stack[z])
            try:
                roi = s.phantom_roi
                assert rows[z, 0] == 0 and roi.filled_area == rows[z, 3] and roi.centroid == (rows[z, 4], rows[z, 5]), (name, z)
            except ValueError:
                assert rows[z, 0] != 0, (name, z)
        res = run_reference(cls, ANALYZE[name])
        check_expectations(name, rows, res, raw.shape[1], px)
        # the region table of the first analyze()'s roll slice, and the reference's own get_regions of it
        roll_slice = res[0].get("origin_slice")
        if roll_slice is not None:
            regions, thres, max_edge, labels = acr_oracle.slice_regions(raw[roll_slice], slopes[roll_slice], intercepts[roll_slice],
                                                                        radius)
            s = rct.Slice(ref, roll_slice, clear_borders=cls.clear_borders)
            larr, ref_regions, num = rct.get_regions(s)
            assert np.array_equal(larr, labels) and num == len(regions)
            for a, b in zip(regions, ref_regions):
                assert (a.filled_area, a.bbox, a.centroid, a.eccentricity) == (b.filled_area, b.bbox, b.centroid, b.eccentricity)
            table = acr_oracle.region_rows(regions, raw.shape[2])
            store[f"{name}/regions"] = np.array(json.dumps(table))
            store[f"{name}/eccentricity"] = np.array([r.eccentricity for r in regions], dtype=np.float64)
            store[f"{name}/region_threshold"] = np.array([thres, max_edge])
        store[f"{name}/rows"] = rows
        store[f"{name}/reference"] = np.array(json.dumps(res))
        print(name, raw.dtype, raw.shape, "in view", int((rows[:, 0] == 0).sum()),
              [(r.get("origin_slice"), r.get("catphan_roll"), r.get("error"), [w[0][:30] for w in r["warnings"]]) for r in res])
    np.savez_compressed("tests/golden/acr_golden.npz", **store)


if __name__ == "__main__":
    main()
