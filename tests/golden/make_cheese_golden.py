"""Generate tests/golden/cheese_golden.npz: the UNMODIFIED reference ``pylinac.cheese.TomoCheese`` / ``CIRS062M`` (stub-imported;
skimage served by oracle/skimage_ct.py, skimage.draw by oracle/skimage_draw.py) on the seeded series of cheese_cases.py, and the
per-slice localization of oracle/ct_oracle.py, checked against the reference's own Slice.phantom_roi.

pydicom is not installed here, so the series reaches the reference through a fake ``DicomImageStack`` holding each slice's HU array
(raw * slope + intercept in float64, as pydicom's apply_rescale gives it) and the SliceThickness / PixelSpacing tags.

Run here (the container that has /root/reference):  python -m tests.golden.make_cheese_golden
"""
from __future__ import annotations

import contextlib
import io
import json
import types
import warnings

import numpy as np

from tests.golden.cheese_cases import ANALYZE, CASES, EXPECT, case_series

ROW_KEYS = ("status", "n_regions", "label", "area", "centroid_row", "centroid_col", "max_edge", "threshold")


def fake_stack_class(hu, px, thk):
    from pylinac.core import image as rimage

    class FakeStack:
        def __init__(self, folder, check_uid=True, min_number=39, **kwargs):
            self.images = [rimage.ArrayImage(a) for a in hu]
            self.metadata = types.SimpleNamespace(SliceThickness=thk, PixelSpacing=[px, px])
            self.slice_spacing = thk

        def __getitem__(self, i):
            return self.images[i]

        def __len__(self):
            return len(self.images)

        def __iter__(self):
            return iter(self.images)

    return FakeStack


def unclipped_threshold(raw, slope, intercept):
    """threshold_otsu of the smoothed edges when the slice is not clipped (what clip_in_localization changes)"""
    from oracle import skimage_ct

    hu = raw.astype(np.float64) * float(slope) + float(intercept)
    return float(skimage_ct.threshold_otsu(skimage_ct.gaussian(skimage_ct.scharr(hu), sigma=1)))


def check_expectations(name, rows, res, raw=None, slopes=None, intercepts=None):
    """assert that case `name` reaches the paths EXPECT names (rows: the golden rows; res: the reference's analyze() records)"""
    e = EXPECT[name]
    statuses = set(rows[:, 0].astype(int).tolist())
    if "statuses" in e:
        assert e["statuses"] <= statuses, (name, statuses)
        if e.get("only"):
            assert statuses == e["statuses"], (name, statuses)
    if e.get("small_edges"):
        assert ((rows[:, 0] == 1) & (rows[:, 6] > 0)).any() and ((rows[:, 0] == 1) & (rows[:, 6] == 0)).any(), name
    if "error" in e:
        assert res[0].get("error") == e["error"], (name, res[0].get("error"))
    else:
        assert "error" not in res[0], (name, res[0])
    if "stdout" in e:
        assert e["stdout"] in res[0]["stdout"], (name, res[0]["stdout"])
    if "roll" in e:
        lo, hi = e["roll"]
        assert lo <= res[0]["catphan_roll"] <= hi, (name, res[0]["catphan_roll"])
    if e.get("clipped") and raw is not None:
        ok = np.flatnonzero(rows[:, 0] == 0)
        changed = [z for z in ok if unclipped_threshold(raw[z], slopes[z], intercepts[z]) != rows[z, 7]]
        assert changed, name


def run_reference(cls, kwargs_list):
    """-> list (per analyze call) of dict: results, or error type / message; plus captured stdout"""
    out = []
    phantom = cls(["unused"])
    for kw in kwargs_list + kwargs_list[:1]:
        buf = io.StringIO()
        rec = {"kwargs": kw}
        try:
            with contextlib.redirect_stdout(buf):
                phantom.analyze(**kw)
                rd = phantom.results_data(as_dict=True)
            rec.update(origin_slice=phantom.origin_slice, catphan_roll=float(phantom.catphan_roll), results=phantom.results(),
                       results_list=phantom.results(as_list=True), results_data=rd,
                       rois={k: r.as_dict() for k, r in phantom.module.rois.items()})
        except Exception as e:  # noqa: BLE001 -- the reference's exception is part of the golden
            rec.update(error=type(e).__name__, message=str(e))
        rec["stdout"] = buf.getvalue()
        out.append(rec)
    return out


def main():
    from oracle import ct_oracle, skimage_ct, skimage_draw
    from oracle.refstub import import_reference

    import_reference()
    from pylinac.core import roi as rroi

    rroi.draw = types.SimpleNamespace(disk=skimage_draw.disk)
    rct = skimage_ct.install()
    from pylinac import cheese

    warnings.simplefilter("ignore")
    store = {}
    for name, c in CASES.items():
        raw, slopes, intercepts, px, thk = case_series(name)
        hu = raw.astype(np.float64) * slopes[:, None, None] + intercepts[:, None, None]
        cls = getattr(cheese, c["phantom"])
        rct.image.DicomImageStack = fake_stack_class(hu, px, thk)
        catphan_size = np.pi * cls.catphan_radius_mm**2 / px**2
        rows = []
        for z in range(len(raw)):
            o = ct_oracle.localize_slice(raw[z], slopes[z], intercepts[z], catphan_size, cls.clear_borders)
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
        check_expectations(name, rows, res, raw, slopes, intercepts)
        store[f"{name}/rows"] = rows
        store[f"{name}/reference"] = np.array(json.dumps(res))
        print(name, raw.dtype, raw.shape, "in view", int((rows[:, 0] == 0).sum()),
              [(r.get("origin_slice"), r.get("catphan_roll"), r.get("error"), r["stdout"].strip()[:40]) for r in res])
    np.savez_compressed("tests/golden/cheese_golden.npz", **store)


if __name__ == "__main__":
    main()
