"""Generate tests/golden/quadrant_golden.npz: pylinac.nuclear.QuadrantResolution (nuclear.py:1248-1367) and pylinac.core.roi.DiskROI
(core/roi.py:39-190) of the UNMODIFIED reference (stub-imported) on the cases of quadrant_cases.py.  Each case's frames are written to
an NM file by tests/nm_writer.py; pydicom is absent, so ``pylinac.core.image.pydicom.dcmread`` reads that file with this package's
host DICOM parser, and ``pylinac.core.image.DicomImage`` is a stand-in that holds the frame and indexes it as BaseImage.__getitem__
does.  skimage is absent too: ``pylinac.core.roi.draw.disk`` is the restatement of oracle/skimage_draw.py, as for the gamma goldens.
masked_array() is not recorded: it calls disk(shape=...), which the restatement leaves out.  Each case is one JSON record: scalars exactly (repr round-trips float64, NaN as NaN), pixel arrays as sha256 digests, the captured
warnings as [category, message] after analyze() and after results(), exceptions as [type, message].
Run here:  python -m tests.golden.make_quadrant_golden"""
from __future__ import annotations

import contextlib
import json
import sys
import tempfile
import types
import warnings
from pathlib import Path

import numpy as np

from tests.golden.make_nuclear_golden import _call
from tests.golden.nuclear_cases import digest
from tests.golden.quadrant_cases import CASES, DISK_CASES
from tests.nm_writer import write_nm

ROI_STATS = ("mean", "std", "pixel_value", "min", "max")


@contextlib.contextmanager
def reference_nm_files():
    """the reference's pylinac.core.image reads NM files through pylinac_b200.dicom while the block runs"""
    import pylinac.core.image as rimage

    from pylinac_b200 import dicom

    def dcmread(path, force=False, stop_before_pixels=False):
        ds = dicom.read_header(path)
        if not stop_before_pixels:
            frames, _ = dicom.read_nm_frames([path])
            ds.pixel_array = frames[0] if len(frames) == 1 else frames
        return ds

    class FrameImage:
        def __init__(self, path, *a, **k):
            self.path = path

        def __getitem__(self, item):
            return self.array[item]

    old = rimage.pydicom, rimage.DicomImage
    rimage.pydicom = types.SimpleNamespace(dcmread=dcmread)
    rimage.DicomImage = FrameImage
    try:
        yield
    finally:
        rimage.pydicom, rimage.DicomImage = old


def install():
    """the stub-imported reference's pylinac.nuclear, with skimage.draw.disk restated in pylinac.core.roi"""
    from oracle import skimage_draw, skimage_nuclear

    rn = skimage_nuclear.install()
    import pylinac.core.roi as rroi

    rroi.draw = types.SimpleNamespace(disk=skimage_draw.disk)
    return rn


def _captured(obj):
    return [[w["category"], w["message"]] for w in obj._captured_warnings]


def roi_record(roi) -> dict:
    rec = {"center": [float(roi.center.x), float(roi.center.y)], "radius": float(roi.radius)}
    mask = _call(roi.circle_mask)
    if "error" in mask:
        rec["circle_mask"] = mask
        return rec
    rec["count"] = int(mask["value"].size)
    rec["circle_mask"] = digest(mask["value"])
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        for name in ROI_STATS:
            v = _call(lambda name=name: getattr(roi, name))
            rec[name] = {"value": float(v["value"])} if "value" in v else v
    rec["stat_warnings"] = [[w.category.__name__, str(w.message)] for w in caught]
    return rec


def record(nuclear, name, tmp: Path, opener=reference_nm_files) -> dict:
    """the record of case `name` by `nuclear`'s QuadrantResolution (the reference's, opened by `opener`, or this package's)"""
    build, kwargs = CASES[name]
    path = write_nm(tmp / f"{name}.dcm", build())
    with opener():
        q = nuclear.QuadrantResolution(path)
    rec = {}
    try:
        q.analyze(**kwargs)
    except Exception as e:  # noqa: BLE001 -- the exception is the golden
        rec["analyze_error"] = [type(e).__name__, str(e)]
    rec["warnings"] = _captured(q)
    if hasattr(q, "rois"):
        rec["rois"] = [[float(k), roi_record(r)] for k, r in q.rois.items()]
    if "analyze_error" in rec:
        return rec
    rec["mtfs"] = [[float(k), float(v)] for k, v in q.mtf.mtfs.items()]
    rec["fwhms"] = [[float(k), float(v)] for k, v in q.mtf.fwhms.items()]
    rec["reprs"] = [_call(lambda r=r: repr(r)) for r in q.rois.values()]
    q._captured_warnings.clear()
    rec["results"] = _call(q.results)
    data = _call(lambda: q.results_data(as_dict=True))
    if "value" in data:
        for k in ("pylinac_version", "date_of_analysis", "warnings"):
            data["value"].pop(k)
    rec["results_dict"] = data
    rec["results_warnings"] = _captured(q)
    return rec


def disk_record(name, roi_module=None) -> list:
    """the records of the DiskROIs of case `name` by `roi_module`'s DiskROI (default: the reference's)"""
    if roi_module is None:
        import pylinac.core.roi as roi_module
    DiskROI, Point = roi_module.DiskROI, roi_module.Point
    build, disks = DISK_CASES[name]
    arr = build()
    out = []
    for cy, cx, r in disks:
        roi = DiskROI(arr, radius=r, center=Point(cx, cy))
        rec = roi_record(roi)
        rec["as_dict"] = _call(roi.as_dict)
        out.append(rec)
    return out


def main():
    rn = install()
    warnings.simplefilter("ignore")
    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in CASES:
            store[name] = np.array(json.dumps(record(rn, name, Path(tmp)), sort_keys=True))
            print(name, str(store[name])[:300])
    for name in DISK_CASES:
        store["disk:" + name] = np.array(json.dumps(disk_record(name), sort_keys=True))
        print("disk:" + name, str(store["disk:" + name])[:200])
    np.savez_compressed("tests/golden/quadrant_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
