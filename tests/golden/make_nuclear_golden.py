"""Generate tests/golden/nuclear_golden.npz: pylinac.nuclear.PlanarUniformity and MaxCountRate of the UNMODIFIED reference
(nuclear.py:39-500, stub-imported) on the frames of nuclear_cases.py.  pydicom is absent and NMImageStack opens the path once per
frame (core/image.py:2216-2249), so ``pylinac.core.image.pydicom.dcmread`` is replaced by a fake that serves the case's frames and
``pylinac.core.image.DicomImage`` by a header-only stand-in; the skimage calls are the restatements of oracle/skimage_nuclear.py.
Each case is stored as one JSON record: scalars exactly (repr round-trips float64), large arrays as sha256 digests, exceptions as
[type, message].  Run here:  python -m tests.golden.make_nuclear_golden"""
from __future__ import annotations

import contextlib
import json
import sys
import types
import warnings

import numpy as np

from tests.golden.nuclear_cases import CASES, COUNT_CASES, digest

FOV_PROPERTIES = ("integral_uniformity", "differential_uniformity", "max_point", "min_point")


def _call(fn):
    try:
        v = fn()
    except Exception as e:  # noqa: BLE001 -- the exception is the golden
        return {"error": [type(e).__name__, str(e)]}
    return {"value": v}


@contextlib.contextmanager
def reference_files(frames, pixel_size, modality="NM"):
    """the reference's pylinac.core.image reads `frames` (and its pixel size) from any path while the block runs"""
    import pylinac.core.image as rimage

    ds = types.SimpleNamespace(Modality=modality, NumberOfFrames=len(frames), pixel_array=frames[0] if len(frames) == 1 else frames,
                               PixelSpacing=[pixel_size, pixel_size])

    class HeaderOnlyDicomImage:
        def __init__(self, path, *a, **k):
            self.path = path
            self.metadata = ds

    old = rimage.pydicom, rimage.DicomImage
    rimage.pydicom = types.SimpleNamespace(dcmread=lambda path, force=False, stop_before_pixels=False: ds)
    rimage.DicomImage = HeaderOnlyDicomImage
    try:
        yield
    finally:
        rimage.pydicom, rimage.DicomImage = old


def fov_record(fov) -> dict:
    rec = {name: _call(lambda name=name: getattr(fov, name)) for name in FOV_PROPERTIES}
    for k in ("max_point", "min_point"):
        if "value" in rec[k]:
            rec[k]["value"] = list(rec[k]["value"])
    du = _call(lambda: fov._differential_uniformities)
    if "value" in du:
        y, x = du["value"]
        rec["du_axes"] = [[len(d), max(d.values()) if d else None, list(max(d, key=d.get)) if d else None] for d in (y, x)]
    rec["fov"] = digest(fov.fov)
    rec["boundary_x"] = digest(fov.boundary_x)
    rec["boundary_y"] = digest(fov.boundary_y)
    return rec


def planar_record(rn, name) -> dict:
    build, pixel_size, kwargs, modality = CASES[name]
    frames = build()
    rec = {}
    with reference_files(frames, pixel_size, modality):
        try:
            pu = rn.PlanarUniformity("case.dcm")
        except Exception as e:  # noqa: BLE001
            rec["init_error"] = [type(e).__name__, str(e)]
            return rec
    try:
        pu.analyze(**kwargs)
    except Exception as e:  # noqa: BLE001
        rec["analyze_error"] = [type(e).__name__, str(e)]
        return rec
    rec["frames"] = {}
    for key, r in pu.frame_results.items():
        rec["frames"][key] = {"binned_frame": digest(r["binned_frame"]), "ufov": fov_record(r["ufov"]), "cfov": fov_record(r["cfov"])}
    rec["results"] = _call(pu.results)
    rec["results_dict"] = _call(lambda: pu.results_data(as_dict=True))
    rec["results_json"] = _call(lambda: pu.results_data(as_json=True))
    return rec


def count_record(rn, name) -> dict:
    build, duration = COUNT_CASES[name]
    frames = build()
    with reference_files(frames, 1.0):
        mcr = rn.MaxCountRate("case.dcm")
    mcr.analyze(frame_duration=duration)
    return {"sums": [mcr.sums[k] for k in sorted(mcr.sums)], "max_countrate": mcr.max_countrate, "max_frame": mcr.max_frame,
            "max_time": mcr.max_time, "results": mcr.results()}


def main():
    from oracle import skimage_nuclear

    rn = skimage_nuclear.install()
    warnings.simplefilter("ignore")
    store = {}
    for name in CASES:
        store[name] = np.array(json.dumps(planar_record(rn, name), sort_keys=True))
        print(name, str(store[name])[:160])
    for name in COUNT_CASES:
        store["count:" + name] = np.array(json.dumps(count_record(rn, name), sort_keys=True))
        print(name, str(store["count:" + name])[:160])
    np.savez_compressed("tests/golden/nuclear_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
