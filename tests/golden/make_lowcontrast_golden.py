"""Generate tests/golden/lowcontrast_golden.npz: pylinac.core.roi.LowContrastDiskROI (core/roi.py:191-408), pylinac.core.contrast and
the low-contrast stage of pylinac.planar_imaging.ImagePhantomBase (planar_imaging.py:140-143, 472-504, 612-627) of the UNMODIFIED
reference (stub-imported) on the cases of lowcontrast_cases.py.  skimage is absent: ``pylinac.core.roi.draw.disk`` is the restatement
of oracle/skimage_draw.py, as for the quadrant goldens.  The batch cases call the reference's unbound ``_sample_low_contrast_background_rois``,
``_sample_low_contrast_rois`` and ``percent_integral_uniformity`` on a namespace that holds the attributes they read.  Each case is one
JSON record: values with their type name (repr round-trips float64, NaN as NaN), warnings as [category, message], exceptions as
[type, message].
Run here:  python -m tests.golden.make_lowcontrast_golden"""
from __future__ import annotations

import json
import sys
import types
import warnings

import numpy as np

from tests.golden.lowcontrast_cases import BATCH_CASES, CONTRAST_CASES, LEEDS_BG, LEEDS_LIKE, Q, ROI_CASES

PROPERTIES = ("pixel_value", "std", "signal_to_noise", "contrast_to_noise", "michelson", "weber", "rms", "ratio", "contrast",
              "cnr_constant", "visibility", "contrast_constant", "passed", "passed_visibility", "passed_contrast_constant",
              "passed_cnr_constant", "plot_color", "plot_color_constant", "plot_color_cnr")


def plain(v):
    """a JSON value of `v` with its type name"""
    if isinstance(v, dict):
        return {k: plain(x) for k, x in v.items()}
    if isinstance(v, (bool, np.bool_)):
        return [type(v).__name__, bool(v)]
    if isinstance(v, str):
        return v
    return [type(v).__name__, float(v)]


def call(fn):
    """{"value": ...} or {"error": [type, message]}, and the warnings the call raised"""
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        try:
            out = {"value": plain(fn())}
        except Exception as e:  # noqa: BLE001 -- the exception is the golden
            out = {"error": [type(e).__name__, str(e)]}
    out["warnings"] = [[w.category.__name__, str(w.message)] for w in caught]
    return out


def install():
    """the stub-imported reference's pylinac.core.roi, with skimage.draw.disk restated"""
    from oracle import skimage_draw
    from oracle.refstub import import_reference

    import_reference()
    import pylinac.core.roi as rroi

    rroi.draw = types.SimpleNamespace(disk=skimage_draw.disk)
    return rroi


def roi_record(roi) -> dict:
    rec = {name: call(lambda name=name: getattr(roi, name)) for name in PROPERTIES}
    rec["as_dict"] = call(roi.as_dict)
    rec["percentile"] = [call(lambda q=q: roi.percentile(q)) for q in Q]
    return rec


def roi_records(name, roi_module) -> list:
    """the records of the LowContrastDiskROIs of case `name` by `roi_module`'s class"""
    build, specs = ROI_CASES[name]
    arr = build()
    return [roi_record(roi_module.LowContrastDiskROI(arr, radius=r, center=roi_module.Point(cx, cy), **kw)) for cy, cx, r, kw in specs]


def contrast_records(contrast_module) -> list:
    out = []
    for fn, args in CONTRAST_CASES:
        args = [np.array(a) if isinstance(a, list) else a for a in args]
        out.append(call(lambda fn=fn, args=args: getattr(contrast_module, fn)(*args)))
    return out


def batch_record(name) -> list:
    """the reference's ImagePhantomBase low-contrast stage on each frame of batch case `name`"""
    import pylinac.planar_imaging as rpi
    from pylinac.core.geometry import Point

    build, geom, kw = BATCH_CASES[name]
    frames = build()
    percentiles = kw.get("percentiles", (1, 99))
    out = []
    for frame in frames:
        ns = types.SimpleNamespace(
            image=frame, phantom_center=Point(*geom["center"]), phantom_angle=geom["angle"], phantom_radius=geom["radius"],
            low_contrast_roi_settings=LEEDS_LIKE, low_contrast_background_roi_settings=LEEDS_BG,
            roi_size_factor=kw.get("roi_size_factor", 1), _low_contrast_threshold=kw.get("contrast_threshold"),
            _low_contrast_method=kw.get("contrast_method", "Michelson"), visibility_threshold=kw.get("visibility_threshold", 0.1))
        ns.low_contrast_background_rois, ns.low_contrast_background_value = rpi.ImagePhantomBase._sample_low_contrast_background_rois(ns)
        ns.low_contrast_rois = rpi.ImagePhantomBase._sample_low_contrast_rois(ns)
        piu = rpi.ImagePhantomBase.percent_integral_uniformity(ns, percentiles)
        rois = [{"median": r.pixel_value, "std": r.std, "contrast": float(r.contrast), "cnr": r.contrast_to_noise,
                 "snr": r.signal_to_noise, "visibility": float(r.visibility), "passed_visibility": bool(r.passed_visibility),
                 "percentiles": [r.percentile(percentiles[0]), r.percentile(percentiles[1])]} for r in ns.low_contrast_rois]
        out.append({"background": float(ns.low_contrast_background_value), "rois": rois, "piu": piu})
    return out


def main():
    rroi = install()
    import pylinac.core.contrast as rcontrast

    store = {"contrast": np.array(json.dumps(contrast_records(rcontrast), sort_keys=True))}
    for name in ROI_CASES:
        store["roi:" + name] = np.array(json.dumps(roi_records(name, rroi), sort_keys=True))
        print("roi:" + name, str(store["roi:" + name])[:200])
    warnings.simplefilter("ignore")
    for name in BATCH_CASES:
        store["batch:" + name] = np.array(json.dumps(batch_record(name), sort_keys=True))
        print("batch:" + name, str(store["batch:" + name])[:200])
    np.savez_compressed("tests/golden/lowcontrast_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
