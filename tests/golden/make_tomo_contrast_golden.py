"""Generate tests/golden/tomo_contrast_golden.npz: pylinac.nuclear.TomographicContrast of the UNMODIFIED reference
(nuclear.py:1553-1856, stub-imported) on the volumes of tomo_contrast_cases.py, read through the fake NM file of make_nuclear_golden.py
and with the skimage calls restated in oracle/skimage_nuclear.py and oracle/skimage_tomo.py.  ``minimize`` is wrapped, unchanged, to record each sphere's
nfev / nit.  Each case is one JSON record: scalars exactly (repr round-trips float64), the analyze() warnings in order as
[category, message], exceptions as [type, message].  Run here:  python -m tests.golden.make_tomo_contrast_golden"""
from __future__ import annotations

import json
import sys

import numpy as np

from tests.golden.make_nuclear_golden import _call, reference_files
from tests.golden.tomo_contrast_cases import CASES


def _py(v):
    """JSON-ready scalars: numpy integers as int, numpy floats as float"""
    if isinstance(v, (np.integer, int)):
        return int(v)
    return float(v)


def record(rn, name, searches) -> dict:
    build, pixel_size, kwargs = CASES[name]
    volume = build()
    with reference_files(volume, pixel_size):
        tc = rn.TomographicContrast("case.dcm")
    rec = {"slice_data_before_analyze": _call(lambda: tc.slice_data)}
    rec["slice_data_before_analyze"].pop("value", None)
    searches.clear()
    try:
        tc.analyze(**kwargs)
    except Exception as e:  # noqa: BLE001 -- the exception is the golden
        rec["analyze_error"] = [type(e).__name__, str(e)]
    rec["warnings"] = [[w["category"], w["message"]] for w in tc._captured_warnings]
    if "slice_data" in tc.__dict__:
        rec["slice_data"] = {k: {"fov diameter": _py(v["fov diameter"]), "center": [_py(v["center"].x), _py(v["center"].y)],
                                 "area": _py(v["area"]), "uniformity": _py(v["uniformity"]), "value": _py(v["value"])}
                             for k, v in tc.slice_data.items()}
    if "analyze_error" in rec:
        return rec
    rec["uniformity_frame"] = tc.uniformity_frame
    rec["uniformity_value"] = _py(tc.uniformity_value)
    rec["search"] = [[int(r.nfev), int(r.nit)] for r in searches]
    rec["rois"] = {k: {"x": _py(r.x), "y": _py(r.y), "z": _py(r.z), "radius": _py(r.radius), "mean": _py(r.mean_value),
                       "min": _py(r.min_value), "mean_contrast": _py(r.mean_contrast), "max_contrast": _py(r.max_contrast)}
                   for k, r in tc.rois.items()}
    tc._captured_warnings.clear()
    rec["results"] = _call(tc.results)
    data = _call(lambda: tc.results_data(as_dict=True))
    if "value" in data:
        for k in ("pylinac_version", "date_of_analysis", "warnings"):
            data["value"].pop(k)
    rec["results_dict"] = data
    rec["results_warnings"] = [[w["category"], w["message"]] for w in tc._captured_warnings]
    return rec


def main():
    from oracle import skimage_tomo

    rn = skimage_tomo.install()
    real_minimize = rn.minimize
    searches = []

    def recording_minimize(*args, **kwargs):
        res = real_minimize(*args, **kwargs)
        searches.append(res)
        return res

    rn.minimize = recording_minimize
    store = {}
    for name in CASES:
        store[name] = np.array(json.dumps(record(rn, name, searches), sort_keys=True))
        print(name, str(store[name])[:200])
    np.savez_compressed("tests/golden/tomo_contrast_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
