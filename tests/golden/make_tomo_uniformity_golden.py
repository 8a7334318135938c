"""Generate tests/golden/tomo_uniformity_golden.npz: pylinac.nuclear.TomographicUniformity of the UNMODIFIED reference
(nuclear.py:1370-1551 on top of PlanarUniformity, nuclear.py:274-500, stub-imported) on the volumes of tomo_uniformity_cases.py, read
through the fake NM file of make_nuclear_golden.py and with the skimage calls restated in oracle/skimage_nuclear.py.  Its
block_reduce is a reshape / transpose whose view has the strides of skimage's view_as_blocks, so numpy sums each block in the same
order (row by row, each row a pairwise sum); that restatement is unpinned (DESIGN.md section 8.5).  Each case is one JSON record:
scalars exactly (repr round-trips float64), arrays as sha256 digests, the captured warnings as [category, message] after analyze()
and after results(), exceptions as [type, message].  Run here:  python -m tests.golden.make_tomo_uniformity_golden"""
from __future__ import annotations

import json
import sys
import warnings

import numpy as np

from tests.golden.make_nuclear_golden import _call, reference_files
from tests.golden.nuclear_cases import digest
from tests.golden.tomo_uniformity_cases import CASES


def _py(v):
    """JSON-ready scalars: numpy integers as int, numpy floats as float"""
    if isinstance(v, (np.integer, int)):
        return int(v)
    return float(v)


def _captured(obj):
    return [[w["category"], w["message"]] for w in obj._captured_warnings]


def fov_record(fov) -> dict:
    rec = {}
    for name in ("integral_uniformity", "differential_uniformity", "max_point", "min_point"):
        v = _call(lambda name=name: getattr(fov, name))
        if "value" in v:
            v["value"] = [int(x) for x in v["value"]] if isinstance(v["value"], tuple) else _py(v["value"])
        rec[name] = v
    du = _call(lambda: fov._differential_uniformities)
    if "value" in du:
        y, x = du["value"]
        rec["du_axes"] = [[len(d), _py(max(d.values())) if d else None, [int(c) for c in max(d, key=d.get)] if d else None]
                          for d in (y, x)]
    rec["fov"] = digest(fov.fov)
    return rec


def record(rn, name) -> dict:
    build, pixel_size, kwargs, calls = CASES[name]
    volume = build()
    with reference_files(volume, pixel_size):
        tu = rn.TomographicUniformity("case.dcm")
    rec = {}
    for _ in range(calls):
        try:
            tu.analyze(**kwargs)
        except Exception as e:  # noqa: BLE001 -- the exception is the golden
            rec["analyze_error"] = [type(e).__name__, str(e)]
    rec["warnings"] = _captured(tu)
    if "analyze_error" in rec:
        return rec
    rec["first_frame"], rec["last_frame"], rec["frame_key"] = tu.first_frame, tu.last_frame, tu.frame_key
    rec["frame_keys"] = list(tu.frame_results)
    rec["center_ratio"] = _py(tu.center_ratio)
    rec["mean_frame"] = digest(tu.stack.frames[0].array)
    tu._captured_warnings.clear()
    rec["results"] = _call(tu.results)
    data = _call(lambda: tu.results_data(as_dict=True))
    if "value" in data:
        for k in ("pylinac_version", "date_of_analysis", "warnings"):
            data["value"].pop(k)
    rec["results_dict"] = data
    rec["results_warnings"] = _captured(tu)
    r = tu.frame_result
    rec["binned_frame"] = digest(r["binned_frame"])
    rec["fovs"] = {k: fov_record(r[k]) for k in ("ufov", "cfov", "center_fov")}
    return rec


def main():
    from oracle import skimage_nuclear

    rn = skimage_nuclear.install()
    warnings.simplefilter("ignore")
    store = {}
    for name in CASES:
        store[name] = np.array(json.dumps(record(rn, name), sort_keys=True))
        print(name, str(store[name])[:300])
    np.savez_compressed("tests/golden/tomo_uniformity_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
