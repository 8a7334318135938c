"""GPU: pylinac_b200.nuclear.TomographicContrast against the goldens of the unmodified reference (bit for bit, through NM files),
the device's slice rows and sphere searches against the numpy oracle on seeded volumes (the maxfun / maxiter limit paths included),
and batches against volume-by-volume calls."""
from __future__ import annotations

import json
import math
import os
import re

import numpy as np
import pytest

from oracle import tomo_contrast_oracle as O
from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from tests.golden.tomo_contrast_cases import CASES, jaszczak
from tests.nm_writer import write_nm

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "tomo_contrast_golden.npz"))


def _call(fn):
    try:
        return {"value": fn()}
    except Exception as e:  # noqa: BLE001 -- compared with the reference's exception
        return {"error": [type(e).__name__, str(e)]}


def _py(v):
    return int(v) if isinstance(v, (np.integer, int)) else float(v)


def _record(path, kwargs) -> dict:
    tc = nuclear.TomographicContrast(path)
    rec = {"slice_data_before_analyze": _call(lambda: tc.slice_data)}
    rec["slice_data_before_analyze"].pop("value", None)
    try:
        tc.analyze(**kwargs)
    except Exception as e:  # noqa: BLE001
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
    rec["search"] = [[int(r._search["nfev"]), int(r._search["nit"])] for r in tc.rois.values()]
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


@pytest.mark.parametrize("name", sorted(CASES))
def test_tomographic_contrast_matches_the_reference(name, tmp_path):
    build, pixel_size, kwargs = CASES[name]
    path = write_nm(tmp_path / "case.dcm", build(), pixel_spacing_mm=pixel_size)
    got = json.dumps(_record(path, kwargs), sort_keys=True)
    assert json.loads(got) == json.loads(str(GOLDEN[name])) or got == str(GOLDEN[name])


def _same(a, b) -> bool:
    a, b = float(a), float(b)
    return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))


def _fuzz_volumes(seed):
    rng = np.random.default_rng(seed)
    nz, h, w = int(rng.integers(10, 26)), int(rng.integers(24, 90)), int(rng.integers(24, 90))
    vols = [jaszczak(seed * 10 + k, shape=(nz, h, w), pixel_size=float(rng.choice([3.0, 4.4, 6.0])),
                     frac=float(rng.uniform(0.5, 0.95)), counts=float(rng.choice([8, 60, 300, 3000])), background=float(rng.uniform(0, 3)),
                     z_extent=(int(rng.integers(0, 3)), nz - int(rng.integers(0, 3))), sphere_gain=float(rng.uniform(0, 2.5)),
                     offset=(float(rng.uniform(-4, 4)), float(rng.uniform(-4, 4))))
            for k in range(int(rng.integers(1, 4)))]
    return np.stack(vols), float(rng.choice([3.0, 4.4, 6.0])), float(rng.choice([0.8, 0.7, 0.95, 1.1]))


def _check_slices(vols, ufov_ratio):
    rows = nat.nt_slices(nat.Context.default(), vols, vols.shape[1], 1 - ufov_ratio).reshape(len(vols), -1)
    for v, vol in enumerate(vols):
        for r, o in zip(rows[v], O.slice_rows(vol, ufov_ratio)):
            if o is None:
                assert r["status"] == nat.NT_NO_COMPONENT
                continue
            assert r["status"] == nat.NT_OK
            assert (r["longest"], r["erosion"], r["area"], r["sum"]) == (o["longest"], o["erosion"], o["area"], o["sum"])
            assert r["centroid_row"] == o["centroid_row"] and r["centroid_col"] == o["centroid_col"]
            assert _same(r["uniformity"], o["uniformity"]) and _same(r["value"], o["value"])
            if o["area"]:
                assert (r["max"], r["min"]) == (o["max"], o["min"])


@pytest.mark.parametrize("seed", range(40))
def test_slices_and_searches_match_the_oracle(seed):
    vols, pixel_size, ufov = _fuzz_volumes(seed)
    _check_slices(vols, ufov)
    res = nuclear.analyze_tomographic_contrast_batch(vols, pixel_size, ufov_ratio=ufov)
    for vol, r in zip(vols, res):
        try:
            o = O.analyze(vol, pixel_size, ufov_ratio=ufov)
        except ValueError as e:
            with pytest.raises(ValueError, match=re.escape(str(e))):
                r.raise_for_status()
            continue
        assert _same(r.uniformity_value, o["baseline"])
        for s, os_ in zip(r.searches, o["spheres"]):
            assert list(s["x"]) == list(os_["x"]) and _same(s["fun"], os_["fun"])
            assert (s["nfev"], s["nit"], s["status"], s["n_empty"]) == (os_["nfev"], os_["nit"], os_["status"], os_["n_empty"])
            assert (s["sum"], s["count"]) == (os_["sum"], os_["count"]) and (s["min"] == os_["min"] or not os_["count"])


@pytest.mark.parametrize("maxfun,maxiter", [(1, 600), (3, 600), (4, 600), (7, 600), (11, 600), (600, 1), (600, 2), (600, 5), (13, 8)])
def test_search_limits_match_the_oracle(maxfun, maxiter):
    """the _MaxFuncCallError path (during the initial simplex, a step or a shrink) and the maxiter path"""
    vol = jaszczak(77, shape=(20, 48, 48), z_extent=(1, 19))
    o = O.analyze(vol, 4.4, maxfun=maxfun, maxiter=maxiter)
    data = o["slice_data"]
    start = max(data, key=lambda k: data[k]["uniformity"])
    u, uz = data[start], int(start) - 1
    inp = np.zeros(6, nat.NT_SPHERE_IN_DTYPE)
    for k, (d, a) in enumerate(zip((38, 31.8, 25.4, 19.1, 15.9, 12.7), (-10, -70, -130, -190, 110, 50))):
        dist = math.sqrt(u["area"] / math.pi) * 0.65
        cx, cy = u["centroid_col"] + dist * math.cos(math.radians(a)), u["centroid_row"] + dist * math.sin(math.radians(a))
        inp[k] = ((cx, cy, uz), (cx - 5, cy - 5, uz - 3), (cx + 5, cy + 5, uz + 3), (d / (2 * 4.4)) ** 2, o["baseline"], 0, 0)
    got = nat.nt_spheres(nat.Context.default(), vol[None], len(vol), inp, maxfun, maxiter)
    for s, os_ in zip(got, o["spheres"]):
        assert list(s["x"]) == list(os_["x"]) and _same(s["fun"], os_["fun"])
        assert (s["nfev"], s["nit"], s["status"]) == (os_["nfev"], os_["nit"], os_["status"])


def test_slices_beyond_shared_memory():
    vols = np.stack([jaszczak(90 + k, shape=(6, 200, 190), z_extent=(1, 5), counts=50) for k in range(2)])
    _check_slices(vols, 0.8)


def test_batch_equals_volume_by_volume_and_device_input():
    vols = np.stack([jaszczak(60 + k, counts=[300, 40, 300][k]) for k in range(3)])
    vols[1] = 0
    res = nuclear.analyze_tomographic_contrast_batch(vols, 4.4)
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        res[1].raise_for_status()
    for k in range(len(vols)):
        one = nuclear.analyze_tomographic_contrast_batch(vols[k], 4.4)[0]
        assert res[k].slice_rows.tobytes() == one.slice_rows.tobytes()
        assert res[k].searches.tobytes() == one.searches.tobytes()
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, vols.reshape(-1, *vols.shape[2:])) as b:
        dev = nuclear.analyze_tomographic_contrast_batch(b, 4.4, slices_per_volume=vols.shape[1])
    for a, d in zip(res, dev):
        assert a.slice_rows.tobytes() == d.slice_rows.tobytes() and a.searches.tobytes() == d.searches.tobytes()
    with pytest.raises(NotImplementedError, match="float32"):
        nuclear.analyze_tomographic_contrast_batch(vols.astype(np.float32), 4.4)
