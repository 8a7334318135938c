"""GPU: pylinac_b200.nuclear.TomographicUniformity against the goldens of the unmodified reference (bit for bit, through NM files),
epid_tu_stages against the numpy oracle stage by stage on seeded batches (bins 1-8, frames beyond shared memory included), and
batches against volume-by-volume calls and device Batches."""
from __future__ import annotations

import json
import math
import os

import numpy as np
import pytest

from oracle import tomo_uniformity_oracle as O
from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from tests.golden.nuclear_cases import digest
from tests.golden.tomo_contrast_cases import jaszczak
from tests.golden.tomo_uniformity_cases import CASES
from tests.nm_writer import write_nm

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "tomo_uniformity_golden.npz"))


def _call(fn):
    try:
        return {"value": fn()}
    except Exception as e:  # noqa: BLE001 -- compared with the reference's exception
        return {"error": [type(e).__name__, str(e)]}


def _py(v):
    return int(v) if isinstance(v, (np.integer, int)) else float(v)


def _captured(obj):
    return [[w["category"], w["message"]] for w in obj._captured_warnings]


def _fov_record(fov) -> dict:
    rec = {}
    for name in ("integral_uniformity", "differential_uniformity", "max_point", "min_point"):
        v = _call(lambda name=name: getattr(fov, name))
        if "value" in v:
            v["value"] = [int(x) for x in v["value"]] if isinstance(v["value"], tuple) else _py(v["value"])
        rec[name] = v
    rec["fov"] = digest(fov.fov)
    return rec


def _record(path, kwargs, calls) -> dict:
    tu = nuclear.TomographicUniformity(path)
    rec = {}
    for _ in range(calls):
        try:
            tu.analyze(**kwargs)
        except Exception as e:  # noqa: BLE001
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
    rec["fovs"] = {k: _fov_record(r[k]) for k in ("ufov", "cfov", "center_fov")}
    return rec


def _same(a, b):
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or a == b
    if isinstance(a, dict) and isinstance(b, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_cases(tmp_path, name):
    build, pixel_size, kwargs, calls = CASES[name]
    want = json.loads(str(GOLDEN[name]))
    for f in want.get("fovs", {}).values():
        f.pop("du_axes", None)
    path = write_nm(tmp_path / "case.dcm", build(), pixel_spacing_mm=pixel_size)
    got = json.loads(json.dumps(_record(str(path), kwargs, calls)))
    assert _same(got, want), {k: (got.get(k), want.get(k)) for k in set(got) | set(want) if not _same(got.get(k), want.get(k))}


def _volume(rng, shape, counts):
    return jaszczak(int(rng.integers(1 << 30)), shape=shape, z_extent=(1, shape[0] - 1), counts=counts, frac=float(rng.uniform(0.5, 0.95)))


def _check_stages(out, vols, pixel_size, first, last, kw):
    for v, vol in enumerate(vols):
        o = O.analyze(vol, pixel_size, first, last, **kw)
        r = out["results"][v]
        for k in ("mean", "binned", "filtered", "cleaned"):
            assert np.array_equal(out[k][v], o[k]), k
        assert _same(float(r["threshold"]), float(o["threshold"]))
        if o["status"] != "ok":
            assert r["status"] == nat.NM_NO_COMPONENT
            continue
        assert r["status"] == nat.NM_OK
        assert np.array_equal(out["edt2"][v], o["edt2"])
        for k, name in enumerate(("ufov", "cfov", "center_fov")):
            f = o[name]
            assert np.array_equal(out["masks"][v, k].astype(bool), f["mask"]), name
            assert r["longest"] == f["longest"] and r["erosion"][k] == f["erosion"]
            assert r["n_fov"][k] == f["n_fov"]
            if f["iu"] is not None:
                wb = out["cleaned"].shape[-1]
                assert r["iu"][k] == f["iu"]
                assert divmod(int(r["max_index"][k]), wb) == f["max_point"] and divmod(int(r["min_index"][k]), wb) == f["min_point"]
            for a in (0, 1):
                assert r["du_count"][2 * k + a] == f[f"du_count_{a}"]
                if f[f"du_{a}"] is not None:
                    wb = out["cleaned"].shape[-1]
                    assert r["du_max"][2 * k + a] == f[f"du_{a}"][0]
                    assert divmod(int(r["du_index"][2 * k + a]), wb) == f[f"du_{a}"][1]
        assert (float(r["center_sum"]), int(r["center_count"])) == o["center"]
        assert (float(r["ring_sum"]), int(r["ring_count"])) == o["ring"]


@pytest.mark.parametrize("seed", range(60))
def test_stages_match_the_oracle(seed):
    rng = np.random.default_rng(1000 + seed)
    b = int(rng.choice([1, 2, 4, 8]))
    if seed % 10 == 9:                                        # 16 bytes a binned pixel beyond shared memory
        h, w = int(rng.integers(120, 140)), int(rng.integers(120, 140))
        b = 1
    else:
        h, w = int(rng.integers(8, 50)) * b + int(rng.integers(0, b)), int(rng.integers(8, 50)) * b + int(rng.integers(0, b))
    nz = int(rng.integers(4, 30))
    count = int(rng.choice([1, 2, 3, 7, 8, 16, 25, nz - 1]))
    count = max(1, min(count, nz - 1))
    first = int(rng.integers(0, nz - count))
    counts = float(rng.choice([5.0, 60.0, 300.0]))
    nvol = int(rng.integers(1, 4))
    vols = np.stack([_volume(rng, (nz, h, w), counts) for _ in range(nvol)])
    if seed % 7 == 3:
        vols[0, :, h // 2, w // 3] = 20000                   # a hot spot
    kw = {"ufov_ratio": float(rng.choice([0.8, 0.95, 0.6])), "cfov_ratio": float(rng.choice([0.75, 0.5, 1.0])),
          "center_ratio": float(rng.choice([0.4, 0.2, 0.0])), "threshold": float(rng.choice([0.75, 0.5, 0.9])),
          "window_size": int(rng.choice([3, 5, 7]))}
    pixel_size = 6.0 / b
    erode = (1 - kw["ufov_ratio"], 1 - kw["cfov_ratio"] * kw["ufov_ratio"], 1 - kw["center_ratio"] * kw["ufov_ratio"])
    out = nat.tu_stages(nat.Context.default(), vols, nz, first, count, b, erode, kw["window_size"], kw["threshold"])
    _check_stages(out, vols, pixel_size, first, first + count, kw)


def test_batch_matches_volume_by_volume_and_device_batches():
    rng = np.random.default_rng(5)
    vols = np.stack([_volume(rng, (20, 64, 64), 200.0) for _ in range(5)])
    res = nuclear.analyze_tomographic_uniformity_batch(vols, 4.4, first_frame=2, last_frame=17)
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, vols.reshape(-1, 64, 64)) as b:
        dev = nuclear.analyze_tomographic_uniformity_batch(b, 4.4, first_frame=2, last_frame=17, slices_per_volume=20)
    for v in range(len(vols)):
        one = nuclear.analyze_tomographic_uniformity_batch(vols[v], 4.4, first_frame=2, last_frame=17)[0]
        for other in (res[v], dev[v]):
            assert other.row.tobytes() == one.row.tobytes()
            assert np.array_equal(other.binned_frame, one.binned_frame) and np.array_equal(other.mean_frame, one.mean_frame)
            for k in ("ufov", "cfov", "center_fov"):
                assert np.array_equal(getattr(other, k).fov, getattr(one, k).fov, equal_nan=True)
        assert res[v].center_border_ratio == one.center_border_ratio


def test_uint8_is_widened_and_other_dtypes_raise():
    v8 = jaszczak(3, counts=60, dtype=np.uint8)
    a = nuclear.analyze_tomographic_uniformity_batch(v8, 4.4)[0]
    b = nuclear.analyze_tomographic_uniformity_batch(v8.astype(np.uint16), 4.4)[0]
    assert a.row.tobytes() == b.row.tobytes()
    for dt in (np.float32, np.int16, np.float64):
        with pytest.raises(NotImplementedError, match=np.dtype(dt).name):
            nuclear.analyze_tomographic_uniformity_batch(v8.astype(dt), 4.4)


def test_center_border_ratio_with_other_arguments(tmp_path):
    """called again with another center size, it analyses the same slab with that center FOV"""
    vol = jaszczak(4)
    path = write_nm(tmp_path / "v.dcm", vol, pixel_spacing_mm=4.4)
    tu = nuclear.TomographicUniformity(str(path))
    tu.analyze()
    o = O.analyze(vol, 4.4, 0, 31)
    c = o["cleaned"]
    center = O.nm.fov(c, 0.5)["mask"] & (c > 0)
    ring = o["ufov"]["mask"] & (c > 0) & ~o["cfov"]["mask"]
    cs, cn = O.nanmean_zero_outside(c, center)
    rs, rn = O.nanmean_zero_outside(c, ring)
    assert tu.center_border_ratio(0.5, 5) == (np.float64(cs) / cn) / (np.float64(rs) / rn)
    assert np.array_equal(tu.frame_result["center_fov"].mask, O.nm.fov(c, 0.5)["mask"])
