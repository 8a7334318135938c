"""GPU: pylinac_b200.nuclear against the goldens of the unmodified reference (bit for bit) and, stage by stage, against the numpy
oracle on seeded floods, including binned frames too large for the shared-memory path."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest

from oracle import nuclear_oracle as orc
from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from tests.golden.nuclear_cases import CASES, COUNT_CASES, digest, flood
from tests.nm_writer import write_nm

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "nuclear_golden.npz"))
FOV_PROPERTIES = ("integral_uniformity", "differential_uniformity", "max_point", "min_point")


def _call(fn):
    try:
        v = fn()
    except Exception as e:  # noqa: BLE001 -- compared with the reference's exception
        return {"error": [type(e).__name__, str(e)]}
    return {"value": list(v) if isinstance(v, tuple) else v}


def _fov_record(fov) -> dict:
    rec = {name: _call(lambda name=name: getattr(fov, name)) for name in FOV_PROPERTIES}
    axes = []
    for axis in (0, 1):
        try:
            v, pos = fov._axis_max(axis)
            axes.append([int(fov._row["du_count"][2 * fov._k + axis]), v, list(pos)])
        except ValueError as e:
            if str(e) != nuclear._EMPTY_MAX:
                break
            axes.append([0, None, None])
    if len(axes) == 2:
        rec["du_axes"] = axes
    rec["fov"] = digest(fov.fov)
    rec["boundary_x"] = digest(fov.boundary_x)
    rec["boundary_y"] = digest(fov.boundary_y)
    return rec


def _planar_record(path, kwargs) -> dict:
    rec = {}
    try:
        pu = nuclear.PlanarUniformity(path)
    except Exception as e:  # noqa: BLE001
        return {"init_error": [type(e).__name__, str(e)]}
    try:
        pu.analyze(**kwargs)
    except Exception as e:  # noqa: BLE001
        return {"analyze_error": [type(e).__name__, str(e)]}
    rec["frames"] = {key: {"binned_frame": digest(r["binned_frame"]), "ufov": _fov_record(r["ufov"]), "cfov": _fov_record(r["cfov"])}
                     for key, r in pu.frame_results.items()}
    rec["results"] = _call(pu.results)
    rec["results_dict"] = _call(lambda: pu.results_data(as_dict=True))
    rec["results_json"] = _call(lambda: pu.results_data(as_json=True))
    return rec


@pytest.mark.parametrize("name", sorted(CASES))
def test_planar_uniformity_matches_the_reference(name, tmp_path):
    build, pixel_size, kwargs, modality = CASES[name]
    path = write_nm(tmp_path / "flood.dcm", build(), pixel_spacing_mm=pixel_size, modality=modality)
    got = json.loads(json.dumps(_planar_record(path, kwargs), sort_keys=True))
    assert got == json.loads(str(GOLDEN[name]))


@pytest.mark.parametrize("name", sorted(COUNT_CASES))
def test_max_count_rate_matches_the_reference(name, tmp_path):
    build, duration = COUNT_CASES[name]
    mcr = nuclear.MaxCountRate(write_nm(tmp_path / "dynamic.dcm", build()))
    mcr.analyze(frame_duration=duration)
    want = json.loads(str(GOLDEN["count:" + name]))
    assert [mcr.sums[k] for k in sorted(mcr.sums)] == want["sums"]
    assert (mcr.max_countrate, mcr.max_frame, mcr.max_time, mcr.results()) == (want["max_countrate"], want["max_frame"],
                                                                             want["max_time"], want["results"])
    data = mcr.results_data(as_dict=True)
    assert data["max_frame"] == want["max_frame"] and data["max_countrate"] == want["max_countrate"]


def _fuzz_frames(seed):
    """a few frames of one shape: circles, rectangles, spots, gradients, stray pixels and blobs at varied count levels"""
    rng = np.random.default_rng(seed)
    h, w = int(rng.integers(24, 180)), int(rng.integers(24, 180))
    frames = []
    for k in range(int(rng.integers(1, 4))):
        blobs = [(int(rng.integers(0, h)), int(rng.integers(0, w)), int(rng.integers(0, 3)), float(rng.uniform(50, 500)))] \
            if rng.random() < 0.4 else []
        frames.append(flood(seed * 10 + k, (h, w), field=rng.choice(["circle", "rect"]), frac=float(rng.uniform(0.1, 0.95)),
                            counts=float(rng.choice([3, 20, 200, 2000])), background=float(rng.uniform(0, 2)),
                            spots=[(rng.uniform(0.2, 0.8), rng.uniform(0.2, 0.8), rng.uniform(0.02, 0.1), rng.uniform(0.5, 1.6))],
                            gradient=float(rng.uniform(-0.4, 0.4)), hot_pixels=int(rng.integers(0, 6)), blobs=blobs))
    pixel_size = float(rng.choice([5.0, 2.5, 1.3, 4.0, 0.9]))
    kw = {"ufov_ratio": float(rng.choice([0.95, 0.8, 1.0])), "cfov_ratio": float(rng.choice([0.75, 0.5])),
          "window_size": int(rng.choice([3, 5, 7])), "threshold": float(rng.choice([0.75, 0.5, 0.9]))}
    return np.stack(frames), pixel_size, kw


def _check_against_oracle(frames, pixel_size, kw):
    ctx = nat.Context.default()
    b = orc.determine_binning(pixel_size)
    st = nat.nm_stages(ctx, frames, b, 1 - kw["ufov_ratio"], 1 - kw["cfov_ratio"] * kw["ufov_ratio"], kw["window_size"], kw["threshold"])
    for i, frame in enumerate(frames):
        o = orc.analyze_frame(frame, pixel_size, **kw)
        row = st["results"][i]
        np.testing.assert_array_equal(st["filtered"][i], o["filtered_s"])
        np.testing.assert_array_equal(st["cleaned"][i], o["cleaned_s"])
        assert np.array_equal(row["threshold"], o["threshold"], equal_nan=True)
        if o["status"] == "no_component":
            assert row["status"] == nat.NM_NO_COMPONENT
            continue
        assert row["status"] == nat.NM_OK
        np.testing.assert_array_equal(st["edt2"][i], o["edt2"])
        hb, wb = frames.shape[1] // b + (frames.shape[1] % b > 0), frames.shape[2] // b + (frames.shape[2] % b > 0)
        for k, name in enumerate(("ufov", "cfov")):
            f = o[name]
            assert row["longest"] == f["longest"] and row["erosion"][k] == f["erosion"]
            np.testing.assert_array_equal(st["masks"][i, k].astype(bool), f["mask"])
            assert row["n_fov"][k] == f["n_fov"]
            if f["iu"] is not None:
                assert row["iu"][k] == f["iu"]
                assert divmod(int(row["max_index"][k]), wb) == f["max_point"]
                assert divmod(int(row["min_index"][k]), wb) == f["min_point"]
            for axis in (0, 1):
                assert row["du_count"][2 * k + axis] == f[f"du_count_{axis}"]
                if f[f"du_{axis}"] is not None:
                    v, pos = f[f"du_{axis}"]
                    assert row["du_max"][2 * k + axis] == v
                    assert divmod(int(row["du_index"][2 * k + axis]), wb) == pos
        assert st["filtered"].shape[1:] == (hb, wb)


@pytest.mark.parametrize("seed", range(120))
def test_stages_match_the_oracle(seed):
    _check_against_oracle(*_fuzz_frames(seed))


@pytest.mark.parametrize("shape,pixel_size", [((139, 140), 5.0), ((400, 380), 5.0), ((1100, 1030), 2.3)])
def test_binned_frames_beyond_shared_memory(shape, pixel_size):
    """12 bytes per binned pixel over the shared-memory limit: the per-frame stages run from the global workspace"""
    frames = np.stack([flood(900 + k, shape, counts=100, spots=[(0.4, 0.6, 0.05, 1.3)], gradient=0.1, hot_pixels=4) for k in range(2)])
    _check_against_oracle(frames, pixel_size, {"ufov_ratio": 0.95, "cfov_ratio": 0.75, "window_size": 5, "threshold": 0.75})


def test_batch_equals_frame_by_frame_and_device_input():
    frames = np.stack([flood(50 + k, (300, 280), counts=[40, 0, 60, 80][k] if k != 1 else 0.0, background=0.0 if k == 1 else 0.3)
                       for k in range(4)])
    res = nuclear.analyze_batch(frames, 1.3)
    assert res[1].status == nat.NM_NO_COMPONENT
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        res[1].raise_for_status()
    for k in range(len(frames)):
        one = nuclear.analyze_batch(frames[k], 1.3)
        assert res.rows[k].tobytes() == one.rows[0].tobytes()
        assert np.array_equal(res[k].binned_frame, one[0].binned_frame)
        if res[k].status == nat.NM_OK:
            assert np.array_equal(res[k].ufov.mask, one[0].ufov.mask) and np.array_equal(res[k].cfov.mask, one[0].cfov.mask)
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, frames) as b:
        dev = nuclear.analyze_batch(b, 1.3, arrays=False)
    assert dev.rows.tobytes() == res.rows.tobytes()


def test_uint8_frames_are_widened_and_other_dtypes_raise():
    f8 = flood(60, (64, 64), counts=50, dtype=np.uint8)
    assert nuclear.analyze_batch(f8, 5.0).rows.tobytes() == nuclear.analyze_batch(f8.astype(np.uint16), 5.0).rows.tobytes()
    with pytest.raises(NotImplementedError, match="float32"):
        nuclear.analyze_batch(f8.astype(np.float32), 5.0)
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, f8[None].astype(np.int32)) as b, pytest.raises(NotImplementedError, match="int32"):
        nuclear.analyze_batch(b, 5.0)


def test_get_fov_matches_the_oracle():
    cleaned = orc.preprocess(flood(70, (120, 100), counts=200, hot_pixels=5, blobs=[(8, 90, 3, 200)]), 1, 0.75)["cleaned"]
    for size in (0.95, 0.7124999999999999, 0.3):
        fov, bx, by = nuclear.get_fov(cleaned, size)
        o = orc.fov(cleaned, size)
        assert np.array_equal(fov, o["fov"]) and np.array_equal(bx, o["boundary_x"]) and np.array_equal(by, o["boundary_y"])
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        nuclear.get_fov(np.zeros((10, 10)), 0.95)


def test_max_count_rate_over_a_long_dynamic_stack(tmp_path):
    rng = np.random.default_rng(80)
    frames = rng.poisson(rng.uniform(10, 400, size=(2000, 1, 1)), size=(2000, 128, 128)).astype(np.uint16)
    mcr = nuclear.MaxCountRate(write_nm(tmp_path / "long.dcm", frames, explicit=False))
    mcr.analyze(frame_duration=0.25)
    want = frames.reshape(2000, -1).sum(1) / 0.25
    assert np.array_equal(np.array([mcr.sums[k] for k in range(2000)]), want)
    assert mcr.max_frame == int(np.argmax(want)) and mcr.max_countrate == want.max()
