"""CPU: the numpy oracle of pylinac.nuclear's PlanarUniformity (oracle/nuclear_oracle.py) against the goldens of the unmodified
reference, and, where the reference tree exists, against the live reference on further seeds."""
from __future__ import annotations

import json
import os
import warnings

import numpy as np
import pytest

from oracle import nuclear_oracle as orc
from tests.golden.nuclear_cases import CASES, digest, flood

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "nuclear_golden.npz"))


def _check_fov(o, want):
    assert digest(o["fov"]) == want["fov"]
    assert digest(o["boundary_x"]) == want["boundary_x"] and digest(o["boundary_y"]) == want["boundary_y"]
    if o["iu"] is None:
        assert want["integral_uniformity"]["error"][0] == "ValueError" and "error" in want["max_point"]
    else:
        assert want["integral_uniformity"]["value"] == o["iu"]
        assert tuple(want["max_point"]["value"]) == o["max_point"] and tuple(want["min_point"]["value"]) == o["min_point"]
    if o["window_too_large"]:
        assert want["differential_uniformity"]["error"] == ["ValueError", "window shape cannot be larger than input array shape"]
        return
    for axis in (0, 1):
        count, v, pos = want["du_axes"][axis]
        assert count == o[f"du_count_{axis}"]
        assert (v, pos) == ((None, None) if o[f"du_{axis}"] is None else (o[f"du_{axis}"][0], list(o[f"du_{axis}"][1])))
    if o["du"] is None:
        assert want["differential_uniformity"]["error"] == ["ValueError", "max() iterable argument is empty"]
    else:
        assert want["differential_uniformity"]["value"] == o["du"]


def _check_case(frames, pixel_size, kwargs, want):
    outs = [orc.analyze_frame(f, pixel_size, **kwargs) for f in frames]
    bad = [o for o in outs if o["status"] != "ok"]
    if bad:
        assert want["analyze_error"] == ["ValueError", "max() iterable argument is empty"]
        return
    assert sorted(want["frames"]) == [str(k + 1) for k in range(len(frames))]
    for k, o in enumerate(outs):
        fr = want["frames"][str(k + 1)]
        assert digest(o["cleaned"]) == fr["binned_frame"]
        _check_fov(o["ufov"], fr["ufov"])
        _check_fov(o["cfov"], fr["cfov"])


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n][3] == "NM"))
def test_oracle_matches_the_goldens(name):
    build, pixel_size, kwargs, _ = CASES[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _check_case(build(), pixel_size, kwargs, json.loads(str(GOLDEN[name])))


def test_determine_binning_and_exact_stage_planes():
    assert [orc.determine_binning(p) for p in (5.0, 4.48, 4.47, 2.4, 1.2, 0.6, 0.3, 0.25)] == [1, 1, 2, 2, 4, 8, 16, 32]
    o = orc.analyze_frame(flood(5, (90, 70), counts=300), 2.3)
    assert np.array_equal(o["filtered_s"] % 1, np.zeros_like(o["filtered_s"]))
    assert np.array_equal(o["cleaned_s"] / 16.0, o["cleaned"])


@pytest.mark.skipif(not os.path.isdir("/root/reference/pylinac"), reason="the reference tree is not available")
@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_the_live_reference(seed):
    from tests.golden import make_nuclear_golden as mk
    from oracle import skimage_nuclear

    rn = skimage_nuclear.install()
    rng = np.random.default_rng(300 + seed)
    shape = (int(rng.integers(40, 140)), int(rng.integers(40, 140)))
    frames = np.stack([flood(400 + seed, shape, field=["circle", "rect"][seed % 2], counts=float(rng.choice([30, 300])),
                             frac=float(rng.uniform(0.3, 0.9)), hot_pixels=3, gradient=float(rng.uniform(-0.3, 0.3)))])
    pixel_size = float(rng.choice([5.0, 2.4, 1.5]))
    kwargs = {"window_size": int(rng.choice([3, 5, 7])), "threshold": float(rng.choice([0.6, 0.75]))}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mk.CASES["live"] = (lambda: frames, pixel_size, kwargs, "NM")
        try:
            want = json.loads(json.dumps(mk.planar_record(rn, "live")))
        finally:
            del mk.CASES["live"]
        _check_case(frames, pixel_size, kwargs, want)
