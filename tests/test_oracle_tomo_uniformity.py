"""CPU: the TomographicUniformity oracle (oracle/tomo_uniformity_oracle.py) against the goldens of the unmodified reference, bit for
bit, and its explicit summation orders (pairwise sum, block sum, convolve2d) against numpy / scipy on seeded non-integer inputs."""
from __future__ import annotations

import json
import math
import os

import numpy as np
import pytest
from scipy.signal import convolve2d

from oracle import skimage_nuclear as sk
from oracle import tomo_uniformity_oracle as O
from tests.golden.nuclear_cases import digest
from tests.golden.tomo_uniformity_cases import CASES

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "tomo_uniformity_golden.npz"))


def _same(a, b) -> bool:
    a, b = float(a), float(b)
    return (math.isnan(a) and math.isnan(b)) or a == b


def _check_fov(got: dict, want: dict, nan_outside: bool):
    if got["iu"] is None:
        assert want["integral_uniformity"]["error"][0] == "ValueError"
    else:
        assert got["iu"] == want["integral_uniformity"]["value"]
        assert list(got["max_point"]) == want["max_point"]["value"] and list(got["min_point"]) == want["min_point"]["value"]
    if got["window_too_large"]:
        assert want["differential_uniformity"]["error"][1] == "window shape cannot be larger than input array shape"
        return
    for axis in (0, 1):
        count, value, pos = want["du_axes"][axis]
        assert got[f"du_count_{axis}"] == count
        if count:
            assert got[f"du_{axis}"][0] == value and list(got[f"du_{axis}"][1]) == pos
    if got["du"] is None:
        assert want["differential_uniformity"]["error"] == ["ValueError", "max() iterable argument is empty"]
    else:
        assert got["du"] == want["differential_uniformity"]["value"]
    # center_border_ratio sets the zeros of the center FOV's own array to nan
    fov = np.where(got["fov"] == 0, np.nan, got["fov"]) if nan_outside else got["fov"]
    assert digest(fov) == want["fov"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_the_reference(name):
    build, pixel_size, kwargs, calls = CASES[name]
    want = json.loads(str(GOLDEN[name]))
    volume = build()
    kw = dict(kwargs)
    try:
        first, last = O.slab(len(volume), kw.pop("first_frame", 0), kw.pop("last_frame", -1))
    except ValueError as e:
        assert want["analyze_error"] == ["ValueError", str(e)]
        return
    if calls > 1:                     # the first analyze() leaves one averaged frame: the slab [0, 0) of it is empty
        first, last = O.slab(1, kwargs.get("first_frame", 0), kwargs.get("last_frame", -1))
    if first >= last:
        assert want["analyze_error"] == ["ValueError", "max() iterable argument is empty"]
        return
    got = O.analyze(volume, pixel_size, first, last, **kw)
    if got["status"] != "ok":
        assert want["analyze_error"] == ["ValueError", "max() iterable argument is empty"]
        return
    assert "analyze_error" not in want
    assert digest(got["mean"]) == want["mean_frame"] and digest(got["cleaned"]) == want["binned_frame"]
    assert _same(got["center_border_ratio"], want["center_ratio"])
    for k in ("ufov", "cfov", "center_fov"):
        _check_fov(got[k], want["fovs"][k], k == "center_fov")


def test_pairwise_sum_matches_numpy():
    rng = np.random.default_rng(7)
    for n in list(range(0, 301)) + list(range(8190, 8201)):
        x = rng.random(n) * 1000 / 7
        assert O.np_sum(x) == np.sum(x), n
        assert O.np_sum(x) == x.sum(), n
    for shape in [(1, 1), (3, 5), (16, 16), (33, 47), (64, 64), (100, 130), (256, 256)]:
        a = rng.random(shape) * 3e4 / 3
        assert O.np_sum(a) == np.sum(a), shape
        nanned = np.where(rng.random(shape) < 0.3, np.nan, a)
        nanned.flat[0] = a.flat[0]
        tot = O.np_sum(np.where(np.isnan(nanned), 0, nanned))
        cnt = int((~np.isnan(nanned)).sum())
        assert np.float64(tot) / cnt == np.nanmean(nanned), shape
        sel = a[a >= np.median(a)]
        assert np.float64(0.0 + O.pw(sel)) / sel.size == sel.mean(), shape


@pytest.mark.parametrize("b", [1, 2, 4, 8, 16, 64])
def test_block_sum_matches_block_reduce(b):
    rng = np.random.default_rng(b)
    for shape in [(b * 3, b * 2), (b * 3 + 1, b * 2 + b - 1), (70, 61)]:
        m = rng.integers(0, 2000, shape) / rng.choice([3.0, 7.0, 25.0])
        assert np.array_equal(O.block_sum(m, b), sk.block_reduce(m, (b, b), np.sum)), shape


def test_filter_matches_convolve2d():
    rng = np.random.default_rng(3)
    kernel = np.array([[1, 2, 1], [2, 4, 2], [1, 2, 1]], dtype=float)
    kernel /= kernel.sum()
    for shape in [(3, 3), (5, 9), (32, 32), (47, 33)]:
        a = rng.random(shape) * 1e4 / 7
        want = convolve2d(a, kernel, mode="same")
        want[0, :] = want[-1, :] = 0
        want[:, 0] = want[:, -1] = 0
        assert np.array_equal(O.nema_filter(a), want), shape
