"""CPU: the TomographicContrast oracle (oracle/tomo_contrast_oracle.py) against the goldens of the unmodified reference, bit for bit,
and against live scipy.optimize.minimize; and a host build of the device's Nelder-Mead search and 4-key argsort
(csrc/nuclear_tomo.cuh, through tests/nt_nm_check.cu) against np.argsort on every weak ordering of 4 keys and against the oracle."""
from __future__ import annotations

import itertools
import json
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import tomo_contrast_oracle as O
from tests.golden.tomo_contrast_cases import CASES, DEFAULT_ANGLES, DEFAULT_DIAMETERS, jaszczak

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "tomo_contrast_golden.npz"))


def _avx512() -> bool:
    try:
        from numpy._core._multiarray_umath import __cpu_features__
    except ImportError:
        return False
    return bool(__cpu_features__.get("AVX512_SKX"))


def _same(a, b) -> bool:
    """equal floats, nan equal to nan, -0.0 distinct from 0.0"""
    a, b = float(a), float(b)
    return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))


def _michelson100(a, b):
    return O.michelson(a, b) * 100


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_the_reference(name):
    build, pixel_size, kwargs = CASES[name]
    want = json.loads(str(GOLDEN[name]))
    try:
        got = O.analyze(build(), pixel_size, **kwargs)
    except ValueError as e:
        assert want["analyze_error"] == ["ValueError", str(e)]
        return
    assert "analyze_error" not in want
    assert sorted(got["slice_data"]) == sorted(want["slice_data"])
    for k, v in got["slice_data"].items():
        w = want["slice_data"][k]
        assert v["longest"] - v["erosion"] == w["fov diameter"] and v["area"] == w["area"]
        assert [v["centroid_col"], v["centroid_row"]] == w["center"]
        assert _same(v["uniformity"], w["uniformity"]) and _same(v["value"], w["value"])
    assert got["uniformity_frame"] == want["uniformity_frame"] and _same(got["baseline"], want["uniformity_value"])
    assert [[s["nfev"], s["nit"]] for s in got["spheres"]] == want["search"]
    for k, s in enumerate(got["spheres"]):
        w = want["rois"][str(k + 1)]
        assert list(s["x"]) == [w["x"], w["y"], w["z"]] and s["radius"] == w["radius"]
        mean = s["sum"] / s["count"] if s["count"] else math.nan
        assert _same(mean, w["mean"]) and _same(s["min"] if s["count"] else math.nan, w["min"])
        assert _same(_michelson100(mean, got["baseline"]), w["mean_contrast"])


def test_argsort4_matches_numpy_on_every_weak_ordering():
    """every weak ordering of 4 keys, each realised with several values (nans, +-0, +-inf) per rank"""
    if not _avx512():
        pytest.skip("numpy's CPU features lack AVX512_SKX: np.argsort orders ties by another network on this host")
    levels = [[-math.inf, -1e300], [-2.5, -1.0], [-0.0, 0.0], [3.0, 7.5], [math.inf, 1e308]]
    n = 0
    for pattern in itertools.product(range(6), repeat=4):
        used = sorted({p for p in pattern if p < 5})
        for shift in range(5 - len(used) + 1):
            for pick in itertools.product(range(2), repeat=4):
                keys = [math.nan if p == 5 else levels[used.index(p) + shift][pick[i]] for i, p in enumerate(pattern)]
                if any(p < 5 for p in pattern) and len({keys[i] for i, p in enumerate(pattern) if p < 5}) != len(used):
                    continue         # two ranks realised by equal values would be another pattern
                assert O.argsort4(keys) == list(np.argsort(np.array(keys))), keys
                n += 1
    assert n > 10000


def _nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


@pytest.fixture(scope="module")
def nm_check(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    exe = str(tmp_path_factory.mktemp("nt") / "nt_nm_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "nt_nm_check.cu")],
                   check=True, capture_output=True)
    return exe


def test_host_build_of_the_device_argsort(nm_check, tmp_path):
    """the device's argsort4 on every key pattern over {nan, -inf, -1, -0.0, 0.0, 2, inf}, against the oracle's"""
    vals = [math.nan, -math.inf, -1.0, -0.0, 0.0, 2.0, math.inf]
    keys = np.array(list(itertools.product(vals, repeat=4)), np.float64)
    src, dst = tmp_path / "keys.bin", tmp_path / "ind.bin"
    keys.tofile(src)
    subprocess.run([nm_check, "argsort", str(src), str(dst)], check=True, capture_output=True)
    got = np.fromfile(dst, np.int32).reshape(-1, 4)
    for k, row in zip(keys, got):
        assert list(row) == O.argsort4(k), k


def _volume(seed):
    rng = np.random.default_rng(seed)
    return jaszczak(seed, shape=(int(rng.integers(14, 24)), int(rng.integers(30, 48)), int(rng.integers(30, 48))),
                    z_extent=(1, int(rng.integers(12, 14))), counts=float(rng.choice([20, 300])), sphere_gain=float(rng.uniform(0, 2)))


@pytest.mark.parametrize("seed", range(6))
def test_host_build_of_the_device_search_matches_the_oracle(nm_check, tmp_path, seed):
    """the device's nelder_mead on the host, fed the oracle's objective values through a table of evaluated points: every sphere
    of a seeded volume, at the default limits and at small maxfun / maxiter"""
    vol = _volume(seed)
    for maxfun, maxiter in ((600, 600), (7, 600), (600, 4), (12, 9)):
        o = O.analyze(vol, 4.4, maxfun=maxfun, maxiter=maxiter)
        base = o["baseline"]
        u = o["slice_data"][max(o["slice_data"], key=lambda k: o["slice_data"][k]["uniformity"])]
        uz = int(max(o["slice_data"], key=lambda k: o["slice_data"][k]["uniformity"])) - 1
        for s, (angle, d) in zip(o["spheres"], zip(DEFAULT_ANGLES, DEFAULT_DIAMETERS)):
            dist = math.sqrt(u["area"] / math.pi) * 0.65
            x0 = (u["centroid_col"] + dist * math.cos(math.radians(angle)), u["centroid_row"] + dist * math.sin(math.radians(angle)), uz)
            lb, ub = (x0[0] - 5, x0[1] - 5, uz - 3), (x0[0] + 5, x0[1] + 5, uz + 3)
            r2 = (d / (2 * 4.4)) ** 2
            inp = np.array([*x0, *lb, *ub, r2, base, maxfun, maxiter], np.float64)
            src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
            np.concatenate([inp, np.asarray(vol.shape, np.float64), vol.astype(np.float64).ravel()]).tofile(src)
            subprocess.run([nm_check, "search", str(src), str(dst)], check=True, capture_output=True)
            out = np.fromfile(dst, np.float64)
            assert list(out[:3]) == list(s["x"]) and _same(out[3], s["fun"]), (maxfun, maxiter)
            assert [int(v) for v in out[4:7]] == [s["nfev"], s["nit"], s["status"]]


@pytest.mark.parametrize("seed", range(3))
def test_oracle_matches_live_scipy(seed):
    """scipy.optimize.minimize(method="Nelder-Mead") with np.argsort on the oracle's objective: the same search, where np.argsort
    is the AVX-512 network the oracle pins"""
    if not _avx512():
        pytest.skip("numpy's CPU features lack AVX512_SKX: np.argsort orders ties by another network on this host")
    from scipy.optimize import minimize

    vol = _volume(100 + seed)
    o = O.analyze(vol, 4.4)
    data = o["slice_data"]
    start = max(data, key=lambda k: data[k]["uniformity"])
    u, uz = data[start], int(start) - 1
    for s, angle, d in zip(o["spheres"], DEFAULT_ANGLES, DEFAULT_DIAMETERS):
        dist = math.sqrt(u["area"] / math.pi) * 0.65
        cx, cy = u["centroid_col"] + dist * math.cos(math.radians(angle)), u["centroid_row"] + dist * math.sin(math.radians(angle))
        r2 = (d / (2 * 4.4)) ** 2
        res = minimize(lambda x: O.objective(vol, x, r2, o["baseline"])[0], x0=(cx, cy, uz), method="Nelder-Mead",
                       bounds=[(cx - 5, cx + 5), (cy - 5, cy + 5), (uz - 3, uz + 3)])
        assert list(res.x) == list(s["x"]) and (res.nfev, res.nit) == (s["nfev"], s["nit"])
