"""CPU: the C layout of the TomographicUniformity row, a host build of the device's pairwise sum (csrc/np_sum.cuh, through
tests/np_sum_check.cu) against numpy, and the frame-argument errors raised before any device call."""
from __future__ import annotations

import os
import shutil
import subprocess

import numpy as np
import pytest

from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from tests.test_cabi import HEADER, python_layout

HERE = os.path.dirname(os.path.abspath(__file__))


def test_row_matches_the_header(tmp_path):
    size, members = python_layout(nat.TU_RESULT_DTYPE)
    prints = ['std::printf("sizeof %zu\\n", sizeof(epid_tu_result));']
    prints += [f'std::printf("{m} %zu %zu\\n", offsetof(epid_tu_result, {m}), sizeof(epid_tu_result::{m}));' for m in members]
    src = tmp_path / "tu_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "tu_layout")], check=True)
    out = subprocess.run([str(tmp_path / "tu_layout")], check=True, capture_output=True, text=True).stdout
    header = {m: tuple(int(v) for v in vals) for m, *vals in (line.split() for line in out.splitlines())}
    assert header.pop("sizeof") == (size,)
    assert header == members


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def test_host_build_of_the_pairwise_sum_matches_numpy(tmp_path):
    """pw and the slot-wise block evaluation for every length 0-8200 (the leaf boundaries 7/8/9, 127/128/129, 135/136 and numpy's
    8192-element buffer included) against np.sum of the same prefix"""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    exe = str(tmp_path / "np_sum_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(HERE, "np_sum_check.cu")],
                   check=True, capture_output=True)
    x = np.random.default_rng(11).random(8200) * 1e4 / 7
    src, dst = tmp_path / "x.bin", tmp_path / "out.bin"
    x.tofile(src)
    subprocess.run([exe, str(src), str(dst)], check=True, capture_output=True)
    got = np.fromfile(dst, np.float64).reshape(-1, 3)
    assert len(got) == len(x) + 1
    for n in range(len(x) + 1):
        want = np.sum(x[:n])
        assert (0.0 + got[n] == want).all(), n


@pytest.mark.parametrize("first,last,msg", [
    (-1, -1, "The first frame index is outside the array bounds"),
    (0, 8, "The last frame index is outside the array bounds"),
    (5, 3, "The first frame index must be less than the last frame index"),
    (4, 4, "The first frame index must be less than the last frame index"),
])
def test_frame_errors_before_the_device(first, last, msg):
    with pytest.raises(ValueError, match=msg):
        nuclear.analyze_tomographic_uniformity_batch(np.zeros((8, 16, 16), np.uint16), 4.4, first_frame=first, last_frame=last)


def test_empty_slab_and_dtypes_before_the_device():
    with pytest.warns(RuntimeWarning, match="Mean of empty slice"), pytest.raises(ValueError, match="max\\(\\) iterable"):
        nuclear.analyze_tomographic_uniformity_batch(np.zeros((1, 16, 16), np.uint16), 4.4)
    with pytest.raises(NotImplementedError, match="float32"):
        nuclear.analyze_tomographic_uniformity_batch(np.zeros((4, 8, 8), np.float32), 4.4)
    with pytest.raises(ValueError, match="got 2-D"):
        nuclear.analyze_tomographic_uniformity_batch(np.zeros((8, 8), np.uint16), 4.4)
    with pytest.raises(ValueError, match="window_size"):
        nuclear.analyze_tomographic_uniformity_batch(np.zeros((4, 8, 8), np.uint16), 4.4, window_size=0)
