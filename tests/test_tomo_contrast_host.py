"""CPU: the C layout of the TomographicContrast rows, the host helpers that keep the reference's behaviour, and the argument errors
raised before any device call."""
from __future__ import annotations

import os
import subprocess

import numpy as np
import pytest

from pylinac_b200 import _native as nat
from pylinac_b200 import nuclear
from tests.test_cabi import HEADER, python_layout


@pytest.mark.parametrize("struct,dtype", [("epid_nt_slice", nat.NT_SLICE_DTYPE), ("epid_nt_sphere_in", nat.NT_SPHERE_IN_DTYPE),
                                          ("epid_nt_sphere", nat.NT_SPHERE_DTYPE)])
def test_rows_match_the_header(tmp_path, struct, dtype):
    size, members = python_layout(dtype)
    prints = [f'std::printf("sizeof %zu\\n", sizeof({struct}));']
    prints += [f'std::printf("{m} %zu %zu\\n", offsetof({struct}, {m}), sizeof({struct}::{m}));' for m in members]
    src = tmp_path / "nt_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "nt_layout")], check=True)
    out = subprocess.run([str(tmp_path / "nt_layout")], check=True, capture_output=True, text=True).stdout
    header = {m: tuple(int(v) for v in vals) for m, *vals in (line.split() for line in out.splitlines())}
    assert header.pop("sizeof") == (size,)
    assert header == members


def test_sphere_helpers_keep_the_reference_behaviour():
    vol = np.arange(4 * 5 * 6, dtype=np.uint16).reshape(4, 5, 6)
    mask = nuclear.create_sphere_mask(vol.shape, row=2.0, col=3.0, zed=1.5, radius=1.2)
    z, y, x = np.nonzero(mask)
    assert np.all((x - 3.0) ** 2 + (y - 2.0) ** 2 + (z - 1.5) ** 2 <= 1.2 ** 2) and mask.sum() == 10
    s = nuclear.sample_sphere(vol, row=2.0, col=3.0, zed=1.5, radius=1.2)
    assert s.dtype == np.float64 and np.array_equal(s[mask], vol[mask]) and np.isnan(s[~mask]).all()
    base = 50.0
    mean = vol[mask].mean()
    assert nuclear.contrast_f(np.array([3.0, 2.0, 1.5]), vol, 1.2, base) == -((mean - base) / (mean + base)) * 100
    with pytest.warns(RuntimeWarning, match="Mean of empty slice"):
        assert nuclear.contrast_f(np.array([30.0, 2.0, 1.5]), vol, 1.2, base) == 0.0


def test_hand_built_roi_samples_its_volume():
    vol = np.random.default_rng(1).integers(1, 100, (6, 9, 9)).astype(np.uint16)
    roi = nuclear.TomographicROI(vol, 40.0, 4.2, 3.9, 2.5, 2.0, 1)
    s = nuclear.sample_sphere(vol, row=3.9, col=4.2, zed=2.5, radius=2.0)
    assert roi.mean_value == float(np.nanmean(s)) and roi.min_value == float(np.nanmin(s))
    assert isinstance(roi.sphere_array, tuple) and np.array_equal(roi.sphere_array[0], s, equal_nan=True)
    dev = nuclear.TomographicROI(None, 40.0, 4.2, 3.9, 2.5, 2.0, 1, stats=(int(vol[~np.isnan(s)].sum()), int((~np.isnan(s)).sum()), 1))
    assert dev.mean_value == roi.mean_value
    with pytest.raises(RuntimeError, match="device batch"):
        dev.sphere_array


def test_argument_errors_before_the_device():
    with pytest.raises(NotImplementedError, match="float32"):
        nuclear.analyze_tomographic_contrast_batch(np.zeros((4, 8, 8), np.float32), 4.4)
    with pytest.raises(ValueError, match="got 2-D"):
        nuclear.analyze_tomographic_contrast_batch(np.zeros((8, 8), np.uint16), 4.4)

