"""CPU: the NM ingest (dicom.read_nm_frames, core.image.NMImageStack), determine_binning, the result row's C layout and the
PlanarUniformity / MaxCountRate text and data formatting from stubbed device rows (no compute calls)."""
from __future__ import annotations

import json
import os
import subprocess

import numpy as np
import pytest

from pylinac_b200 import _native as nat
from pylinac_b200 import dicom, nuclear
from pylinac_b200.core.image import NMImageStack
from tests.nm_writer import write_nm
from tests.test_cabi import HEADER, python_layout


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("n", [1, 4])
def test_reader_returns_the_written_frames(tmp_path, explicit, dtype, n):
    frames = np.random.default_rng(n).integers(0, np.iinfo(dtype).max, (n, 13, 11)).astype(dtype)
    path = write_nm(tmp_path / "nm.dcm", frames, pixel_spacing_mm=2.4, explicit=explicit, preamble=explicit)
    stack = NMImageStack(path)
    assert len(stack) == n and stack.path == path
    assert stack.as_3d_array().dtype == dtype and np.array_equal(stack.as_3d_array(), frames)
    assert [float(v) for v in stack.metadata.PixelSpacing] == [2.4, 2.4]
    assert all(np.array_equal(f.array, frames[k]) for k, f in enumerate(stack.frames))


def test_batched_reader_concatenates_files_and_read_frames_still_rejects_stacks(tmp_path):
    a = np.arange(3 * 6 * 5, dtype=np.uint16).reshape(3, 6, 5)
    b = a[:2] + 1000
    pa, pb = write_nm(tmp_path / "a.dcm", a), write_nm(tmp_path / "b.dcm", b, explicit=False)
    out, headers = dicom.read_nm_frames([pa, pb])
    assert np.array_equal(out, np.concatenate([a, b])) and len(headers) == 2
    with pytest.raises(ValueError, match="out must be"):
        dicom.read_nm_frames([pa], out=np.empty((2, 6, 5), np.uint16))
    with pytest.raises(ValueError):
        dicom.read_frames([pa])
    with pytest.raises(ValueError, match="differs"):
        dicom.read_nm_frames([pa, write_nm(tmp_path / "c.dcm", a[:, :5])])


def test_non_nm_files_raise_type_error(tmp_path):
    path = write_nm(tmp_path / "ct.dcm", np.zeros((2, 4, 4), np.uint16), modality="CT")
    with pytest.raises(TypeError, match="The file is not a NM image"):
        NMImageStack(path)
    with pytest.raises(TypeError, match="The file is not a NM image"):
        nuclear.PlanarUniformity(path)


def test_determine_binning():
    cases = {8.32: 1, 4.48: 1, 4.4799: 2, 2.24: 2, 2.2399: 4, 1.2: 4, 0.6: 8, 0.3: 16, 0.25: 32, 0.1: 64}
    assert {p: nuclear.determine_binning(p) for p in cases} == cases


def test_integral_uniformity_is_michelson_x100():
    assert nuclear.integral_uniformity(np.array([90.0, np.nan, 110.0])) == (110.0 - 90.0) / (110.0 + 90.0) * 100


def test_result_row_matches_the_header(tmp_path):
    size, members = python_layout(nat.NM_RESULT_DTYPE)
    prints = ['std::printf("sizeof %zu\\n", sizeof(epid_nm_result));']
    prints += [f'std::printf("{m} %zu %zu\\n", offsetof(epid_nm_result, {m}), sizeof(epid_nm_result::{m}));' for m in members]
    src = tmp_path / "nm_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "nm_layout")], check=True)
    out = subprocess.run([str(tmp_path / "nm_layout")], check=True, capture_output=True, text=True).stdout
    header = {m: tuple(int(v) for v in vals) for m, *vals in (line.split() for line in out.splitlines())}
    assert header.pop("sizeof") == (size,)
    assert header == members


def _stub_result(rows, shape=(20, 30), window=5):
    return nuclear.UniformityBatchResult(rows, 1, window, shape, nuclear._DeviceArrays(None, None))


def _row(iu=(1.2345, 0.5), du=(0.75, 2.5, 0.25, 0.125), n_fov=(10, 10), counts=(4, 4, 4, 4)):
    r = np.zeros((), nat.NM_RESULT_DTYPE)
    r["iu"], r["du_max"], r["n_fov"], r["du_count"] = iu, du, n_fov, counts
    r["max_index"], r["min_index"], r["du_index"] = (61, 62), (95, 96), (31, 32, 33, 34)
    return r


def test_results_and_results_data_from_stubbed_rows():
    pu = nuclear.PlanarUniformity.__new__(nuclear.PlanarUniformity)
    res = _stub_result(np.stack([_row(), _row(iu=(3.0, 4.0))]))
    pu.frame_results = {str(k + 1): {"ufov": r.ufov, "cfov": r.cfov} for k, r in enumerate(res)}
    assert pu.results() == ("Frame 1:\nUFOV integral uniformity: 1.23%\nUFOV differential uniformity 2.50%\n"
                            "CFOV integral uniformity: 0.50%\nCFOV differential uniformity 0.25%\n\n"
                            "Frame 2:\nUFOV integral uniformity: 3.00%\nUFOV differential uniformity 2.50%\n"
                            "CFOV integral uniformity: 4.00%\nCFOV differential uniformity 0.25%\n\n")
    d = pu.results_data(as_dict=True)
    assert d["Frame 1"] == {"ufov_integral_uniformity": 1.2345, "ufov_differential_uniformity": 2.5, "cfov_integral_uniformity": 0.5,
                            "cfov_differential_uniformity": 0.25}
    assert json.loads(json.loads(pu.results_data(as_json=True))["Frame 2"])["cfov_integral_uniformity"] == 4.0
    assert isinstance(pu.results_data()["Frame 1"], nuclear.PlanarUniformityResults)
    u = res[0].ufov
    assert u.max_point == (2, 1) and u.min_point == (3, 5) and u.differential_uniformity_y == (0.75, (1, 1))
    assert u.differential_uniformity_x == (2.5, (1, 2))


def test_stubbed_rows_raise_the_reference_exceptions():
    res = _stub_result(np.stack([_row(n_fov=(0, 3), counts=(0, 0, 1, 0))]))
    u, c = res[0].ufov, res[0].cfov
    with pytest.raises(ValueError, match="zero-size array to reduction operation fmax"):
        u.integral_uniformity
    with pytest.raises(ValueError, match="All-NaN slice encountered"):
        u.max_point
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        u.differential_uniformity
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        c.differential_uniformity
    small = _stub_result(np.stack([_row()]), shape=(4, 30))
    with pytest.raises(ValueError, match="window shape cannot be larger than input array shape"):
        small[0].ufov.differential_uniformity
    with pytest.raises(RuntimeError, match="arrays=False"):
        res[0].binned_frame
    row = _row()
    row["status"] = nat.NM_NO_COMPONENT
    with pytest.raises(ValueError, match=r"max\(\) iterable argument is empty"):
        _stub_result(np.stack([row]))[0].raise_for_status()


def test_window_size_must_be_a_positive_integer():
    with pytest.raises(ValueError, match="window_size"):
        nuclear.analyze_batch(np.zeros((8, 8), np.uint16), 5.0, window_size=0)
