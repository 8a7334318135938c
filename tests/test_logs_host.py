"""CPU: the machine-log parser and MLC statistics against the unmodified reference (tests/golden/log_golden.npz), the reference's
exceptions for malformed files, and the numpy statement of calc_map (oracle/log_oracle.py) pinned to the golden fluence maps."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from oracle import log_oracle
from pylinac_b200 import _native as nat
from pylinac_b200 import log_analyzer as la
from tests.golden.log_cases import BAD_CASES, CASES, MAP_SETTINGS, SUB_COLS, SUB_ROWS, SUBBEAM_SETTINGS, write_case

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "log_golden.npz"))
EXC = {"builtins.ValueError": ValueError, "struct.error": struct.error, "pylinac.log_analyzer.DynalogMatchError": la.DynalogMatchError,
       "pylinac.log_analyzer.NotALogError": la.NotALogError}


def sha1(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(a, dtype=np.float64).tobytes()).digest(), np.uint8)


def check_map(key, a):
    assert tuple(G[f"{key}/shape"]) == a.shape, key
    assert np.array_equal(G[f"{key}/sub"], a[SUB_ROWS, SUB_COLS]), key
    assert np.array_equal(G[f"{key}/sha1"], sha1(a)), key


@pytest.fixture(scope="module")
def logs(tmp_path_factory):
    out = {}
    for name in CASES:
        d = tmp_path_factory.mktemp(name)
        path = write_case(name, d)
        for f in sorted(os.listdir(d)):
            digest = hashlib.sha1(open(os.path.join(d, f), "rb").read()).digest()
            assert np.array_equal(G[f"{name}/file_sha1/{f}"], np.frombuffer(digest, np.uint8)), f"{name}: writer output changed"
        out[name] = la.load_log(path)
    return out


@pytest.mark.parametrize("name", CASES)
def test_parser_matches_reference(logs, name):
    log = logs[name]
    meta = json.loads(str(G[f"{name}/meta"]))
    assert log.treatment_type == meta["treatment_type"]
    assert log.num_beamholds == meta["num_beamholds"]
    assert hasattr(log, "fluence") == meta["has_fluence"]
    for k, v in meta["header"].items():
        got = getattr(log.header, k)
        assert (got.tolist() if isinstance(got, np.ndarray) else got) == v, k
    ax = log.axis_data
    if isinstance(log, la.TrajectoryLog):
        assert log.txt == meta["txt"] and log.is_hdmlc == meta["is_hdmlc"]
        if "metadata" in meta:
            assert vars(log.header.metadata) == meta["metadata"]
        for k, (s, m) in enumerate(zip(log.subbeams, meta["subbeams"])):
            assert (s.control_point, s.mu_delivered, s.rad_time, s.sequence_num, s.beam_name) == (
                m["control_point"], m["mu_delivered"], m["rad_time"], m["sequence_num"], m["beam_name"])
            assert np.array_equal(np.asarray(s._snapshots, np.int64), G[f"{name}/subbeam{k}/snapshots"])
        axes = {"collimator": ax.collimator, "gantry": ax.gantry, "mu": ax.mu, "beam_hold": ax.beam_hold,
                "control_point": ax.control_point, "couch_vert": ax.couch.vert, "carriage_A": ax.carriage_A}
        if ax.couch.pitch is not None:
            axes["couch_pitch"] = ax.couch.pitch
    else:
        assert int(ax.num_snapshots) == meta["num_snapshots"]
        axes = {"gantry": ax.gantry, "collimator": ax.collimator, "mu": ax.mu, "beam_hold": ax.beam_hold, "beam_on": ax.beam_on,
                "carriage_A": ax.carriage_A}
    axes.update({"x1": ax.jaws.x1, "x2": ax.jaws.x2, "y1": ax.jaws.y1, "y2": ax.jaws.y2})
    for k, a in axes.items():
        assert np.array_equal(np.asarray(a.actual, np.float64), G[f"{name}/axis/{k}/actual"]), k
        if a.expected is not None:
            assert np.array_equal(np.asarray(a.expected, np.float64), G[f"{name}/axis/{k}/expected"]), k
    mlc = ax.mlc
    assert np.array_equal(np.asarray(mlc.snapshot_idx, np.int64), G[f"{name}/snapshot_idx"])
    leaves = np.stack([mlc.leaf_axes[i].actual for i in range(1, mlc.num_leaves + 1)])
    assert np.array_equal(sha1(leaves), G[f"{name}/leaves_actual_sha1"])
    assert np.array_equal(np.stack([mlc.leaf_axes[7].actual, mlc.leaf_axes[7].expected]), G[f"{name}/leaf7"])


@pytest.mark.parametrize("name", CASES)
def test_mlc_statistics_are_bit_identical(logs, name):
    mlc = logs[name].axis_data.mlc
    meta = json.loads(str(G[f"{name}/meta"]))
    assert np.array_equal(np.asarray(mlc.moving_leaves, np.int64), G[f"{name}/moving_leaves"])
    calls = {"rms_avg": lambda: mlc.get_RMS_avg(), "rms_avg_moving": lambda: mlc.get_RMS_avg(only_moving_leaves=True),
             "rms_max": lambda: mlc.get_RMS_max(), "rms_max_a": lambda: mlc.get_RMS_max("A"), "rms_p95": lambda: mlc.get_RMS_percentile(95),
             "err_p95": lambda: mlc.get_error_percentile(95), "err_p50_b": lambda: mlc.get_error_percentile(50, "B"),
             "err_p95_moving": lambda: mlc.get_error_percentile(95, only_moving_leaves=True)}
    assert list(calls) == meta["stats_keys"]
    raised = meta.get("stats_raised", {})
    for k, want in zip(meta["stats_keys"], G[f"{name}/stats"]):
        if k in raised:
            with pytest.raises(IndexError):
                calls[k]()
        else:
            assert float(calls[k]()) == want, k
    assert np.array_equal(np.asarray(mlc.get_RMS("both"), np.float64), G[f"{name}/rms"])
    assert np.array_equal(np.array([mlc.leaf_under_y_jaw(p) for p in range(1, mlc.num_pairs + 1)]), G[f"{name}/under_y_jaw"])


@pytest.mark.parametrize("name", BAD_CASES)
def test_malformed_files_raise_the_reference_exception(tmp_path, name):
    path = write_case(name, tmp_path)
    with pytest.raises(EXC[str(G[f"{name}/raised"])]):
        la.load_log(path)


@pytest.mark.parametrize("name", [c for c in CASES if c != "tlog_no_mu"])
def test_oracle_fluence_matches_reference(logs, name):
    log = logs[name]
    for res, eq in MAP_SETTINGS:
        for kind in ("actual", "expected"):
            check_map(f"{name}/map/{kind}/{res}/{int(eq)}", log_oracle.fluence_of(getattr(log.fluence, kind), res, eq))


@pytest.mark.parametrize("name", [c for c in CASES if c.startswith("tlog")])
def test_oracle_subbeam_fluence_matches_reference(logs, name):
    for k, s in enumerate(logs[name].subbeams):
        for res, eq in SUBBEAM_SETTINGS:
            for kind in ("actual", "expected"):
                check_map(f"{name}/subbeam{k}/map/{kind}/{res}/{int(eq)}", log_oracle.fluence_of(getattr(s.fluence, kind), res, eq))


def test_log_fluence_is_exported_and_reports_no_device(tmp_path):
    import ctypes

    handle = ctypes.CDLL(nat.LIB_PATH)
    for sym in ("epid_log_fluence", "epid_hist_invert", "epid_gamma_stats"):
        assert hasattr(handle, sym)
    if nat.device_count() > 0:
        pytest.skip("a CUDA device is present")
    path = write_case("tlog_v21_millennium", tmp_path)
    log = la.load_log(path)
    with pytest.raises(nat.NoDeviceError):
        log.fluence.actual.calc_map(0.5)
    with pytest.raises(nat.NoDeviceError):
        la.analyze_batch([path])
