"""Generate tests/golden/log_golden.npz by running the UNMODIFIED reference's log analyzer (log_analyzer.py, stub-imported) on the
seeded logs of log_cases.py: headers, axis arrays, snapshot indices, subbeam snapshots, MLC statistics, treatment type, fluence maps
(sha1 + a subsample) at every MAP_SETTINGS entry, subbeam fluences, gamma maps / avg_gamma / pass_prcnt and the exception type of
every malformed file, plus each written file's sha1.

Run from the repository root, where oracle/refstub.py can import the unmodified reference:  python -m tests.golden.make_log_golden
"""
from __future__ import annotations

import glob
import hashlib
import json
import os
import sys
import tempfile
import warnings

import numpy as np

from oracle.refstub import import_reference
from tests.golden.log_cases import BAD_CASES, CASES, GAMMA_SETTINGS, MAP_SETTINGS, SUB_COLS, SUB_ROWS, SUBBEAM_SETTINGS, write_case


def sha1(b: bytes) -> np.ndarray:
    return np.frombuffer(hashlib.sha1(b).digest(), dtype=np.uint8)


def exc_name(e: BaseException) -> str:
    return f"{type(e).__module__}.{type(e).__qualname__}"


def store_map(store, key, a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    store[f"{key}/sha1"] = sha1(a.tobytes())
    store[f"{key}/shape"] = np.array(a.shape)
    store[f"{key}/sub"] = a[SUB_ROWS, SUB_COLS]


def main():
    warnings.simplefilter("ignore")
    import_reference()
    from pylinac import log_analyzer as R

    store = {}
    for name in CASES + BAD_CASES:
        d = tempfile.mkdtemp()
        path = write_case(name, d)
        for f in sorted(glob.glob(os.path.join(d, "*"))):
            store[f"{name}/file_sha1/{os.path.basename(f)}"] = sha1(open(f, "rb").read())
        try:
            log = R.load_log(path)
        except Exception as e:  # noqa: BLE001 -- the exception type is the golden
            store[f"{name}/raised"] = np.array(exc_name(e))
            print(name, "raised", exc_name(e), e)
            continue
        store[f"{name}/raised"] = np.array("")
        meta = {"treatment_type": log.treatment_type, "num_beamholds": log.num_beamholds, "has_fluence": hasattr(log, "fluence")}
        if isinstance(log, R.TrajectoryLog):
            h = log.header
            meta["header"] = {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in vars(h).items() if k != "metadata"}
            if hasattr(h, "metadata"):
                meta["metadata"] = dict(vars(h.metadata))
            meta["txt"] = log.txt
            meta["is_hdmlc"] = log.is_hdmlc
            meta["subbeams"] = [{"control_point": s.control_point, "mu_delivered": s.mu_delivered, "rad_time": s.rad_time,
                                 "sequence_num": s.sequence_num, "beam_name": s.beam_name,
                                 "gantry_angle": [float(s.gantry_angle.actual), float(s.gantry_angle.expected)]} for s in log.subbeams]
            for k, s in enumerate(log.subbeams):
                store[f"{name}/subbeam{k}/snapshots"] = np.asarray(s._snapshots, np.int64)
            ax = log.axis_data
            axes = {"collimator": ax.collimator, "gantry": ax.gantry, "x1": ax.jaws.x1, "x2": ax.jaws.x2, "y1": ax.jaws.y1,
                    "y2": ax.jaws.y2, "mu": ax.mu, "beam_hold": ax.beam_hold, "control_point": ax.control_point,
                    "couch_vert": ax.couch.vert, "carriage_A": ax.carriage_A}
            if ax.couch.pitch is not None:
                axes["couch_pitch"] = ax.couch.pitch
        else:
            h = log.header
            meta["header"] = {k: v for k, v in vars(h).items()}
            ax = log.axis_data
            meta["num_snapshots"] = int(ax.num_snapshots)
            axes = {"gantry": ax.gantry, "collimator": ax.collimator, "x1": ax.jaws.x1, "x2": ax.jaws.x2, "y1": ax.jaws.y1,
                    "y2": ax.jaws.y2, "mu": ax.mu, "beam_hold": ax.beam_hold, "beam_on": ax.beam_on, "carriage_A": ax.carriage_A}
        for k, a in axes.items():
            store[f"{name}/axis/{k}/actual"] = np.asarray(a.actual, np.float64)
            if a.expected is not None:
                store[f"{name}/axis/{k}/expected"] = np.asarray(a.expected, np.float64)
        mlc = ax.mlc
        store[f"{name}/snapshot_idx"] = np.asarray(mlc.snapshot_idx, np.int64)
        leaves = np.stack([mlc.leaf_axes[i].actual for i in range(1, mlc.num_leaves + 1)])
        store[f"{name}/leaves_actual_sha1"] = sha1(np.ascontiguousarray(leaves, np.float64).tobytes())
        store[f"{name}/leaf7"] = np.stack([mlc.leaf_axes[7].actual, mlc.leaf_axes[7].expected])
        store[f"{name}/moving_leaves"] = np.asarray(mlc.moving_leaves, np.int64)
        calls = {"rms_avg": lambda: mlc.get_RMS_avg(), "rms_avg_moving": lambda: mlc.get_RMS_avg(only_moving_leaves=True),
                 "rms_max": lambda: mlc.get_RMS_max(), "rms_max_a": lambda: mlc.get_RMS_max("A"),
                 "rms_p95": lambda: mlc.get_RMS_percentile(95), "err_p95": lambda: mlc.get_error_percentile(95),
                 "err_p50_b": lambda: mlc.get_error_percentile(50, "B"),
                 "err_p95_moving": lambda: mlc.get_error_percentile(95, only_moving_leaves=True)}
        stats = {}
        for k, fn in calls.items():
            try:
                stats[k] = float(fn())
            except Exception as e:  # noqa: BLE001 -- e.g. an empty moving-leaf list indexes with floats
                stats[k] = np.nan
                meta.setdefault("stats_raised", {})[k] = exc_name(e)
        store[f"{name}/stats"] = np.array(list(stats.values()))
        meta["stats_keys"] = list(stats)
        store[f"{name}/rms"] = np.asarray(mlc.get_RMS("both"), np.float64)
        store[f"{name}/under_y_jaw"] = np.array([mlc.leaf_under_y_jaw(p) for p in range(1, mlc.num_pairs + 1)])
        store[f"{name}/meta"] = np.array(json.dumps(meta, default=lambda v: v.item() if hasattr(v, "item") else str(v)))
        if hasattr(log, "fluence"):
            for res, eq in MAP_SETTINGS:
                for kind in ("actual", "expected"):
                    fl = getattr(log.fluence, kind)
                    fl.calc_map.cache_clear() if hasattr(fl.calc_map, "cache_clear") else None
                    store_map(store, f"{name}/map/{kind}/{res}/{int(eq)}", fl.calc_map(res, eq))
            for k, setting in enumerate(GAMMA_SETTINGS):
                doseTA, distTA, threshold, res = setting
                # the reference reuses a map already computed at this resolution: start from the non-equal-aspect maps
                log.fluence.actual.calc_map(res, False)
                log.fluence.expected.calc_map(res, False)
                g = log.fluence.gamma.calc_map(doseTA, distTA, threshold, res)
                store_map(store, f"{name}/gamma{k}", g)
                store[f"{name}/gamma{k}/avg_pct"] = np.array([float(log.fluence.gamma.avg_gamma), float(log.fluence.gamma.pass_prcnt)])
                store[f"{name}/gamma{k}/histogram"] = log.fluence.gamma.histogram()[0]
        if isinstance(log, R.TrajectoryLog):
            for k, s in enumerate(log.subbeams):
                for res, eq in SUBBEAM_SETTINGS:
                    store_map(store, f"{name}/subbeam{k}/map/actual/{res}/{int(eq)}", s.fluence.actual.calc_map(res, eq))
                    store_map(store, f"{name}/subbeam{k}/map/expected/{res}/{int(eq)}", s.fluence.expected.calc_map(res, eq))
        print(name, "ok")
    np.savez_compressed("tests/golden/log_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
