"""Machine-log throughput: fluence maps and fluence gamma of a batch of synthetic VMAT trajectory logs.

Workload: --logs trajectory logs (v3.0, Millennium MLC, 3000-6000 snapshots each, seeded) written to a temporary directory.
Prints one JSON line with, each number named for what it covers:
  * fluence_host_inputs_ms: the host half of a launch (descriptors, the reference's per-pair decisions, row bounds), built once
    and kept out of the timed windows below;
  * fluence_call_ms: wall time of the native epid_log_fluence call alone (H2D copy of the arena span, output memsets, kernel; the
    call returns after its stream synchronisation), median of --reps;
  * fluence_kernel_ms / fluence_h2d_ms: device time of k_log_fluence and of the host-to-device copies inside one such call, from the
    CUDA activity records of torch.profiler (device timestamps);
  * gamma_call_ms: wall time of the device gamma pipeline on the device-resident maps (epid_hist_invert, epid_ground,
    epid_normalize, epid_gamma, epid_gamma_stats; each call ends in its stream synchronisation), and gamma_device_ms: the device
    time of every kernel, memset and copy inside it;
  * e2e_ms: analyze_batch(paths) from the files (read into one page-locked arena, host parse and MLC statistics, H2D copy, fluence
    and gamma on the device, two numbers per log back);
  * the same fluence maps from the numpy oracle on one host core (a subset of logs, per log), for comparison;
  * the GPU name and power limit, read in the same run.
Writes nothing except its temporary directory (removed) unless --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import log_oracle  # noqa: E402
from pylinac_b200 import _native as nat  # noqa: E402
from pylinac_b200 import log_analyzer as la  # noqa: E402
from tests import log_writer as lw  # noqa: E402

RES = 0.1


def write_logs(directory: str, n: int, seed: int) -> list[str]:
    rng = np.random.default_rng(seed)
    paths = []
    for i in range(n):
        nsnap = int(rng.integers(3000, 6001))
        cols = lw.vmat_delivery(nsnap, seed + i, holds=int(rng.integers(0, 3)), jaw_y=float(rng.uniform(6, 12)))
        paths.append(lw.write_tlog(os.path.join(directory, f"P{i:04d}_arc.bin"), cols, version=3.0, subbeams=((0, "Arc 1"), (25, "Arc 2"))))
    return paths


def timed(fn, reps: int):
    """median wall time (ms) over `reps` calls of a function that returns after its stream synchronisation"""
    ts, out = [], None
    for _ in range(reps):
        if out is not None:
            release(out)
        t = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts)), ts, out


def release(out):
    for o in out if isinstance(out, tuple) else (out,):
        b = getattr(o, "batch", o)
        if hasattr(b, "free"):
            b.free()


def device_ms(fn, match):
    """device time (ms) of the CUDA activity inside one call of fn whose name satisfies match(name) -> (ms, result)"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
    tot = 0.0
    for ev in prof.key_averages():
        if match(ev.key):
            tot += getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)
    return tot / 1000.0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-logs", type=int, default=4, help="logs the host oracle computes (time per log)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if nat.device_count() == 0:
        raise SystemExit("bench_logs needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    ctx = nat.Context.default()
    with tempfile.TemporaryDirectory() as tmp:
        paths = write_logs(tmp, args.logs, 7000)
        logs = la._read_all(paths, True)
        items = [(lg.fluence, lg.fluence.actual._src()) for lg in logs]
        snaps = sum(len(lg.axis_data.mlc.snapshot_idx) for lg in logs)
        t = time.perf_counter()
        inp = la._fluence_inputs(items, RES, False, 3, True)
        host_ms = (time.perf_counter() - t) * 1e3
        release(inp.launch(ctx))                                    # warm-up: context, allocations, scratch
        fl_ms, fl_all, (a, e) = timed(lambda: inp.launch(ctx), args.reps)
        release((a, e))
        k_ms, (a, e) = device_ms(lambda: inp.launch(ctx), lambda k: "k_log_fluence" in k)
        release((a, e))
        h2d_ms, (a, e) = device_ms(lambda: inp.launch(ctx), lambda k: "Memcpy HtoD" in k)
        release(la._gamma_maps(a.batch, e.batch, 1, 1, 0.1, RES, ctx)[0])
        gm_ms, gm_all, (g, avg, pct) = timed(lambda: la._gamma_maps(a.batch, e.batch, 1, 1, 0.1, RES, ctx), args.reps)
        g.free()
        gdev_ms, (g, _, _) = device_ms(lambda: la._gamma_maps(a.batch, e.batch, 1, 1, 0.1, RES, ctx), lambda k: True)
        g.free()
        # correctness of the timed configuration: the first logs against the numpy oracle
        ha, he = a.host(), e.host()
        t = time.perf_counter()
        k = min(args.oracle_logs, len(logs))
        for i in range(k):
            assert np.array_equal(ha[i], log_oracle.fluence_of(logs[i].fluence.actual, RES))
            assert np.array_equal(he[i], log_oracle.fluence_of(logs[i].fluence.expected, RES))
        oracle_per_log_ms = (time.perf_counter() - t) * 1e3 / k
        release((a, e))
        e2e_ms, e2e_all, rows = timed(lambda: la.analyze_batch(paths), args.reps)
        assert all(r.pass_prcnt is not None for r in rows)
    n = args.logs
    W = int(400 / RES)
    steps = int(2 * 60 * W * snaps)
    result = {
        "gpu": gpu, "logs": n, "snapshots_total": snaps, "resolution_mm": RES, "map_shape": [60, W], "arena_bytes": int(inp.arena.nbytes),
        "fluence_host_inputs_ms": host_ms,
        "fluence_call_ms": fl_ms, "fluence_call_ms_all": fl_all, "fluence_call_logs_per_s": n / (fl_ms / 1e3),
        "fluence_kernel_ms": k_ms, "fluence_kernel_logs_per_s": n / (k_ms / 1e3), "fluence_kernel_steps_per_s_upper_bound": steps / (k_ms / 1e3),
        "fluence_h2d_ms": h2d_ms, "fluence_h2d_GB_per_s": inp.arena.nbytes / (h2d_ms / 1e3) / 1e9,
        "gamma_call_ms": gm_ms, "gamma_call_ms_all": gm_all, "gamma_device_ms": gdev_ms,
        "e2e_ms": e2e_ms, "e2e_ms_all": e2e_all, "e2e_logs_per_s": n / (e2e_ms / 1e3),
        "oracle_fluence_ms_per_log_one_core": oracle_per_log_ms,
        "pixel_snapshot_steps_if_every_pair_moves": steps,
    }
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
