"""core.roi.analyze_low_contrast_batch throughput (epid_disk_stats and epid_disk_percentiles, csrc/roi.cu).

Workload: N device-resident seeded 1024 x 1024 uint16 frames, N = --frames (default 512), each with a Leeds-like set of 18
low-contrast disks and 2 background disks (radius 18 px, about 1 000 pixels each) at a fixed phantom geometry: the daily-QA case.
Each number is named for what it covers:
  * disk_stats_ms / disk_percentiles_ms: one call on the device batch for all 20N / 18N disks (disk upload, kernel, result download,
    the call's synchronisation and its host work), timed by CUDA events recorded on either side of it; the call returns only after
    its stream has finished.  Median of --reps;
  * disk_stats_device_ms / disk_percentiles_device_ms: the device time inside one call, its kernel and copies (torch.profiler CUDA
    activity, a pass of its own after the timed ones), and k_disk_stats_ms / k_disk_percentiles_ms, the kernels alone;
  * batch_ms: one analyze_low_contrast_batch call end to end (geometry, bounds checks, both device calls, the per-disk numpy
    arithmetic and the per-frame results), timed the same way; batch_host_top: the functions of one batch call with the most own
    time under cProfile (which slows the host, so only their shares mean something).
The GPU name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pylinac_b200 import _native as nat  # noqa: E402
from pylinac_b200.core import roi  # noqa: E402
from tests.golden.lowcontrast_cases import LEEDS_BG, LEEDS_LIKE, phantom  # noqa: E402

SHAPE = (1024, 1024)
CENTER, RADIUS = (512.3, 511.7), 400.0


def event_ms(fn, reps: int) -> float:
    import torch

    fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    distinct = phantom(7, n=8, shape=SHAPE, center=CENTER, radius=RADIUS)
    frames = np.stack([distinct[k % len(distinct)] for k in range(args.frames)])
    out = {"gpu": gpu_info(), "frames": args.frames, "shape": list(SHAPE)}
    ctx = nat.Context.default()

    def run(b):
        return roi.analyze_low_contrast_batch(b, CENTER, 0.0, RADIUS, LEEDS_LIKE, LEEDS_BG)

    with nat.Batch.upload(ctx, frames) as b:
        res = run(b)
        lc = [(f, c.y, c.x, r) for f in range(args.frames) for c, r in zip(res[f].centers, res[f].radii)]
        bg = []
        for f in range(args.frames):
            for s in LEEDS_BG.values():
                p = roi.DiskROI._get_shifted_center(s["angle"], RADIUS * s["distance from center"], roi.Point(*CENTER))
                bg.append((f, p.y, p.x, RADIUS * s["roi radius"]))
        out["disks"] = len(lc) + len(bg)
        out["disk_stats_ms"] = event_ms(lambda: nat.disk_stats(ctx, b, bg + lc), args.reps)
        out["disk_percentiles_ms"] = event_ms(lambda: nat.disk_percentiles(ctx, b, lc, (1, 99)), args.reps)
        out["batch_ms"] = event_ms(lambda: run(b), args.reps)
        out["piu_frame0"] = res[0].piu
        import cProfile
        import pstats

        import torch
        from torch.profiler import ProfilerActivity, profile

        pr = cProfile.Profile()
        pr.runcall(run, b)
        st = pstats.Stats(pr)
        total = sum(v[2] for v in st.stats.values())
        top = sorted(st.stats.items(), key=lambda kv: -kv[1][2])[:6]
        out["batch_host_top"] = [[f"{os.path.basename(k[0])}:{k[2]}", round(v[2] / total, 3)] for k, v in top]

        for name, fn in (("disk_stats", lambda: nat.disk_stats(ctx, b, bg + lc)),
                         ("disk_percentiles", lambda: nat.disk_percentiles(ctx, b, lc, (1, 99)))):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
            dev = [ev for ev in prof.key_averages() if ev.device_type == torch.autograd.DeviceType.CUDA]
            out[name + "_device_ms"] = sum(ev.device_time_total for ev in dev) / 1000.0
            out["k_" + name + "_ms"] = sum(ev.device_time_total for ev in dev if "k_" + name in ev.key) / 1000.0
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
