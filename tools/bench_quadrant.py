"""pylinac_b200.nuclear.QuadrantResolution throughput (epid_disk_stats, csrc/roi.cu).

Workload: N device-resident seeded 1024 x 1024 uint16 four-quadrant bar frames, N = --frames (default 512), at the default geometry
(four disks of radius 70 px, 15 389 pixels each, 130 px from the centre).  Each number is named for what it covers:
  * disk_stats_ms: wall time of one epid_disk_stats call on the device batch for all 4N disks (the disk upload, k_disk_stats, the
    result download and the call's synchronisation), median of --reps;
  * batch_ms: one analyze_quadrant_resolution_batch call (the host bounds check, that device call and the per-frame result objects);
  * kernel_ms: device time of k_disk_stats in one call (torch.profiler CUDA activity, a run of its own, --profile);
  * pixel_bytes_mb: the disk pixels' compulsory bytes (2 per pixel), and hbm_bound_ms, that traffic at 3.35 TB/s: a computed floor.
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
from pylinac_b200 import nuclear  # noqa: E402
from tests.golden.quadrant_cases import WIDTHS, bars  # noqa: E402

SHAPE = (1024, 1024)
HBM_PEAK = 3.35e12


def wall_ms(fn, reps: int) -> float:
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
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
    ap.add_argument("--profile", action="store_true", help="torch.profiler kernel time (a run of its own)")
    args = ap.parse_args()
    distinct = np.concatenate([bars(900 + k, SHAPE, widths_px=(12, 9, 7, 5), high=700, low=300) for k in range(8)])
    frames = np.stack([distinct[k % len(distinct)] for k in range(args.frames)])
    out = {"gpu": gpu_info(), "frames": args.frames, "shape": list(SHAPE)}
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, frames) as b:
        res = nuclear.analyze_quadrant_resolution_batch(b, WIDTHS)
        centers = res[0].centers
        disks = np.array([(f, c.y, c.x, 70.0) for f in range(args.frames) for c in centers])
        npix = int(sum(r.counts[k] for r in res for k in range(len(centers))))
        out["disks"], out["pixel_bytes_mb"] = len(disks), 2.0 * npix / 1e6
        out["hbm_bound_ms"] = 2.0 * npix / HBM_PEAK * 1e3
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            nat.disk_stats(ctx, b, disks)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                nat.disk_stats(ctx, b, disks)
            out["kernel_ms"] = sum((getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)) / 1000.0
                                   for ev in prof.key_averages() if "k_disk_stats" in ev.key)
        else:
            out["disk_stats_ms"] = wall_ms(lambda: nat.disk_stats(ctx, b, disks), args.reps)
            out["batch_ms"] = wall_ms(lambda: nuclear.analyze_quadrant_resolution_batch(b, WIDTHS), args.reps)
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
