"""Exact frame statistics and frame histograms on the GPU.

Workloads (uint16 frames, device-resident before timing):
  * stats_64x1024x4096: epid_frame_stats on 64 frames of 1024 x 4096 (min / max / sum, row and column sums, p0.5 / p50 / p99.5).
    Views wider than 2040 columns are the ones k_hist_view cuts into column strips.
  * hist_512x1024x1024: epid_frame_histogram on 512 frames of 1024 x 1024.
  * hist_512x1024x1024_uniform: the same on uniformly random pixels, where the shared-memory bin cache hits least.
The first two use PicketFence benchmark frames (oracle.synth), four side by side for the 4096-column frames.

For each workload one JSON line:
  * call_ms: median and minimum over --iters calls of the whole entry point, between CUDA events, after --warmup calls.  The call
    includes the copy of its results to the host (for a histogram, 256 KB per frame into pageable memory);
  * device_us: device time of one call by kernel, memset and copy (torch.profiler CUDA activity records over --prof-iters calls,
    after the timed ones), and their total;
  * digest: a hash of the results, equal for two builds that compute the same numbers;
  * the GPU name and power limit, read in the same run, and the library measured (EPID_LIB selects another build).
Writes nothing.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from pylinac_b200 import _native as nat  # noqa: E402


def workloads():
    pf = synth.bench_pf_batch(16, unique=16)
    wide = np.concatenate([pf[0:4], pf[4:8], pf[8:12], pf[12:16]], axis=2)             # 4 x 1024 x 4096
    stats_frames = np.stack([wide[i % 4] + np.uint16(i // 4) for i in range(64)])
    hist_frames = np.stack([pf[i % 16] + np.uint16(i // 16) for i in range(512)])
    uniform = np.random.default_rng(0).integers(0, 65536, (512, 1024, 1024), dtype=np.uint16)
    qs = (0.5, 50, 99.5)
    return [("stats_64x1024x4096", stats_frames, lambda ctx, b: nat.frame_stats(ctx, b, percentiles=qs)),
            ("hist_512x1024x1024", hist_frames, lambda ctx, b: nat.frame_histogram(ctx, b)),
            ("hist_512x1024x1024_uniform", uniform, lambda ctx, b: nat.frame_histogram(ctx, b))]


def digest(out) -> str:
    h = hashlib.sha256()
    for a in (out.values() if isinstance(out, dict) else [out]):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def gpu_info():
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
        return dict(zip(("gpu", "power_limit"), [s.strip() for s in line.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"gpu": None, "power_limit": None}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--prof-iters", type=int, default=5)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    assert nat.device_count() > 0, "bench_stats needs a CUDA device"
    ctx = nat.Context.default()
    info = gpu_info()
    for name, frames, fn in workloads():
        b = nat.Batch.upload(ctx, frames)
        try:
            for _ in range(args.warmup):
                out = fn(ctx, b)
            ts = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(ctx, b)            # returns after its stream has finished
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.prof_iters):
                    fn(ctx, b)
            dev = {}
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA:       # kernels, memsets and copies of the calls
                    key = ev.key.split("(")[0].replace("void ", "").replace("epid::", "").strip()
                    dev[key] = dev.get(key, 0.0) + ev.device_time_total / args.prof_iters
        finally:
            b.free()
        print(json.dumps({"workload": name, "call_ms": {"median": round(float(np.median(ts)), 3), "min": round(float(np.min(ts)), 3)},
                          "device_us": {"total": round(sum(dev.values()), 1), **{k: round(v, 1) for k, v in sorted(dev.items())}},
                          "digest": digest(out), "lib": os.path.relpath(nat.LIB_PATH, ROOT), **info}), flush=True)


if __name__ == "__main__":
    main()
