"""Light / radiation field coincidence throughput on the GPU: 512 seeded 1280 x 1280 uint16 FC-2 frames (half of them with fields just
under 100 mm, so every BB is near the field edge and goes through the adaptive histogram equalisation), device-resident.

Reports frames/s of ``planar_imaging.analyze_batch`` on the resident batch (host clock around calls that end in the stream sync),
the device time per kernel from torch.profiler in a separate run, and the card name and power limit read in the same run.

    python tools/bench_lightrad.py [--frames 512] [--iters 5] [--out results/bench_lightrad.json]
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


def frames(n: int, seed: int = 0):
    from tests.golden.lightrad_cases import lightrad_case

    near = lightrad_case("fc2_10_near")
    far = lightrad_case("fc2_10_far")
    rng = np.random.default_rng(seed)
    out = np.empty((n, 1280, 1280), np.uint16)
    for i in range(n):
        base = (near if i % 2 == 0 else far)["frame"].astype(np.int32)
        out[i] = np.clip(base + rng.integers(-20, 21, base.shape), 0, 65535)
    return out, near["dpmm"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from pylinac_b200 import _native as nat
    from pylinac_b200 import planar_imaging as pi

    if nat.device_count() == 0:
        raise SystemExit("bench_lightrad needs a CUDA device")
    f, dpmm = frames(a.frames)
    ctx = nat.Context.default()
    b = nat.Batch.upload(ctx, f)
    res = pi.analyze_batch(b, dpmm)                 # warm-up: module load, scratch allocation
    n_ok = sum(1 for r in res.rows if int(r["status"]) == 0)
    n_near = sum(1 for r in res.rows if int(r["near_edge_mask"]) != 0)
    times = []
    for _ in range(a.iters):
        t0 = time.perf_counter()
        pi.analyze_batch(b, dpmm)
        times.append(time.perf_counter() - t0)
    best = min(times)
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pi.analyze_batch(b, dpmm)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.count:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            kernels[ev.key[:80]] = round(t / 1000.0, 3)
    b.free()
    out = {"card": card(), "frames": a.frames, "frames_ok": n_ok, "frames_near_edge": n_near, "iters": a.iters,
           "seconds_per_batch": [round(t, 5) for t in times], "frames_per_s": round(a.frames / best, 1),
           "kernel_ms_one_batch": dict(sorted(kernels.items(), key=lambda kv: -kv[1])),
           "algorithmic_bytes_per_frame": {"raw_read": 1280 * 1280 * 2}}
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
