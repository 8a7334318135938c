"""pylinac_b200.nuclear throughput: PlanarUniformity's frame pipeline (csrc/nuclear.cu) and MaxCountRate's frame sums.

Workloads:
  * "1024_bin8": 512 device-resident 1024 x 1024 uint16 floods at 0.6 mm (bin 8 -> 128 x 128 binned frames);
  * "256_bin2": 512 device-resident 256 x 256 uint16 floods at 2.4 mm (bin 2 -> 128 x 128).
Each batch holds 8 distinct seeded Poisson floods (circular field, a hot spot, a gradient) repeated to 512 frames.
Per workload, each number named for what it covers:
  * call_ms: wall time of one analyze_batch call on the device batch (kernels, result download and the call's stream synchronisation),
    median of --reps, with the cleaned frames and masks kept on the device (arrays) and without them (no_arrays);
  * bin_kernel_ms / frame_kernel_ms: device time of k_nm_bin (the streaming stage) and of k_nm_frame (every per-frame stage) in one
    call (torch.profiler CUDA activity, a run of its own);
  * hbm_bound_ms: the least time the streaming stage's compulsory traffic (2 bytes per raw pixel) takes at 3.35 TB/s, and
    bin_hbm_share = hbm_bound_ms / bin_kernel_ms.
MaxCountRate: frame_sums of a 2000-frame 128 x 128 uint16 stack from host memory (upload + epid_frame_stats), and MaxCountRate.analyze
on the same stack read from an NM file (the read is outside the timed call).
The GPU name and power limit are read in the same run.
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

from pylinac_b200 import _native as nat  # noqa: E402
from pylinac_b200 import nuclear  # noqa: E402
from tests.golden.nuclear_cases import flood  # noqa: E402
from tests.nm_writer import write_nm  # noqa: E402

HBM_PEAK = 3.35e12


def wall_ms(fn, reps: int) -> float:
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def kernel_ms(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    out = {"k_nm_bin": 0.0, "k_nm_frame": 0.0}
    for ev in prof.key_averages():
        for k in out:
            if k + "<" in ev.key:
                out[k] += (getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)) / 1000.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if nat.device_count() == 0:
        raise SystemExit("bench_nuclear needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    ctx = nat.Context.default()
    res = {"gpu": gpu, "frames": args.frames, "workloads": {}}
    for name, size, pixel in (("1024_bin8", 1024, 0.6), ("256_bin2", 256, 2.4)):
        distinct = np.stack([flood(k, (size, size), counts=40.0 * (1024 // size) ** 2 / 16, spots=[(0.4, 0.6, 0.05, 1.3)],
                                   gradient=0.1) for k in range(8)])
        frames = np.ascontiguousarray(np.resize(distinct, (args.frames, size, size)))
        with nat.Batch.upload(ctx, frames) as b:
            with_arrays = wall_ms(lambda: nuclear.analyze_batch(b, pixel), args.reps)
            no_arrays = wall_ms(lambda: nuclear.analyze_batch(b, pixel, arrays=False), args.reps)
            ks = kernel_ms(lambda: nuclear.analyze_batch(b, pixel, arrays=False))
            rows = nuclear.analyze_batch(b, pixel, arrays=False).rows
        bound = frames.size * 2 / HBM_PEAK * 1e3
        res["workloads"][name] = {
            "call_ms_arrays": round(with_arrays, 3), "call_ms_no_arrays": round(no_arrays, 3),
            "bin_kernel_ms": round(ks["k_nm_bin"], 4), "frame_kernel_ms": round(ks["k_nm_frame"], 4),
            "hbm_bound_ms": round(bound, 4), "bin_hbm_share": round(bound / ks["k_nm_bin"], 3) if ks["k_nm_bin"] else None,
            "binned_shape": [-(-size // nuclear.determine_binning(pixel))] * 2, "frames_ok": int((rows["status"] == nat.NM_OK).sum()),
        }
        print(name, res["workloads"][name], flush=True)
    rng = np.random.default_rng(7)
    stack = rng.poisson(rng.uniform(10, 400, size=(2000, 1, 1)), size=(2000, 128, 128)).astype(np.uint16)
    res["max_count_rate"] = {"frame_sums_ms": round(wall_ms(lambda: nuclear.frame_sums(stack), args.reps), 3)}
    with tempfile.TemporaryDirectory() as d:
        mcr = nuclear.MaxCountRate(write_nm(os.path.join(d, "dynamic.dcm"), stack))
        res["max_count_rate"]["analyze_ms"] = round(wall_ms(lambda: mcr.analyze(frame_duration=0.5), args.reps), 3)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
