"""gamma_2d throughput: device-resident batches of (reference, evaluation) pairs through epid_gamma2d.

Workload: --pairs float64 pairs per batch at each --sizes (square frames), DTA in --dtas, global and local dose, 1 % dose to agreement,
5 % threshold, cap 2, NaN fill.  Two kinds of pair: "agree" (a smooth, broad field; the evaluation is the reference times
1 + N(0, 0.2 %)) and "shifted" (the evaluation is the field moved by (2, 3) pixels and scaled by 1.01).
Per configuration, each number named for what it covers:
  * call_ms: wall time of one epid_gamma2d call on the device-resident batch (per-pair max, normalisation, search; the call returns
    after its stream synchronisation), median of --reps; full_call_ms the same with the early exit disabled;
  * kernel_ms / full_kernel_ms: device time of the search kernel k_gamma2d alone in one such call (torch.profiler CUDA activity);
  * evaluated: pixels above the threshold (epid_gamma_stats count); disk: offsets in the disk;
  * visited_mean: offsets the early exit visits per evaluated pixel, counted by the numpy oracle (oracle/gamma2d_oracle.py) on a
    centred --crop x --crop window of the first pair;
  * full_fp64_tflops: 4 fp64 operations (difference, square, sum, min) per term over full_kernel_ms, where the term count is exact
    (evaluated x disk); min_bytes_ms: the least time the call's compulsory traffic (read both frames and write the map, 24 B per
    pixel) takes at 3.35 TB/s;
  * e2e: gamma_2d of one 1024 x 1024 numpy pair, and gamma_2d_batch of --pairs numpy pairs at 1024 x 1024 (upload, compute,
    download), DTA 3, global, "agree".
The GPU name and power limit are read in the same run.  --reference instead times the reference's own loop on the host (a 256 x 256
crop, the reference checkout imported through oracle/refstub.py) and prints the per-megapixel figure as an extrapolation.
"""
from __future__ import annotations

import argparse
import json
import os
import platform
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gamma2d_oracle  # noqa: E402
from pylinac_b200 import _native as nat  # noqa: E402
from pylinac_b200.core import gamma as G  # noqa: E402

FP64_PEAK = 34e12        # H100 SXM data sheet, FP64 without tensor cores (the kernel uses none)
HBM_PEAK = 3.35e12
OPS_PER_TERM = 4


def make_pairs(n: int, size: int, kind: str, seed: int = 0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float64)
    c = (size - 1) / 2

    def field(dy=0.0, dx=0.0):
        r2 = ((yy - c - dy) / (0.35 * size)) ** 2 + ((xx - c - dx) / (0.3 * size)) ** 2
        return 1000.0 * np.exp(-r2 ** 3) + 300.0 * np.exp(-r2) + 10.0

    base = field()
    ev_base = field(2.0, 3.0) * 1.01 if kind == "shifted" else base
    noise = rng.normal(0, 0.002, (size, size))
    refs = np.empty((n, size, size))
    evs = np.empty((n, size, size))
    for k in range(n):
        s = 1.0 + 0.01 * k / n
        refs[k] = base * s
        evs[k] = ev_base * s * (1.0 + np.roll(noise, (7 * k, 13 * k), axis=(0, 1)))
    return refs, evs


def median_ms(fn, reps: int) -> float:
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def kernel_ms(fn) -> float:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    tot = 0.0
    for ev in prof.key_averages():
        if "k_gamma2d<" in ev.key:
            tot += getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)
    return tot / 1000.0


def reference_timing():
    from oracle import skimage_draw
    from oracle.refstub import import_reference

    import_reference()
    import pylinac.core.gamma as rgamma

    rgamma.disk = skimage_draw.disk
    refs, evs = make_pairs(1, 1024, "agree")
    sl = slice(384, 640)
    out = {"host": platform.processor() or platform.machine(), "crop": [256, 256]}
    for dta in (1, 3, 10):
        t = time.perf_counter()
        rgamma.gamma_2d(refs[0][sl, sl], evs[0][sl, sl], distance_to_agreement=dta)
        s = time.perf_counter() - t
        out[f"dta{dta}_s_per_crop"] = round(s, 3)
        out[f"dta{dta}_s_per_megapixel_extrapolated"] = round(s * 1e6 / 256 ** 2, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--sizes", default="1024,1280")
    ap.add_argument("--dtas", default="1,3,10,20")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--crop", type=int, default=160)
    ap.add_argument("--reference", action="store_true", help="time the reference's loop on the host instead (no GPU)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.reference:
        res = {"reference_host": reference_timing()}
    else:
        if nat.device_count() == 0:
            raise SystemExit("bench_gamma2d needs a CUDA device")
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        ctx = nat.Context.default()
        rows = []
        for size in (int(s) for s in args.sizes.split(",")):
            for kind in ("agree", "shifted"):
                refs, evs = make_pairs(args.pairs, size, kind)
                lo = (size - args.crop) // 2
                crop = slice(lo, lo + args.crop)
                with nat.Batch.upload(ctx, refs) as rb, nat.Batch.upload(ctx, evs) as eb:
                    for dta in (int(d) for d in args.dtas.split(",")):
                        for global_dose in (True, False):
                            kw = dict(distance_to_agreement=dta, global_dose=global_dose)

                            def call(full=False):
                                G.gamma_2d_batch(rb, eb, **kw, device=True, full_search=full, ctx=ctx).free()

                            call()
                            maps, st = G.gamma_2d_batch(rb, eb, **kw, device=True, stats=True, ctx=ctx)
                            maps.free()
                            evaluated = int(st["evaluated"].sum())
                            disk = len(G._disk_offsets(dta)[0])
                            row = dict(size=size, kind=kind, dta=dta, mode="global" if global_dose else "local", evaluated=evaluated,
                                       disk=disk, call_ms=median_ms(call, args.reps), kernel_ms=kernel_ms(call))
                            row["full_call_ms"] = median_ms(lambda: call(True), args.reps)
                            row["full_kernel_ms"] = kernel_ms(lambda: call(True))
                            visited, _ = gamma2d_oracle.offsets_visited(refs[0][crop, crop], evs[0][crop, crop], **kw)
                            row["visited_mean"] = float(visited[visited > 0].mean())
                            row["full_fp64_tflops"] = OPS_PER_TERM * evaluated * disk / (row["full_kernel_ms"] * 1e-3) / 1e12
                            row["min_bytes_ms"] = 24 * args.pairs * size * size / HBM_PEAK * 1e3
                            rows.append({k: (round(v, 3) if isinstance(v, float) else v) for k, v in row.items()})
                            print(json.dumps(rows[-1]), flush=True)
        refs, evs = make_pairs(args.pairs, 1024, "agree")
        G.gamma_2d(refs[0], evs[0], distance_to_agreement=3)
        e2e = {"gamma_2d_1024_ms": median_ms(lambda: G.gamma_2d(refs[0], evs[0], distance_to_agreement=3), args.reps),
               "gamma_2d_batch_1024_ms": median_ms(lambda: G.gamma_2d_batch(refs, evs, distance_to_agreement=3), args.reps)}
        res = {"gpu": gpu, "pairs": args.pairs, "reps": args.reps, "fp64_peak_tflops": FP64_PEAK / 1e12, "configs": rows, "e2e": e2e}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
