"""pylinac_b200.nuclear.TomographicContrast throughput (csrc/nuclear_tomo.cu).

Workload: N device-resident seeded 64 x 128 x 128 uint16 Jaszczak-like volumes at 4.4 mm with six cold spheres (the reference's default
diameters and angles), N = --volumes (default 64).  Each number is named for what it covers:
  * slices_ms: wall time of one epid_nt_slices call on the device batch (k_nt_max + k_nt_slices, the row download and the call's
    synchronisation), median of --reps;
  * spheres_ms: the same for one epid_nt_spheres call with every sphere of every volume (k_nt_spheres, 6 N CTAs);
  * call_ms: one analyze_tomographic_contrast_batch call (both device calls and the host selection);
  * kernel_ms: device time of each kernel in one call (torch.profiler CUDA activity, a run of its own);
  * evals_per_sphere: Nelder-Mead objective evaluations (nfev) per sphere, mean and max;
  * oracle_s_per_volume / reference_s_per_volume (--cpu): one volume through oracle/tomo_contrast_oracle.py and, where the reference
    is importable, through the unmodified reference, on one CPU core.
The GPU name and power limit are read in the same run.
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
from tests.golden.tomo_contrast_cases import jaszczak  # noqa: E402

SHAPE = (64, 128, 128)
DIAMETERS = (38, 31.8, 25.4, 19.1, 15.9, 12.7)
ANGLES = (-10, -70, -130, -190, 110, 50)


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


def volumes(n: int) -> np.ndarray:
    distinct = np.stack([jaszczak(500 + k, shape=SHAPE, z_extent=(8, 56)) for k in range(min(n, 8))])
    return np.stack([distinct[k % len(distinct)] for k in range(n)])


def cpu_times(vol: np.ndarray) -> dict:
    from oracle import tomo_contrast_oracle as O

    t = time.perf_counter()
    O.analyze(vol, 4.4)
    out = {"oracle_s_per_volume": time.perf_counter() - t}
    try:
        import warnings

        from oracle import skimage_tomo
        from tests.golden.make_nuclear_golden import reference_files

        rn = skimage_tomo.install()
        with reference_files(vol, 4.4):
            tc = rn.TomographicContrast("bench.dcm")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            t = time.perf_counter()
            tc.analyze()
            out["reference_s_per_volume"] = time.perf_counter() - t
    except Exception as e:  # noqa: BLE001 -- the reference is optional
        out["reference_s_per_volume"] = f"not measured: {type(e).__name__}: {e}"
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--volumes", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", action="store_true", help="torch.profiler kernel times (a run of its own)")
    ap.add_argument("--cpu", action="store_true", help="also time one volume through the oracle and the reference on the CPU")
    args = ap.parse_args()
    vols = volumes(args.volumes)
    out = {"gpu": gpu_info(), "volumes": args.volumes, "shape": list(SHAPE)}
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, vols.reshape(-1, *SHAPE[1:])) as b:
        nz = SHAPE[0]
        res = nuclear.analyze_tomographic_contrast_batch(b, 4.4, slices_per_volume=nz)
        for r in res:
            r.raise_for_status()
        inp, _ = nuclear._sphere_inputs(res, 4.4, DIAMETERS, ANGLES, 5, 3)
        searches = np.concatenate([r.searches for r in res])
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                nuclear.analyze_tomographic_contrast_batch(b, 4.4, slices_per_volume=nz)
            ks = {"k_nt_max": 0.0, "k_nt_slices": 0.0, "k_nt_spheres": 0.0}
            for ev in prof.key_averages():
                for k in ks:
                    if k + "(" in ev.key or ev.key.endswith(k) or k + "<" in ev.key:
                        ks[k] += (getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)) / 1000.0
            out["kernel_ms"] = ks
        else:
            out["slices_ms"] = wall_ms(lambda: nat.nt_slices(ctx, b, nz, 1 - 0.8), args.reps)
            out["spheres_ms"] = wall_ms(lambda: nat.nt_spheres(ctx, b, nz, inp), args.reps)
            out["call_ms"] = wall_ms(lambda: nuclear.analyze_tomographic_contrast_batch(b, 4.4, slices_per_volume=nz), args.reps)
        nfev = searches["nfev"].astype(np.int64)
        out["spheres"] = len(nfev)
        out["evals_per_sphere"] = {"mean": float(nfev.mean()), "max": int(nfev.max())}
    if args.cpu:
        out.update(cpu_times(vols[0]))
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
