"""pylinac_b200.nuclear.TomographicUniformity throughput (csrc/nuclear_tu.cu).

Workload: N device-resident seeded 64 x 128 x 128 uint16 Jaszczak-like volumes at 4.4 mm (bin 2: 64 x 64 binned frames), N = --volumes
(default 64), the slab of slices 6 .. 57 (52 slices).  Each number is named for what it covers:
  * uniformity_ms: wall time of one epid_tu_uniformity call on the device batch (k_tu_bin + k_tu_frame, the row download and the call's
    synchronisation), median of --reps, without the mean / cleaned / mask planes;
  * call_ms: one analyze_tomographic_uniformity_batch call with those planes kept on the device;
  * kernel_ms: device time of each kernel in one call (torch.profiler CUDA activity, a run of its own);
  * hbm_bound_ms: the least time k_tu_bin's compulsory traffic (2 bytes per slab voxel) takes at 3.35 TB/s, a computed floor, and
    bin_hbm_share = hbm_bound_ms / kernel_ms["k_tu_bin"].
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
FIRST, LAST = 6, 58
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


def volumes(n: int) -> np.ndarray:
    distinct = np.stack([jaszczak(700 + k, shape=SHAPE, z_extent=(4, 60)) for k in range(min(n, 8))])
    return np.stack([distinct[k % len(distinct)] for k in range(n)])


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--volumes", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", action="store_true", help="torch.profiler kernel times (a run of its own)")
    args = ap.parse_args()
    vols = volumes(args.volumes)
    nz = SHAPE[0]
    out = {"gpu": gpu_info(), "volumes": args.volumes, "shape": list(SHAPE), "slab": [FIRST, LAST]}
    out["hbm_bound_ms"] = 2.0 * args.volumes * (LAST - FIRST) * SHAPE[1] * SHAPE[2] / HBM_PEAK * 1e3
    ctx = nat.Context.default()
    erode = (1 - 0.8, 1 - 0.75 * 0.8, 1 - 0.4 * 0.8)
    with nat.Batch.upload(ctx, vols.reshape(-1, *SHAPE[1:])) as b:
        run = lambda: nuclear.analyze_tomographic_uniformity_batch(b, 4.4, FIRST, LAST, slices_per_volume=nz)  # noqa: E731
        for r in run():
            r.raise_for_status()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
            ks = {"k_tu_bin": 0.0, "k_tu_frame": 0.0}
            for ev in prof.key_averages():
                for k in ks:
                    if k + "(" in ev.key or ev.key.endswith(k) or k + "<" in ev.key:
                        ks[k] += (getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)) / 1000.0
            out["kernel_ms"] = ks
            if ks["k_tu_bin"] > 0:
                out["bin_hbm_share"] = out["hbm_bound_ms"] / ks["k_tu_bin"]
        else:
            out["uniformity_ms"] = wall_ms(lambda: nat.tu_uniformity(ctx, b, nz, FIRST, LAST - FIRST, 2, erode, 5, 0.75, arrays=False),
                                           args.reps)
            out["call_ms"] = wall_ms(run, args.reps)
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
