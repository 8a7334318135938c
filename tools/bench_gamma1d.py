"""gamma_geometric / gamma_1d throughput: batches of profile pairs through one device call each.

Workload: --pairs pairs of physical profiles per batch at 0.1 mm per sample, --sizes samples per profile (1201 and 4096: a 12 cm and
a 41 cm profile), criteria 1 %/1 mm, 2 %/2 mm and 3 %/3 mm, threshold 5 %, cap 2, global dose; the evaluation is the reference field
moved by 0.3 mm and scaled by 1.01, both with N(0, 0.2 %) noise.  Per configuration:
  * call_ms: host clock around one gamma_*_batch call from numpy (argument checks, O(n) preparation, packing, upload, kernel,
    download, result arrays; the call returns after its stream synchronisation), median of --reps after a warm-up call;
    native_ms the same around the _native call alone on pre-packed arrays;
  * kernel_ms: device time of k_gamma_geometric / k_gamma1d in one call (torch.profiler CUDA activity, --profile, a separate run);
  * points: evaluated reference points; work: window segments (gamma_geometric, counted from the window indices) or samples
    (gamma_1d: points x int(DTA * 3 * 2 + 1)); work_per_s: work over kernel_ms.
The GPU name and power limit are read in the same run.  --reference instead times the reference's own functions on the host, one
pair per configuration (the reference checkout imported through oracle/refstub.py); that needs no GPU.
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
from pylinac_b200.core import gamma as G  # noqa: E402

CRITERIA = [(1, 1), (2, 2), (3, 3)]


def make_pairs(n: int, size: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    x = (np.arange(size) - (size - 1) / 2) * 0.1
    width = 0.6 * (x.max() - x.min())

    def field(c):
        return 200 + 800 / (1 + np.exp(-(x - c + width / 2) / 1.5)) / (1 + np.exp((x - c - width / 2) / 1.5))

    ref, ev = field(0.0), field(0.3) * 1.01
    refs = [ref * (1 + rng.normal(0, 0.002, size)) for _ in range(n)]
    evs = [ev * (1 + rng.normal(0, 0.002, size)) for _ in range(n)]
    return refs, evs, [x] * n, [x] * n


def segments(ref, ev, x, dose, dta):
    """segments of gamma_geometric's windows, from the window indices (np.searchsorted; ties counted either way)"""
    mask = ~(ref * 100 / (ref.max() * dose) < 5 / dose)
    nx = x / dta
    t = nx[mask]

    def near(v):
        i = np.clip(np.searchsorted(nx, v), 1, len(nx) - 1)
        return np.where(np.abs(nx[i - 1] - v) <= np.abs(nx[i] - v), i - 1, i)

    left = np.maximum(near(t - dta) - 1, 0)
    right = np.minimum(near(t + dta) + 1, len(nx) - 1)
    return int(mask.sum()), int((right - left).sum())


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": f"unknown ({e})"}


def timed(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def packed_call(fn, refs, evs, xs, dose, dta):
    """the _native call of one batch on arrays packed beforehand (what gamma_*_batch hands it)"""
    ctx = nat.Context.default()
    if fn == "geometric":
        preps = [G._prepare_geometric(r, e, x, x, dose, dta, 5) for r, e, x in zip(refs, evs, xs)]
        args = (G._offsets([len(p[1]) for p in preps]), G._offsets([len(p[4]) for p in preps]), [p[3] for p in preps],
                np.concatenate([p[1] for p in preps]), np.concatenate([p[2] for p in preps]), np.concatenate([p[4] for p in preps]),
                np.concatenate([p[5] for p in preps]), float(dta), 2.0)
        return lambda: nat.gamma_geometric(ctx, *args)
    num = int(dta * 3 * 2 + 1)
    preps = [G._prepare_1d(r, e, x, x, dose, dta, True, 5, 3, num) for r, e, x in zip(refs, evs, xs)]
    args = (G._offsets([len(p[1]) for p in preps]), G._offsets([len(p[3]) for p in preps]), [p[6] for p in preps],
            np.concatenate([p[1] for p in preps]), np.concatenate([p[2] for p in preps]), np.concatenate([p[3] for p in preps]),
            np.concatenate([p[4] for p in preps]), np.concatenate([p[5] for p in preps]), float(dta), float(dta ** 2), num, 2.0)
    return lambda: nat.gamma1d(ctx, *args)


def kernel_ms(call) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile

    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.name.find("k_gamma") >= 0 and e.device_type.name == "CUDA":
            key = "k_gamma_geometric" if "geometric" in e.name else "k_gamma1d"
            out[key] = out.get(key, 0.0) + e.device_time / 1e3
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1201, 4096])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="kernel times from torch.profiler (run separately from the timings)")
    ap.add_argument("--reference", action="store_true", help="time the reference's functions on the host, one pair each")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = []
    if a.reference:
        from oracle.refstub import import_reference

        import_reference()
        import pylinac.core.gamma as rgamma
        import platform

        for size in a.sizes:
            refs, evs, xs, _ = make_pairs(1, size)
            for dose, dta in CRITERIA:
                for fn, f in (("geometric", rgamma.gamma_geometric), ("1d", rgamma.gamma_1d)):
                    t0 = time.perf_counter()
                    f(refs[0], evs[0], xs[0], xs[0], dose_to_agreement=dose, distance_to_agreement=dta)
                    rows.append(dict(function=fn, size=size, criteria=f"{dose}%/{dta}mm", reference_s_per_pair=time.perf_counter() - t0,
                                     host=platform.processor() or platform.machine()))
                    print(json.dumps(rows[-1]), flush=True)
    else:
        info = gpu_info()
        for size in a.sizes:
            refs, evs, xs, _ = make_pairs(a.pairs, size)
            for dose, dta in CRITERIA:
                pts, segs = segments(refs[0], evs[0], xs[0], dose, dta)
                for fn in ("geometric", "1d"):
                    batch = G.gamma_geometric_batch if fn == "geometric" else G.gamma_1d_batch
                    call = packed_call(fn, refs, evs, xs, dose, dta)
                    row = dict(function=fn, pairs=a.pairs, size=size, criteria=f"{dose}%/{dta}mm", points=pts * a.pairs,
                               work=(segs if fn == "geometric" else pts * int(dta * 3 * 2 + 1)) * a.pairs, **info)
                    if a.profile:
                        row.update(kernel_ms(call))
                        k = next(v for key, v in row.items() if key.startswith("k_gamma"))
                        row["work_per_s"] = row["work"] / (k / 1e3)
                    else:
                        row["call_ms"] = timed(lambda: batch(refs, evs, xs, xs, dose_to_agreement=dose, distance_to_agreement=dta),
                                               a.reps)
                        row["native_ms"] = timed(call, a.reps)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
