"""Time the cheese-phantom localization on one GPU: a seeded 512 x 512 x 200 int16 series (water cylinder with inserts, air end
slices) is written as DICOM to a temporary directory, then read, copied to the device, localized (epid_ct_localize: CUDA events, and
per-kernel times from torch.profiler in a separate run) and analyzed end to end (TomoCheese(...).analyze()).  The numpy oracle's time
per slice is measured on the host for comparison.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_cheese.py [--slices 200] [--reps 5]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pylinac_b200 import _native as nat  # noqa: E402
from pylinac_b200 import cheese  # noqa: E402


def series(n, size=512, px=0.8, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:size, 0:size]
    c = size / 2 - 0.5
    r = np.hypot(xx - c, yy - c) * px
    base = np.where(r <= 152.0, 2.0, -1000.0)
    vol = np.empty((n, size, size), np.int16)
    for z in range(n):
        hu = base.copy() if 10 <= z < n - 10 else np.full((size, size), -1000.0)
        if n // 3 <= z < 2 * n // 3:
            for k, ang in enumerate([-75, -45, -15, 15, 45, 75, 105, 135, 165, -165, -135, -105]):
                a = np.deg2rad(ang)
                hu[np.hypot(xx - c - np.cos(a) * 110 / px, yy - c - np.sin(a) * 110 / px) * px <= 12.5] = {0: -850.0, 3: 950.0}.get(k, 0.0)
        vol[z] = np.rint(hu + rng.normal(0, 6.0, hu.shape) + 1024).astype(np.int16)
    return vol, px


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the torch.profiler trace (default: none written)")
    a = ap.parse_args()
    import torch

    from oracle import ct_oracle
    from tests.ct_writer import write_series

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    vol, px = series(a.slices)
    size = np.pi * 150.0**2 / px**2
    out = {"gpu": smi.strip().splitlines()[0] if smi.strip() else "unknown", "slices": a.slices, "shape": list(vol.shape)}
    with tempfile.TemporaryDirectory() as d:
        write_series(d, vol, slice_thickness=2.0, pixel_spacing=px, slope=1.0, intercept=-1024.0)
        t = time.perf_counter()
        ph = cheese.TomoCheese(d)
        out["read_s"] = time.perf_counter() - t
        ctx = nat.Context.default()
        b = nat.Batch.upload(ctx, ph.dicom_stack.volume)      # warm-up of the upload path
        b.free()
        ctx.sync()
        t = time.perf_counter()
        b = nat.Batch.upload(ctx, ph.dicom_stack.volume)
        ctx.sync()
        out["h2d_s"] = time.perf_counter() - t
        sl = np.arange(a.slices)
        nat.ct_localize(ctx, b, 1.0, -1024.0, sl, size, True)
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rows = nat.ct_localize(ctx, b, 1.0, -1024.0, sl, size, True)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        out["localize_ms"] = sorted(times)
        out["in_view"] = int((rows["status"] == nat.CT_OK).sum())
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.ct_localize(ctx, b, 1.0, -1024.0, sl, size, True)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and (ev.key.startswith("_ZN") or "k_" in ev.key):
                name = next((k for k in ("k_ct_scharr", "k_correlate1d", "k_ct_otsu", "k_ct_binarize", "k_ccl_union", "k_ct_flatten",
                                         "k_ct_mark_border", "k_ct_clear_flagged", "k_ct_background", "k_ct_fill", "k_ct_region_sums",
                                         "k_ct_select") if k in ev.key), ev.key[:40])
                kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1000.0
        out["kernel_ms"] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.out, "bench_cheese.pt.trace.json"))
        b.free()
        e2e = []
        for _ in range(2):
            t = time.perf_counter()
            ph = cheese.TomoCheese(d)
            ph.analyze()
            e2e.append(time.perf_counter() - t)
        out["analyze_end_to_end_s"] = e2e
        out["origin_slice"], out["roll"] = ph.origin_slice, float(ph.catphan_roll)
    t = time.perf_counter()
    for z in range(0, a.slices, a.slices // 4):
        ct_oracle.localize_slice(vol[z], 1.0, -1024.0, size, True)
    out["oracle_ms_per_slice"] = (time.perf_counter() - t) * 1000 / len(range(0, a.slices, a.slices // 4))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
