"""Time the ACR CT path on one GPU: a seeded 512 x 512 x N int16 ACR 464 series (tests/golden/acr_cases.py's acr_512, continued in z
with water slices to N slices) is written as DICOM to a temporary directory and read back, then
  * epid_ct_localize on the Slice branch (Otsu over the 110 mm disk) and on the ndarray branch (clipped, the cheese phantoms'), on the
    same device-resident series, the two interleaved call by call (CUDA events);
  * epid_ct_regions of the HU module slice (CUDA events per call);
  * ACRCT(...).analyze() end to end, with reading the files as a separate leg;
  * the numpy oracle's time per slice of the Slice-branch localization on the host.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_acr.py [--slices 200] [--reps 7]
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
from pylinac_b200 import acr  # noqa: E402


def series(n):
    """acr_512's 48 slices (0.5 mm pixels, 2.5 mm apart), continued to n slices with copies of its last (water) slice"""
    from tests.golden.acr_cases import case_series

    raw, slopes, intercepts, px, thk = case_series("acr_512")
    idx = np.minimum(np.arange(n), len(raw) - 1)
    return raw[idx], slopes[idx], intercepts[idx], px, thk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch

    from oracle import acr_oracle
    from tests.ct_writer import write_ct_slice

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    vol, slopes, intercepts, px, thk = series(a.slices)
    size = np.pi * 100.0**2 / px**2
    radius = 110 / px
    out = {"gpu": smi.strip().splitlines()[0] if smi.strip() else "unknown", "slices": a.slices, "shape": list(vol.shape)}
    ctx = nat.Context.default()
    b = nat.Batch.upload(ctx, vol)
    sl = np.arange(a.slices)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), r

    slice_branch = lambda: nat.ct_localize(ctx, b, slopes, intercepts, sl, size, False, False, otsu_disk_radius=radius)  # noqa: E731
    nd_branch = lambda: nat.ct_localize(ctx, b, slopes, intercepts, sl, size, False, True)  # noqa: E731
    slice_branch(), nd_branch()
    ts, tn = [], []
    for _ in range(a.reps):
        t, rows = timed(slice_branch)
        ts.append(t)
        tn.append(timed(nd_branch)[0])
    out["localize_slice_branch_ms"] = sorted(round(t, 3) for t in ts)
    out["localize_ndarray_branch_ms"] = sorted(round(t, 3) for t in tn)
    out["in_view"] = int((rows["status"] == nat.CT_OK).sum())
    z = 4
    nat.ct_regions(ctx, b, slopes, intercepts, z, radius)
    tr = [timed(lambda: nat.ct_regions(ctx, b, slopes, intercepts, z, radius))[0] for _ in range(a.reps)]
    out["regions_ms"] = sorted(round(t, 3) for t in tr)
    out["regions"] = len(nat.ct_regions(ctx, b, slopes, intercepts, z, radius)[0])
    b.free()
    with tempfile.TemporaryDirectory() as d:
        for k in range(a.slices):
            write_ct_slice(os.path.join(d, f"CT{k:04d}.dcm"), vol[k], series_uid="1.2.826.0.1.3680043.2.9", z=k * thk,
                           slice_thickness=thk, pixel_spacing=px, slope=slopes[k], intercept=intercepts[k])
        read, e2e = [], []
        for _ in range(2):
            t = time.perf_counter()
            ph = acr.ACRCT(d)
            read.append(time.perf_counter() - t)
            t = time.perf_counter()
            ph.analyze()
            e2e.append(time.perf_counter() - t)
        out["read_s"] = [round(t, 3) for t in read]
        out["analyze_s"] = [round(t, 3) for t in e2e]
        out["origin_slice"], out["roll"] = ph.origin_slice, float(ph.catphan_roll)
    t = time.perf_counter()
    zs = range(0, a.slices, max(1, a.slices // 4))
    for z in zs:
        acr_oracle.localize_slice(vol[z], slopes[z], intercepts[z], size, False, radius)
    out["oracle_ms_per_slice"] = round((time.perf_counter() - t) * 1000 / len(zs), 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
