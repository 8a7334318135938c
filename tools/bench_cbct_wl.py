"""WinstonLutz.from_cbct throughput on a clinical-size CBCT series.

Workload: a seeded 512 x 512 x 200 int16 series (0.908 mm pixels, 1.99 mm slices; air at about -1000 with noise and a 5 mm-radius
BB near the isocentre) written as DICOM slices to a temporary directory.  Prints one JSON line with, each number named for what it
covers (medians of --reps unless stated):
  * read_ms: DicomImageStack(dir, min_number=10, raw_pixels=True): threaded header pass, sort, pixel read into one page-locked volume;
  * h2d_ms: the synchronous upload of that volume (Batch.upload);
  * mip_kernel_us: device time of one k_stack_mip launch (CUDA activity records of torch.profiler over --iters launches of
    epid_stack_mip on the resident volume), and mip_gbps / mip_share_of_3350: the algorithmic bytes N * H * W * 2 read once over that
    time, and its share of the H100 SXM data-sheet 3.35 TB/s;
  * frames_ms: cbct_frames(volume, ratio): upload, epid_stack_mip, epid_zoom of both projections, epid_cbct_views;
  * wl_ms: the Winston-Lutz analysis of the four device-resident frames and the host set-level solve (analyze + results_data);
  * e2e_ms: WinstonLutz.from_cbct(dir, raw_pixels=True).analyze() + results_data() from the files;
  * the GPU name and power limit, read in the same run.
Writes nothing except its temporary directory (removed) unless --out is given.
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
from pylinac_b200 import winston_lutz as wl  # noqa: E402
from pylinac_b200.core import image  # noqa: E402
from tests import ct_writer  # noqa: E402

PIXEL_MM, SLICE_MM = 0.908, 1.99


def make_volume(n: int, size: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    vol = rng.integers(-1015, -984, size=(n, size, size)).astype(np.int16)
    # BB of radius 5 mm offset (1.2, -0.8, 1.5) mm from the volume centre, the sigmoid profile of the reference's phantom
    c = [(k / 2 - 0.5) * s + o for k, s, o in zip((n, size, size), (SLICE_MM, PIXEL_MM, PIXEL_MM), (1.5, 1.2, -0.8))]
    lo = [max(0, int((ci - 8) / s)) for ci, s in zip(c, (SLICE_MM, PIXEL_MM, PIXEL_MM))]
    hi = [min(k, int((ci + 8) / s) + 2) for ci, s, k in zip(c, (SLICE_MM, PIXEL_MM, PIXEL_MM), (n, size, size))]
    z, y, x = np.meshgrid(*[np.arange(a, b) * s for a, b, s in zip(lo, hi, (SLICE_MM, PIXEL_MM, PIXEL_MM))], indexing="ij")
    d = np.sqrt((z - c[0]) ** 2 + (y - c[1]) ** 2 + (x - c[2]) ** 2)
    bb = np.round(1000 * (1 / (1 + np.exp(-np.clip(5.0 - d, 0, None))) - 0.5)).astype(np.int16)
    vol[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] += bb
    return vol


def median_ms(fn, reps: int):
    ts, out = [], None
    for _ in range(reps):
        t = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=200)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200, help="epid_stack_mip launches in the profiled window")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if nat.device_count() == 0:
        raise SystemExit("bench_cbct_wl needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    ctx = nat.Context.default()
    vol = make_volume(args.slices, args.size, 2024)
    nbytes = vol.nbytes
    res = {"gpu": gpu, "shape": list(vol.shape), "dtype": str(vol.dtype), "volume_mb": nbytes / 1e6}
    with tempfile.TemporaryDirectory() as tmp:
        order = np.random.default_rng(5).permutation(len(vol))
        ct_writer.write_series(tmp, vol, slice_thickness=SLICE_MM, pixel_spacing=PIXEL_MM, order=order)
        image.DicomImageStack(tmp, min_number=10, raw_pixels=True)           # warm: page cache, thread pool, pinned allocator
        res["read_ms"], stack = median_ms(lambda: image.DicomImageStack(tmp, min_number=10, raw_pixels=True), args.reps)
        assert np.array_equal(stack.volume, vol)

        def upload():
            b = nat.Batch.upload(ctx, stack.volume)
            b.free()

        upload()
        res["h2d_ms"], _ = median_ms(upload, args.reps)
        res["h2d_gbps"] = nbytes / (res["h2d_ms"] * 1e-3) / 1e9

        from torch.profiler import ProfilerActivity, profile

        vb = nat.Batch.upload(ctx, stack.volume)
        for _ in range(5):
            for o in nat.stack_mip(ctx, vb):
                o.free()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                for o in nat.stack_mip(ctx, vb):
                    o.free()
        tot_us, count = 0.0, 0
        for ev in prof.key_averages():
            if "k_stack_mip" in ev.key:
                tot_us += getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)
                count += ev.count
        vb.free()
        assert count == args.iters, count
        res["mip_kernel_us"] = tot_us / count
        res["mip_gbps"] = nbytes / (res["mip_kernel_us"] * 1e-6) / 1e9
        res["mip_share_of_3350"] = res["mip_gbps"] / 3350.0

        ratio = stack.metadata.SliceThickness / stack.metadata.PixelSpacing[0]

        def frames():
            groups = wl.cbct_frames(stack.volume, ratio)
            for b, _ in groups:
                b.free()

        frames()
        res["frames_ms"], _ = median_ms(frames, args.reps)

        groups = wl.cbct_frames(stack.volume, ratio)
        st = wl.WinstonLutz._from_stack(stack)

        def analyse():
            st._groups = groups
            st.analyze()
            return st.results_data()

        analyse()
        res["wl_ms"], rd = median_ms(analyse, args.reps)
        for b, _ in groups:
            b.free()

        def e2e():
            s = wl.WinstonLutz.from_cbct(tmp, raw_pixels=True)
            s.analyze()
            return s.results_data()

        e2e()
        res["e2e_ms"], rd = median_ms(e2e, args.reps)
        sv = rd.bb_shift_vector
        res["bb_shift_vector"] = [round(sv["x"], 4), round(sv["y"], 4), round(sv["z"], 4)]
        res["max_2d_cax_to_bb_mm"] = round(rd.max_2d_cax_to_bb_mm, 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
