"""XIM decode throughput on the GPU (csrc/xim.cu): 512 frames of 1280 x 1280 at bytes_per_pixel 4 (what EPIDs write), at two
compressibilities -- a smooth synthetic EPID field (mostly 1-byte diffs) and a noisy one (2-byte diffs).

Reports, per compressibility:
  * device-resident decode: the k_xim_* kernel time of one batch (torch.profiler, CUDA activities, in a run of its own), frames/s
    and GB/s of the algorithmic bytes (lookup table + compressed pixels read once, the output written once) -- an HBM-bound leg;
  * end to end from the page-locked compressed arena to a device uint16 batch (epid_xim_decode: one H2D copy + decode, host clock
    around a synchronous call), next to the upload of the same frames as raw uint16 from page-locked memory in the same run -- the
    PCIe-bound leg;
  * the GPU name and power limit.

    python tools/bench_xim.py [--frames 512] [--reps 5] [--out results.json]

The last line printed is the whole result as JSON; --out also writes it to a file.
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
from pylinac_b200 import xim  # noqa: E402
from tests import xim_writer as xw  # noqa: E402
from tests.golden.xim_cases import smooth_field  # noqa: E402

H = W = 1280
DISTINCT = 16          # distinct encoded frames, repeated through the batch (the decode does not depend on repetition)


def build_arena(kind: str, n: int):
    enc = []
    for i in range(DISTINCT):
        v = smooth_field(H, W, 500 + i, noise=3.0 if kind == "smooth" else 3000.0)
        enc.append((v, *xw.encode_pixels(v, 4)))
    desc = np.zeros((n, 4), np.int64)
    pos = 0
    for i in range(n):
        _, lut, pix = enc[i % DISTINCT]
        desc[i] = (pos, len(lut), pos + ((len(lut) + 15) & ~15), len(pix))
        pos = int(desc[i, 2]) + ((len(pix) + 15) & ~15)
    arena = nat.pinned_empty((pos,), np.uint8)
    for i in range(n):
        _, lut, pix = enc[i % DISTINCT]
        arena[desc[i, 0]: desc[i, 0] + len(lut)] = np.frombuffer(lut, np.uint8)
        arena[desc[i, 2]: desc[i, 2] + len(pix)] = np.frombuffer(pix, np.uint8)
    raw = nat.pinned_empty((n, H, W), np.uint16)
    for i in range(n):
        raw[i] = np.clip(enc[i % DISTINCT][0], 0, 65535).astype(np.uint16)
    return arena, desc, raw, enc


def kernel_ms(arena, desc, n) -> float:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        b, st = xim.decode_arena(arena, desc, H, W, 4, np.uint16)
        b.free()
    tot = 0.0                            # microseconds of every k_xim_* kernel
    for ev in prof.key_averages():
        if "k_xim_" in ev.key:
            tot += getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0.0)
    return tot / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if nat.device_count() == 0:
        raise SystemExit("bench_xim needs a CUDA device")
    n = args.frames
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    ctx = nat.Context.default()
    result = {"gpu": gpu, "frames": n, "shape": [H, W], "bytes_per_pixel": 4, "legs": {}}
    for kind in ("smooth", "noisy"):
        arena, desc, raw, enc = build_arena(kind, n)
        lut_bytes, pix_bytes = int(desc[:, 1].sum()), int(desc[:, 3].sum())
        algo_bytes = lut_bytes + pix_bytes + n * H * W * 2          # U16 output written once
        # correctness of the timed configuration: every distinct frame against its source array
        b, st = xim.decode_arena(arena, desc, H, W, 4, np.uint16)
        got = b.download()
        b.free()
        assert not st.any() and all(np.array_equal(got[i], np.clip(enc[i % DISTINCT][0], 0, 65535)) for i in range(DISTINCT))
        e2e, up = [], []
        for _ in range(args.reps):       # alternate the two legs
            t = time.perf_counter()
            b, st = xim.decode_arena(arena, desc, H, W, 4, np.uint16)
            e2e.append(time.perf_counter() - t)
            b.free()
            t = time.perf_counter()
            ub = nat.Batch.upload(ctx, raw)
            up.append(time.perf_counter() - t)
            ub.free()
        k_ms = kernel_ms(arena, desc, n)
        result["legs"][kind] = {
            "compressed_bytes_per_pixel": pix_bytes / (n * H * W), "lookup_bytes": lut_bytes, "compressed_bytes": pix_bytes,
            "algorithmic_bytes": algo_bytes,
            "decode_kernels_ms": k_ms, "decode_frames_per_s": n / (k_ms / 1e3), "decode_GB_per_s": algo_bytes / (k_ms / 1e3) / 1e9,
            "e2e_ms_min": min(e2e) * 1e3, "e2e_ms_all": [x * 1e3 for x in e2e], "e2e_frames_per_s": n / min(e2e),
            "raw_u16_upload_ms_min": min(up) * 1e3, "raw_u16_upload_ms_all": [x * 1e3 for x in up],
        }
        print(kind, json.dumps(result["legs"][kind]))
        del arena, raw
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
