"""Median filter speed on uint16 1024 x 1024 frames: k = 3, 5 and 10 (VMAT's size) and k = 51, for one or more builds of
libepid.so, alternating the builds run by run in one invocation.

    python tools/bench_filters.py [--lib NAME=PATH ...] [--frames 8] [--reps 20] [--rounds 3]

Each run is a fresh process (the library is chosen at import through EPID_LIB).  A call is timed with CUDA events around
the device work of epid_median_filter on a resident batch (the call ends in a stream synchronise).  Prints one JSON line per
(build, round, k) and the card's name and power limit read in the same invocation."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(frames: int, reps: int, ks) -> None:
    sys.path.insert(0, ROOT)
    import ctypes as C

    import numpy as np
    import torch

    from pylinac_b200 import _native as nat

    ctx = nat.Context.default()
    a = np.random.default_rng(0).integers(0, 65536, (frames, 1024, 1024)).astype(np.uint16)
    out = {}
    with nat.Batch.upload(ctx, a) as b:
        for k in ks:
            def call():
                h = C.c_void_p()
                rc = nat.lib().epid_median_filter(ctx.handle, b.handle, int(k), C.byref(h))
                if rc != nat.EPID_OK:
                    return None
                nat.lib().epid_batch_free(h)
                return True
            if call() is None:          # size refused by this build
                out[k] = None
                continue
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(reps):
                call()
            ev1.record()
            torch.cuda.synchronize()
            out[k] = ev0.elapsed_time(ev1) / reps / frames
    print(json.dumps(out))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of a libepid.so build (default: this tree's)")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--k", type=int, nargs="*", default=[3, 5, 10, 51])
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args.frames, args.reps, args.k)
        return
    libs = [x.split("=", 1) for x in args.lib] or [["this", os.path.join(ROOT, "pylinac_b200", "libepid.so")]]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card, "frames": args.frames, "shape": [1024, 1024], "dtype": "uint16", "unit": "ms per frame"}))
    for rnd in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ, EPID_LIB=os.path.abspath(path))
            cmd = [sys.executable, __file__, "--worker", "--frames", str(args.frames), "--reps", str(args.reps), "--k", *map(str, args.k)]
            res = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
            print(json.dumps({"build": name, "round": rnd, "ms_per_frame": json.loads(res.stdout.strip().splitlines()[-1])}))


if __name__ == "__main__":
    main()
