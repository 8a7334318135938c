"""Outputs and speed of the calls that label connected components (ccl.cu's k_ccl_union and the flatten kernels after it), for one or
more builds of libepid.so, alternating the builds run by run in one invocation.

    python tools/bench_labelling.py [--lib NAME=PATH ...] [--reps 5] [--rounds 3]

Each run is a fresh process (the library is chosen at import through EPID_LIB) on seeded inputs:
  * locate_disk / locate_field: epid_global_locate in disk mode (4-connected) and field mode (8-connected) on 32 device-resident
    1024 x 1024 uint16 frames (one labelling chunk; 8 distinct oracle/synth.py frames repeated);
  * canny: epid_canny on 8 device-resident 1280 x 1280 float64 frames (a blurred field with noise, sigma 1, thresholds 0.1 / 0.2);
  * ct_clear / ct_keep: epid_ct_localize on tools/bench_cheese.py's seeded 512 x 512 x 200 int16 series (four chunks of 64 slices),
    clear_borders on and off;
  * nm: epid_nm_uniformity on tools/bench_nuclear.py's 1024_bin8 batch (512 floods, 0.6 mm), without arrays.
Per call and run it prints:
  * sha256: of the sorted region records with their counts and flags (locate), the edge maps (canny), the rows and the scharr,
    smoothed, filled and label planes of ct_localize(stages=True) (ct), the result rows (nm);
  * call_ms: CUDA-event times of --reps calls (ct without the host planes, as DESIGN.md §4.19 measures it);
  * kernel_ms: in a separate profiled call (torch.profiler, CUDA activity), the device time of each union and flatten kernel (for nm
    the frame kernel, which labels in shared memory).
The last line summarises per build the hashes (one per call if every run agrees) and the range of every time over the rounds; the
card's name and power limit are read in the same invocation."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the union kernels of builds before k_ccl_union too, so that such a build can be compared
KERNELS = ("k_ccl_union", "k_gl_union", "k_hyst_union", "k_ct_union", "k_gl_flatten", "k_hyst_mark", "k_ct_flatten", "k_nm_frame")


def worker(reps: int) -> None:
    sys.path.insert(0, ROOT)
    import ctypes as C

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import synth
    from pylinac_b200 import _native as nat
    from pylinac_b200 import nuclear
    from pylinac_b200.metrics import image as mi
    from tests.golden.nuclear_cases import flood
    from tools.bench_cheese import series

    def sha(*arrays) -> str:
        h = hashlib.sha256()
        for a in arrays:
            h.update(np.ascontiguousarray(a).tobytes())
        return h.hexdigest()

    ctx = nat.Context.default()
    batches = []

    def resident(a):
        b = nat.Batch.upload(ctx, a)
        batches.append(b)
        return b

    calls = {}      # name -> (timed call, call returning the hash)

    # whole-frame locators
    def locate(b, n, params, cap=1024):
        regs = np.zeros((n, cap), nat.REGION_DTYPE)
        counts, flags = np.zeros(n, np.int32), np.zeros(n, np.int32)
        nat.check(nat.lib().epid_global_locate(ctx.handle, b.handle, C.byref(params), nat._ptr(regs), cap, nat._ptr(counts),
                                              nat._ptr(flags)))
        # the call returns each frame's records sorted by (threshold, root), one record per pair; REGION_DTYPE has no padding
        return sha(counts, flags, *(regs[f, : counts[f]] for f in range(n)))

    fr = synth.epid1024()
    wl = np.stack([synth.winstonlutz_frame(synth.epid1024(), field_size_mm=(20 + 5 * (k % 4), 20 + 5 * (k % 4)), bb_size_mm=5.0,
                                           offset_mm_left=0.5 * k, offset_mm_up=-0.3 * k, noise_sigma=0.002, seed=k) for k in range(8)])
    of = np.stack([synth.openfield_frame(synth.epid1024(), field_size_mm=(100 + 10 * k, 120 - 5 * k), cax_offset_mm=(k - 4, 3 - k),
                                         seed=k) for k in range(8)])
    disk_p = mi.GlobalSizedDiskLocator(radius_mm=2.5, radius_tolerance_mm=1.0)._params(fr.dpmm)
    field_p = mi.GlobalSizedFieldLocator.from_physical(120.0, 120.0, 30.0)._params(fr.dpmm)
    for name, a, p in (("locate_disk", wl, disk_p), ("locate_field", of, field_p)):
        b = resident(np.ascontiguousarray(np.resize(a, (32, 1024, 1024))))
        calls[name] = (lambda b=b, p=p: locate(b, 32, p), lambda b=b, p=p: locate(b, 32, p))

    # Canny
    rng = np.random.default_rng(1)
    cf = np.stack([synth.openfield_frame(synth.as1200(), field_size_mm=(150 + 20 * k, 150), seed=k, noise_sigma=0.0) for k in range(8)])
    cf = cf.astype(np.float64) / 65535.0 + rng.normal(0.0, 0.02, cf.shape)
    cb = resident(cf)
    w, lw = nat.gaussian_kernel1d(1.0)

    def canny(download):
        h = C.c_void_p()
        nat.check(nat.lib().epid_canny(ctx.handle, cb.handle, nat._ptr(w), int(lw), 0.1, 0.2, C.byref(h)))
        with nat.Batch(ctx, h) as out:
            return sha(out.download()) if download else None
    calls["canny"] = (lambda: canny(False), lambda: canny(True))

    # CT localization
    vol, px = series(200)
    vb = resident(vol)
    size = np.pi * 150.0**2 / px**2
    sl = np.arange(200)

    def ct(clear, stages):
        r = nat.ct_localize(ctx, vb, 1.0, -1024.0, sl, size, clear, stages=stages)
        if not stages:
            return None
        rows, planes = r
        return sha(rows, planes["scharr"], planes["smoothed"], planes["filled"], planes["labels"])
    for name, clear in (("ct_clear", True), ("ct_keep", False)):
        calls[name] = (lambda clear=clear: ct(clear, False), lambda clear=clear: ct(clear, True))

    # nuclear floods
    distinct = np.stack([flood(k, (1024, 1024), counts=40.0 / 16, spots=[(0.4, 0.6, 0.05, 1.3)], gradient=0.1) for k in range(8)])
    nb = resident(np.ascontiguousarray(np.resize(distinct, (512, 1024, 1024))))
    calls["nm"] = (lambda: nuclear.analyze_batch(nb, 0.6, arrays=False),
                   lambda: sha(nuclear.analyze_batch(nb, 0.6, arrays=False).rows))

    out = {"sha256": {}, "call_ms": {}, "kernel_ms": {}}
    for name, (timed, hashed) in calls.items():
        out["sha256"][name] = hashed()
        timed()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            timed()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        out["call_ms"][name] = sorted(round(t, 3) for t in ts)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            timed()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            k = next((k for k in KERNELS if k in ev.key), None)
            if k and ev.device_type.name == "CUDA":
                kern[k] = kern.get(k, 0.0) + (getattr(ev, "self_device_time_total", None) or ev.device_time_total) / 1000.0
        out["kernel_ms"][name] = {k: round(v, 3) for k, v in kern.items()}
    for b in batches:
        b.free()
    print(json.dumps(out))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of a libepid.so build (default: this tree's)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args.reps)
        return
    libs = [x.split("=", 1) for x in args.lib] or [["this", os.path.join(ROOT, "pylinac_b200", "libepid.so")]]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card, "reps": args.reps, "unit": "ms"}), flush=True)
    runs = {name: [] for name, _ in libs}
    for rnd in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ, EPID_LIB=os.path.abspath(path))
            cmd = [sys.executable, __file__, "--worker", "--reps", str(args.reps)]
            res = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
            r = json.loads(res.stdout.strip().splitlines()[-1])
            runs[name].append(r)
            print(json.dumps({"build": name, "round": rnd, **r}), flush=True)
    summary = {}
    for name, rs in runs.items():
        calls = rs[0]["sha256"]
        summary[name] = {
            "sha256": {c: (rs[0]["sha256"][c] if all(r["sha256"][c] == rs[0]["sha256"][c] for r in rs) else "differs between runs")
                       for c in calls},
            "call_ms_range": {c: [min(min(r["call_ms"][c]) for r in rs), max(max(r["call_ms"][c]) for r in rs)] for c in calls},
            "kernel_ms_range": {c: {k: [min(r["kernel_ms"][c].get(k, 0.0) for r in rs), max(r["kernel_ms"][c].get(k, 0.0) for r in rs)]
                                    for k in rs[0]["kernel_ms"][c]} for c in calls},
        }
    print(json.dumps({"summary": summary}))


if __name__ == "__main__":
    main()
