"""block_find_peaks (pylinac_b200/csrc/peaks.cuh) against scipy, on every path it takes.

It is the device routine behind every 1-D result: PicketFence pickets, Starshot rows, FieldAnalysis edges, VMAT / DLG and
core.profile.find_peaks.  tests/peaks_harness.cu runs it on its own, one CTA per run over a ragged batch, built twice: with the
library's skip table (512 blocks of 32 samples: the table walks up to 16384 samples, the per-lane prominence walks and linear width
walks above) and with the PicketFence units' table of 2 blocks (every profile longer than 64 samples takes the per-lane walks).
Each build runs with 128 threads (DLG), 256 (every other caller) and 1024.

Every run is compared with _ref_peaks_stable: scipy.signal.find_peaks restated from scipy's public, sort-free pieces with the tie
order the kernel promises (equal heights in the distance stage and equal keys at the max_number cut: the right-most ranks highest).
On tie-free profiles, where no tie can decide the outcome, every run is also compared with scipy itself through
oracle.pf_oracle.ref_find_peaks.  Indices, bases, prominences, width heights and the interpolated positions are compared bit for bit:
the kernel performs scipy's fp64 operations in scipy's order and is built without FMA contraction.

The last tests go through the public API (core.profile.find_peaks, MultiProfile) in the library build: profiles longer than the
skip table, more than 768 distance candidates (the bitonic ranking), argument parsing at its edges, the max_number slice and the
ValueError of fwxm_height > 1."""
import os
import shutil
import subprocess
import warnings

import numpy as np
import pytest
from scipy import signal

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "pylinac_b200", "csrc")

LENGTHS = (31, 32, 33, 63, 64, 65, 1024, 1280, 12800, 16384, 16385, 20000)
BUILDS = (512, 2)          # EPID_PK_MAXBLK: the library's table, the PicketFence units' table
BLOCKS = (128, 256, 1024)

# (hmin, distance, pmin, wmin, rel_height, max_number, sort_by_height)
#   hmin: "inf" | ("rel", r): min + r * range | ("abs", q): the q-quantile of the profile
#   distance: int | ("rel", f): max(int(f * n), 1) | "big": n + 5
#   pmin: None | absolute value | ("rel", f): f * range
ARGS = (
    ("inf", 1, None, 0.0, 0.5, None, 0),
    ("inf", 2, None, 0.0, 0.5, None, 0),
    ("inf", 3, None, 0.0, 0.5, None, 0),
    ("inf", 3, None, 0.0, 0.0, None, 1),
    ("inf", ("rel", 0.02), None, 0.0, 0.5, None, 0),
    ("inf", "big", None, 0.0, 0.5, None, 0),
    (("rel", 0.0), 1, None, 0.0, 0.0, None, 0),
    (("rel", 0.5), 3, 0.0, 0.0, 1.0, None, 0),
    (("rel", 1.0), 1, None, 0.0, 0.5, None, 0),
    (("abs", 0.9), 2, ("rel", 0.02), 0.0, 0.5, None, 0),
    ("inf", 1, ("rel", 0.4), 0.0, 0.5, None, 0),
    ("inf", 1, None, 1.5, 0.5, None, 0),
    ("inf", 3, ("rel", 0.02), 4.0, 1.0, 2, 1),
    ("inf", 1, None, 0.0, 0.5, 1, 0),
    ("inf", 1, None, 0.0, 0.5, 1, 1),
    ("inf", 3, None, 0.0, 1.0, 1, 0),
    ("inf", 1, None, 1.5, 0.5, 1, 1),
    ("inf", 2, None, 0.0, 0.5, 2, 0),
    ("inf", 2, None, 0.0, 0.0, 2, 1),
    ("inf", 1, None, 0.0, 0.5, 10 ** 6, 0),
    ("inf", 3, ("rel", 0.02), 0.0, 0.5, 3, 0),
    ("inf", 1, None, 0.0, 0.5, 4, 1),
    (("rel", 0.5), ("rel", 0.02), ("rel", 0.02), 0.0, 0.5, 3, 1),
    (("abs", 0.5), 3, 0.0, 1.5, 0.0, 5, 0),
    ("inf", 1, ("rel", 0.4), 4.0, 1.0, 3, 1),
    (("abs", 0.3), "big", None, 0.0, 1.0, 2, 1),
)


# ---------------------------------------------------------------------------------------------------------------- reference

def _distance_keep_stable(peaks, heights, distance):
    """scipy's _select_by_peak_distance with a stable priority order: among equal heights the right-most is visited first."""
    keep = np.ones(len(peaks), bool)
    pk = peaks.tolist()
    for j in np.argsort(heights, kind="stable")[::-1].tolist():
        if not keep[j]:
            continue
        k = j - 1
        while k >= 0 and pk[j] - pk[k] < distance:
            keep[k] = False
            k -= 1
        k = j + 1
        while k < len(pk) and pk[k] - pk[j] < distance:
            keep[k] = False
            k += 1
    return keep


def _ref_peaks_stable(x, hmin, distance, pmin, wmin, rel_height, max_number, by_height):
    """scipy.signal.find_peaks(x, height=hmin, distance, prominence=pmin, width=wmin, rel_height) and the reference's max_number
    cut (core/profile.py:2615-2623), with the stable tie order."""
    peaks = signal.find_peaks(x, height=hmin)[0]           # plateau midpoints of the local maxima, height filter
    if distance > 1 and len(peaks) > 1:
        peaks = peaks[_distance_keep_stable(peaks, x[peaks], distance)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                    # zero prominences / widths
        prom, lb, rb = signal.peak_prominences(x, peaks)
        if pmin is not None:
            k = prom >= pmin
            peaks, prom, lb, rb = peaks[k], prom[k], lb[k], rb[k]
        wid, wh, lip, rip = signal.peak_widths(x, peaks, rel_height=rel_height, prominence_data=(prom, lb, rb))
    k = wid >= wmin
    peaks, prom, lb, rb, wh, lip, rip = peaks[k], prom[k], lb[k], rb[k], wh[k], lip[k], rip[k]
    key = x[peaks] if by_height else prom
    sel = np.sort(np.argsort(key, kind="stable")[::-1][:max_number])
    return {"idx": peaks[sel], "lb": lb[sel], "rb": rb[sel], "prom": prom[sel], "wh": wh[sel], "lip": lip[sel], "rip": rip[sel]}


def _resolve(x, spec):
    """Kernel arguments of one ARGS entry on profile x, and the ref_find_peaks keywords that parse to the same arguments (None when
    an absolute threshold falls in [0, 1], which the reference reads as a ratio)."""
    hs, ds, ps, wmin, rel, mx, sbh = spec
    n = len(x)
    lo = x.min()
    rng = x.max() - lo
    if hs == "inf":
        hmin = thr = -np.inf
    elif hs[0] == "rel":
        hmin, thr = lo + hs[1] * rng, hs[1]
    else:
        hmin = float(np.quantile(x, hs[1]))
        thr = None if 0 <= hmin <= 1 else hmin
    if ds == "big":
        dist = sep = n + 5
    elif isinstance(ds, tuple):
        dist, sep = max(int(ds[1] * n), 1), ds[1]
    else:
        dist, sep = ds, (0 if ds == 1 else ds)
    pmin = ps[1] * rng if isinstance(ps, tuple) else ps
    args = dict(hmin=hmin, distance=dist, pmin=pmin, wmin=wmin, rel_height=rel, max_number=mx, by_height=sbh)
    kw = None if thr is None else dict(threshold=thr, peak_separation=sep, max_number=mx, fwxm_height=1 - rel, min_width=wmin,
                                       peak_sort="peak_heights" if sbh else "prominences", required_prominence=pmin)
    return args, kw


def _ref_scipy(x, kw):
    from oracle.pf_oracle import ref_find_peaks

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        idx, p = ref_find_peaks(x, **kw)
    return {"idx": idx, "lb": p["left_bases"], "rb": p["right_bases"], "prom": p["prominences"], "wh": p["width_heights"],
            "lip": p["left_ips"], "rip": p["right_ips"]}


# ---------------------------------------------------------------------------------------------------------------- profiles

def _gaussians(rng, n, noise):
    t = np.arange(n, dtype=np.float64)
    x = np.full(n, 0.05)
    for _ in range(int(rng.integers(1, 6))):
        c, s, h = rng.uniform(0, n), max(1.0, rng.uniform(0.005, 0.2) * n), rng.uniform(0.2, 1.0)
        x += h * np.exp(-0.5 * ((t - c) / s) ** 2)
    return x + noise * rng.standard_normal(n) if noise else x


def _field(rng, n, noise):
    """a flat-topped field: one dominant peak whose bases and width crossings lie far apart"""
    t = np.arange(n, dtype=np.float64)
    c, half, s = rng.uniform(0.4, 0.6) * n, rng.uniform(0.2, 0.35) * n, 0.01 * n + 1.0
    return 1.0 / (1.0 + np.exp((np.abs(t - c) - half) / s)) + noise * rng.standard_normal(n)


def _plateaus(rng, n):
    """piecewise constant, random even and odd run lengths (crossing 32-sample steps and warp segments), plateaus at both ends"""
    x = np.empty(n)
    i = 0
    while i < n:
        w = int(rng.integers(1, 41))
        x[i : i + w] = rng.integers(0, 12)
        i += w
    e = max(1, min(n // 4, int(rng.integers(2, 9))))
    x[:e] = 12.0
    x[n - e :] = 12.0
    return x


def _boundary_plateaus(n):
    """a plateau of width 2..6 at every 32-sample step (stage 1 sweeps from 1 + 32 j), shifted so it starts before, on and after
    the step; heights repeat (ties), the profile ends on plateaus"""
    x = np.zeros(n)
    for j, b in enumerate(range(1, n, 32)):
        w = 2 + j % 5
        s = b - j % (w + 1)
        x[max(s, 0) : s + w] = 1 + (7 * j) % 5
    x[:2] = 9.0
    x[n - 3 :] = 9.0
    return x


def _placed(n, knots):
    """piecewise linear through (position, value) knots"""
    k = np.asarray(sorted(knots), dtype=np.float64)
    return np.interp(np.arange(n, dtype=np.float64), k[:, 0], k[:, 1])


def _placed_profiles():
    """peaks, bases and width crossings at offsets 0, 31, 32 and 63 of 32-sample blocks.  With rel_height 1 the evaluation height
    is the higher base: the walk on that side ends on the base (a sample equal to the height, no interpolation)."""
    out = []
    n = 4096
    for i, (po, lo, ro) in enumerate(((0, 31, 32), (31, 32, 63), (32, 63, 0), (63, 0, 31))):
        p, lb, rb = 32 * 64 + po, 32 * 5 + lo, 32 * 110 + ro
        out.append((f"placed{i}a", _placed(n, [(0, 3.0), (lb, 0.0), (p, 10.0), (rb, 1.0), (n - 1, 4.0)]), True))
        out.append((f"placed{i}b", _placed(n, [(0, 3.0), (lb, 1.0), (p, 10.0), (rb, 0.0), (n - 1, 4.0)]), True))
    # bases in the peak's own block or the adjacent one
    for i, (q, lb, rb) in enumerate(((32 * 40 + 31, 32 * 40, 32 * 41), (32 * 41, 32 * 40 + 31, 32 * 41 + 31),
                                     (32 * 41 + 31, 32 * 41, 32 * 42), (32 * 40, 32 * 39 + 31, 32 * 40 + 31))):
        out.append((f"placed{i}c", _placed(n, [(0, 3.0), (lb, 0.5), (q, 10.0), (rb, 1.5), (n - 1, 4.0)]), True))
        out.append((f"placed{i}d", _placed(n, [(0, 3.0), (lb, 1.5), (q, 10.0), (rb, 0.5), (n - 1, 4.0)]), True))
    # equal minima in one block on each side: the left base is the right-most of them, the right base the left-most
    kn = [(0, 5.0), (32 * 7 + 3, 0.0), (32 * 7 + 11, 0.7), (32 * 7 + 20, 0.0), (32 * 30, 10.0),
          (32 * 50 + 4, 0.0), (32 * 50 + 13, 0.9), (32 * 50 + 29, 0.0), (n - 1, 6.0)]
    out.append(("equalmin", _placed(n, kn), False))
    for m in (64, 65):             # the same at the edge of the 2-block table
        out.append((f"placed{m}", _placed(m, [(0, 3.0), (31, 0.0), (32, 10.0), (63 if m > 64 else 62, 1.0), (m - 1, 4.0)]), True))
    return out


def _profiles():
    """(name, x, tie_free) with fixed seeds"""
    rng = np.random.default_rng(20261017)
    out = []
    for n in LENGTHS:
        out.append((f"noise{n}", rng.standard_normal(n), True))
        out.append((f"gaussnoise{n}", _gaussians(rng, n, 0.01), True))
        out.append((f"field{n}", _field(rng, n, 0.002), True))
        out.append((f"gauss{n}", _gaussians(rng, n, 0.0), False))
        out.append((f"fieldsmooth{n}", _field(rng, n, 0.0), False))
        out.append((f"int{n}", rng.integers(0, 5, n).astype(np.float64), False))
        out.append((f"intgauss{n}", np.round(30 * _gaussians(rng, n, 0.02)), False))
        out.append((f"plateau{n}", _plateaus(rng, n), False))
        out.append((f"bplateau{n}", _boundary_plateaus(n), False))
    # combs of 768 and 769 local maxima two samples apart: either side of the distance stage's rank-counting limit (PK_RANK_MAX),
    # every candidate in conflict with its neighbours; rising heights make one chain that settles one candidate per round
    for k in (768, 769):
        for name, h, tf in (("comb", rng.uniform(1.0, 2.0, k), True), ("combint", rng.integers(1, 4, k).astype(np.float64), False),
                            ("combramp", np.linspace(1.0, 2.0, k), True)):
            x = np.zeros(2 * k + 1)
            x[1::2] = h
            out.append((f"{name}{k}", x, tf))
    for n in (3, 33, 1024):
        out.append((f"up{n}", np.arange(n, dtype=np.float64), False))
        out.append((f"down{n}", np.arange(n, 0, -1, dtype=np.float64), False))
    for n in (3, 64, 20000):
        out.append((f"const{n}", np.full(n, 2.0), False))
    for i, v in enumerate(([0.0, 1.0, 0.0], [1.0, 0.0, 1.0], [0.0, 1.0, 1.0, 0.0], [0.0, 2.0, 1.0, 3.0], [3.0, 1.0, 2.0, 0.0],
                           [0.0, 2.0, 0.0, 2.0], [1.0, 1.0, 1.0, 1.0])):
        out.append((f"tiny{i}", np.asarray(v), False))
    return out + _placed_profiles()


class Batch:
    """All runs: profile x args (cap = every local maximum fits), with the expected results."""

    def __init__(self):
        self.profiles = _profiles()
        self.xs = np.concatenate([x for _, x, _ in self.profiles])
        self.offs = np.cumsum([0] + [len(x) for _, x, _ in self.profiles])[:-1]
        self.runs = []          # (profile no, args, cap)
        self.expect = []        # stable reference
        self.scipy = []         # scipy itself (tie-free profiles, representable arguments), else None
        for pi, (_, x, tie_free) in enumerate(self.profiles):
            for spec in ARGS:
                args, kw = _resolve(x, spec)
                # The kernel's distance rounds settle a chain of equal heights one candidate per round, and every round walks the
                # whole distance window: on a long profile full of ties, a window of thousands of candidates costs the kernel
                # seconds per run.  Such windows run on the profiles of up to 2000 samples.
                if not tie_free and len(x) > 2000 and args["distance"] > 64:
                    continue
                self.runs.append((pi, args, len(x) // 2 + 1))
                self.expect.append(_ref_peaks_stable(x, **args))
                self.scipy.append(_ref_scipy(x, kw) if tie_free and kw is not None else None)

    def describe(self, r):
        pi, args, cap = self.runs[r]
        return f"run {r}: {self.profiles[pi][0]} (n={len(self.profiles[pi][1])}) {args} cap={cap}"


@pytest.fixture(scope="module")
def batch():
    return Batch()


# ---------------------------------------------------------------------------------------------------------------- harness

def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def compile_harness(nvcc, out_dir, maxblk, src=os.path.join(HERE, "peaks_harness.cu"), csrc=CSRC):
    """the library's flags (pylinac_b200/csrc/Makefile) and EPID_PK_MAXBLK = maxblk"""
    exe = os.path.join(str(out_dir), f"peaks_harness_{maxblk}")
    return exe, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-fmad=false", "-std=c++17", f"-DEPID_PK_MAXBLK={maxblk}",
                 "-I", csrc, "-o", exe, src]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("peaks_harness")
    jobs = {mb: compile_harness(nvcc, d, mb) for mb in BUILDS}
    procs = {mb: subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for mb, (_, cmd) in jobs.items()}
    for mb, p in procs.items():
        try:
            out, _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            for q in procs.values():
                q.kill()
                q.communicate()
            raise
        assert p.returncode == 0, out
    return {mb: exe for mb, (exe, _) in jobs.items()}


def run_harness(exe, xs, runs, block, tmp):
    """runs: (offset, n, cap, args) -> per run -1 or the dict of its outputs"""
    nr = len(runs)
    col = lambda f, dt: np.asarray([f(r) for r in runs], dt)  # noqa: E731
    a = lambda r: r[3]  # noqa: E731
    with open(os.path.join(tmp, "in.bin"), "wb") as f:
        f.write(np.int32(nr).tobytes() + np.int64(len(xs)).tobytes())
        for arr in (col(lambda r: r[0], "<i8"), col(lambda r: r[1], "<i4"), col(lambda r: r[2], "<i4"),
                    col(lambda r: a(r)["distance"], "<i4"), col(lambda r: a(r)["max_number"] or 0, "<i4"),
                    col(lambda r: a(r)["by_height"], "<i4"), col(lambda r: a(r)["hmin"], "<f8"),
                    col(lambda r: -1.0 if a(r)["pmin"] is None else a(r)["pmin"], "<f8"), col(lambda r: a(r)["wmin"], "<f8"),
                    col(lambda r: a(r)["rel_height"], "<f8"), np.asarray(xs, "<f8")):
            f.write(arr.tobytes())
    out = subprocess.run([exe, os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin"), str(block)], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    buf = open(os.path.join(tmp, "out.bin"), "rb").read()
    count = np.frombuffer(buf, "<i4", nr)
    pos = 4 * nr
    res = []
    for c in count.tolist():
        if c <= 0:
            res.append(-1 if c < 0 else {k: np.empty(0) for k in ("idx", "lb", "rb", "prom", "wh", "lip", "rip")})
            continue
        r = {}
        for k, dt in (("idx", "<i4"), ("lb", "<i4"), ("rb", "<i4"), ("prom", "<f8"), ("wh", "<f8"), ("lip", "<f8"), ("rip", "<f8")):
            r[k] = np.frombuffer(buf, dt, c, pos)
            pos += c * np.dtype(dt).itemsize
        res.append(r)
    assert pos == len(buf)
    return res


def mismatches(got, want, label):
    """bit-exact comparison of one run; returns a list of messages"""
    if got == -1:
        return [f"{label}: capacity return -1"]
    if len(got["idx"]) != len(want["idx"]):
        return [f"{label}: {len(got['idx'])} peaks, expected {len(want['idx'])}: {got['idx'][:8]} vs {want['idx'][:8]}"]
    bad = []
    for k in ("idx", "lb", "rb", "prom", "wh", "lip", "rip"):
        g, w = np.asarray(got[k]), np.asarray(want[k])
        diff = np.flatnonzero(g != w)          # a NaN counts as a difference
        if len(diff):
            i = int(diff[0])
            bad.append(f"{label}: {k}[{i}] = {g[i]!r}, expected {w[i]!r} ({len(diff)} differ)")
    return bad


def compare_batch(b, exe, block, tmp):
    runs = [(int(b.offs[pi]), len(b.profiles[pi][1]), cap, args) for pi, args, cap in b.runs]
    res = run_harness(exe, b.xs, runs, block, tmp)
    bad = []
    for r, got in enumerate(res):
        bad += mismatches(got, b.expect[r], b.describe(r))
        if b.scipy[r] is not None:
            bad += mismatches(got, b.scipy[r], b.describe(r) + " vs scipy")
    return bad


# ---------------------------------------------------------------------------------------------------------------- tests

def test_stable_reference_is_scipy_on_tie_free_profiles(batch):
    """The stable restatement equals ref_find_peaks (scipy itself) wherever no tie can decide the outcome; no GPU needed."""
    checked = 0
    for r, want in enumerate(batch.scipy):
        if want is None:
            continue
        checked += 1
        bad = mismatches(batch.expect[r], want, batch.describe(r))
        assert not bad, "\n".join(bad[:20])
    assert checked > 500


@pytest.mark.gpu
@pytest.mark.parametrize("block", BLOCKS)
@pytest.mark.parametrize("maxblk", BUILDS)
def test_block_find_peaks_matches_scipy_bit_for_bit(batch, harness, tmp_path, maxblk, block):
    bad = compare_batch(batch, harness[maxblk], block, str(tmp_path))
    assert not bad, f"{len(bad)} mismatches:\n" + "\n".join(bad[:30])


@pytest.mark.gpu
@pytest.mark.parametrize("maxblk", BUILDS)
def test_capacity_overflow_returns_minus_one(harness, tmp_path, maxblk):
    """-1 exactly when more local maxima pass the height threshold than `cap` holds; at or under the capacity the full result"""
    rng = np.random.default_rng(7)
    profs = [rng.standard_normal(1024), rng.integers(0, 5, 20000).astype(np.float64), _boundary_plateaus(1280),
             rng.standard_normal(65), np.full(40, 1.0)]
    xs = np.concatenate(profs)
    offs = np.cumsum([0] + [len(x) for x in profs])[:-1]
    runs, expect = [], []
    for x, off in zip(profs, offs):
        for hs in ("inf", ("rel", 0.5)):
            args, _ = _resolve(x, (hs, 3, None, 0.0, 0.5, 2, 0))
            c = len(signal.find_peaks(x, height=args["hmin"])[0])
            for cap in sorted({0, max(c - 1, 0), c, c + 1}):
                runs.append((int(off), len(x), cap, args))
                expect.append(-1 if c > cap else _ref_peaks_stable(x, **args))
    res = run_harness(harness[maxblk], xs, runs, 256, str(tmp_path))
    for r, (got, want) in enumerate(zip(res, expect)):
        if want == -1:
            assert got == -1, f"run {r}: cap {runs[r][2]} exceeded, got a result"
        else:
            bad = mismatches(got, want, f"run {r}")
            assert not bad, bad


# ---- the public API (library build)

def _api_equal(x, **kw):
    from oracle.pf_oracle import ref_find_peaks
    from pylinac_b200.core.profile import find_peaks

    idx, p = find_peaks(x, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ridx, rp = ref_find_peaks(x, **kw)
    np.testing.assert_array_equal(idx, ridx, err_msg=str(kw))
    assert set(p) == set(rp)
    for k in rp:
        np.testing.assert_array_equal(p[k], rp[k], err_msg=f"{k} {kw}")
    return idx


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16384, 16385, 20000])
def test_public_find_peaks_beyond_the_skip_table(n):
    rng = np.random.default_rng(n)
    t = np.arange(n)
    field = 1.0 / (1.0 + np.exp((np.abs(t - 0.47 * n) - 0.3 * n) / (0.01 * n))) + 0.002 * rng.standard_normal(n)
    for x in (rng.standard_normal(n), field):
        for kw in ({}, {"threshold": 0.5, "peak_separation": 3}, {"max_number": 1}, {"max_number": 1, "fwxm_height": 0.8},
                   {"required_prominence": 0.3, "min_width": 2}, {"max_number": 3, "peak_sort": "peak_heights", "fwxm_height": 0.2}):
            _api_equal(x, **kw)


@pytest.mark.gpu
def test_public_find_peaks_more_than_768_distance_candidates():
    from oracle.pf_oracle import ref_find_peaks
    from pylinac_b200.core.profile import MultiProfile

    rng = np.random.default_rng(768)
    for n in (2600, 3000, 5000):
        x = rng.standard_normal(n)
        assert len(signal.find_peaks(x)[0]) > 768
        _api_equal(x, peak_separation=3)
        _api_equal(x, peak_separation=7.5, max_number=40)
        mp = MultiProfile(x)
        idx, vals = mp.find_peaks(threshold=0.2, min_distance=3)
        ridx, rp = ref_find_peaks(x, threshold=0.2, peak_separation=3)
        np.testing.assert_array_equal(idx, ridx)
        np.testing.assert_array_equal(vals, rp["peak_heights"])
        vidx, _ = mp.find_valleys(threshold=0.2, min_distance=3)
        np.testing.assert_array_equal(vidx, ref_find_peaks(-x, threshold=0.2, peak_separation=3)[0])


@pytest.mark.gpu
def test_public_find_peaks_argument_parsing():
    rng = np.random.default_rng(11)
    n = 1000
    x = rng.standard_normal(n)
    for kw in ({"threshold": 0}, {"threshold": 1}, {"threshold": 0.0, "peak_separation": 0}, {"peak_separation": 1},
               {"peak_separation": 0.0}, {"peak_separation": 1.0}, {"peak_separation": 2.5}, {"peak_separation": 4.01},
               {"search_region": (0.25, 0.75)}, {"search_region": (0.5, 0.5)}, {"search_region": (0.7, 0.3)},
               {"search_region": (0.0, 0.999)}, {"search_region": (100, 900)}, {"search_region": (n - 50, n + 500)},
               {"search_region": (n + 5, n + 50)}, {"search_region": (500, 100)}, {"search_region": (2, 4)},
               {"max_number": None}, {"max_number": 0}, {"max_number": -1}, {"max_number": -2}, {"max_number": 1},
               {"max_number": -2, "peak_sort": "peak_heights"}, {"max_number": -1, "search_region": (100, 900), "peak_separation": 3},
               {"max_number": 0, "search_region": (0.5, 0.5)}, {"max_number": -10 ** 6}):
        _api_equal(x, **kw)
    assert len(_api_equal(x, max_number=0)) == 0
    assert len(_api_equal(x, max_number=-1)) == len(_api_equal(x)) - 1


@pytest.mark.gpu
def test_public_find_peaks_max_number_slice_on_tied_keys():
    """[:max_number] of the descending order for every sign of max_number, with ties at the cut: the right-most of equal keys
    ranks first (negative values take a second launch that keeps count + max_number)"""
    from pylinac_b200.core.profile import find_peaks

    rng = np.random.default_rng(5)
    for x in (rng.integers(0, 5, 3000).astype(np.float64), _boundary_plateaus(1280), np.round(30 * _gaussians(rng, 5000, 0.02))):
        for mx in (None, 0, 1, 2, 7, -1, -2, -7, -10 ** 6):
            for sort in ("prominences", "peak_heights"):
                idx, p = find_peaks(x, peak_separation=3, max_number=mx, peak_sort=sort)
                got = {"idx": idx, "lb": p["left_bases"], "rb": p["right_bases"], "prom": p["prominences"], "wh": p["width_heights"],
                       "lip": p["left_ips"], "rip": p["right_ips"]}
                want = _ref_peaks_stable(x, -np.inf, 3, None, 0, 0.5, mx, sort == "peak_heights")
                bad = mismatches(got, want, f"n={len(x)} max_number={mx} {sort}")
                assert not bad, bad
                np.testing.assert_array_equal(p["widths"], want["rip"] - want["lip"])


@pytest.mark.gpu
def test_public_find_peaks_rejects_fwxm_height_above_one():
    from oracle.pf_oracle import ref_find_peaks
    from pylinac_b200.core.profile import find_peaks

    x = np.random.default_rng(3).standard_normal(500)
    for kw in ({"fwxm_height": 1.2}, {"fwxm_height": 1.0000001, "max_number": 0}, {"fwxm_height": 2.0, "search_region": (0.5, 0.5)}):
        with pytest.raises(ValueError, match="rel_height"):
            ref_find_peaks(x, **kw)
        with pytest.raises(ValueError, match="rel_height"):
            find_peaks(x, **kw)
    _api_equal(x, fwxm_height=1.0)
    _api_equal(x, fwxm_height=0.0)
