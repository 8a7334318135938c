"""CPU: the gamma_geometric / gamma_1d oracle against the reference's goldens (and the live reference where it is present), the
window search against np.argmin, the fma emulation against exact rational arithmetic, the host build of the device's segment
distance against the oracle and math.dist, and the argument errors of core.gamma (raised before anything reaches a device)."""
import math
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle import gamma1d_oracle as O
from pylinac_b200.core import gamma as G
from tests.golden.gamma1d_cases import CASES, ERROR_CASES, case_args, error_args

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "gamma1d_golden.npz"))
FUNCS = {"geometric": O.gamma_geometric, "1d": O.gamma_1d}


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _reference():
    try:
        from oracle.refstub import import_reference

        import_reference()
        import pylinac.core.gamma as rgamma
        return rgamma
    except Exception:  # noqa: BLE001 -- the reference is absent
        return None


def assert_gamma_1d_close(got, want):
    """gamma_1d's gamma: nan in the same places, the rest within 2 units in the last place (the reference squares with libm pow)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_array_max_ulp(got[ok], want[ok], maxulp=2)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(name):
    fn, ref, ev, rc, ec, kw = case_args(name)
    if "error:" + name in GOLDEN:
        kind, msg = GOLDEN["error:" + name]
        with pytest.raises(Exception) as info:
            FUNCS[fn](ref, ev, rc, ec, **kw)
        assert type(info.value).__name__ == kind and str(info.value) == msg
        return
    with np.errstate(all="ignore"):
        got = FUNCS[fn](ref, ev, rc, ec, **kw)
    if fn == "geometric":
        assert got.dtype == GOLDEN[name].dtype
        np.testing.assert_array_equal(got, GOLDEN[name])
    else:
        assert got[0].dtype == GOLDEN[name].dtype
        assert_gamma_1d_close(got[0], GOLDEN[name])
        np.testing.assert_array_equal(got[1], GOLDEN[name + ":samples"])
        np.testing.assert_array_equal(got[2], GOLDEN[name + ":x"])


def test_oracle_equals_live_reference_on_seeded_pairs():
    rgamma = _reference()
    if rgamma is None:
        pytest.skip("the reference is absent")
    rng = np.random.default_rng(17)
    for k in range(12):
        n = int(rng.integers(20, 120))
        x = np.cumsum(rng.uniform(0.2, 1.0, n))
        ref = 1000 * np.exp(-((x - x.mean()) / (np.ptp(x) / 3)) ** 2) + rng.normal(0, 5, n)
        ev = np.interp(x + rng.uniform(-1, 1), x, ref) * rng.uniform(0.97, 1.03)
        kw = dict(dose_to_agreement=float(rng.choice([1, 2, 3])), distance_to_agreement=float(rng.choice([0.5, 1, 2, 3])))
        if k % 2:
            x = x[::-1].copy()
        np.testing.assert_array_equal(O.gamma_geometric(ref, ev, x, x, **kw), rgamma.gamma_geometric(ref, ev, x, x, **kw))
        with np.errstate(all="ignore"):
            got, want = O.gamma_1d(ref, ev, x, x, **kw), rgamma.gamma_1d(ref, ev, x, x, **kw)
        assert_gamma_1d_close(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])


@pytest.mark.parametrize("dec", [False, True])
def test_window_search_is_argmin_on_tie_grids(dec):
    rng = np.random.default_rng(int(dec))
    for _ in range(300):
        step = float(rng.choice([1.0, 0.5, 0.25, 0.1, 3.0]))
        x = np.arange(int(rng.integers(1, 60)), dtype=float) * step + float(rng.choice([0.0, -7.0, 0.3]))
        if dec:
            x = x[::-1].copy()
        for t in list(x[:5] + step / 2) + list(x[-5:] - step / 2) + [x.min() - 10, x.max() + 10, float(rng.uniform(x.min(), x.max()))]:
            assert O.argmin_abs(x, t, dec) == int(np.argmin(np.abs(x - t))), (x, t)


def test_fma_emulation_is_correctly_rounded():
    rng = np.random.default_rng(5)
    a, b = rng.normal(size=20000) * 10.0 ** rng.integers(-5, 5, 20000), rng.normal(size=20000)
    c = -a * b * (1 + rng.normal(size=20000) * 1e-12)                   # cancellation, the hard case
    c[::2] = rng.normal(size=10000)
    got = O.fma(a, b, c)
    for i in range(0, 20000, 7):
        assert got[i] == float(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))), i


def test_host_build_of_the_device_distance():
    """tests/gamma1d_dist_check.cu runs the device's segment_distance on the host: 10**6 seeded segments against the oracle, its
    Python-dist against math.dist, and 2000 of them against the reference's _compute_distance where it is present"""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "gamma1d_dist_check")
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Xcompiler", "-ffp-contract=off", "-o", exe,
                        os.path.join(HERE, "gamma1d_dist_check.cu")], check=True, capture_output=True)
        rng = np.random.default_rng(23)
        n = 1_000_000
        seg = rng.normal(size=(n, 6)) * rng.choice([1e-3, 1.0, 10.0, 300.0], size=(n, 1))
        seg[: n // 4, 3] = seg[: n // 4, 5]              # flat segments
        seg[n // 4: n // 2, 2:4] = seg[n // 4: n // 2, 0:2] + rng.normal(size=(n // 4, 2)) * 1e-9
        seg[10, 2:] = [1.0, 2.0, 1.0, 2.0]               # a zero-length segment: pinv is 0
        seg[11, 3] = np.nan                              # a nan vertex: the reference raises
        src, dst = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        seg.tofile(src)
        r = subprocess.run([exe, src, dst], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        out = np.fromfile(dst).reshape(3, n)
    d, bad = O.segment_distance(*seg.T)
    np.testing.assert_array_equal(out[2] != 0, bad)
    np.testing.assert_array_equal(out[0][~bad], d[~bad])
    np.testing.assert_array_equal(out[1], O.py_dist(seg[:, 0], seg[:, 1], seg[:, 2], seg[:, 3]))
    for i in range(0, n, 97):
        assert out[1, i] == math.dist(seg[i, :2], seg[i, 2:4]), i
    rgamma = _reference()
    if rgamma is not None:
        for i in list(range(0, n, n // 1000)) + list(range(n // 4, n // 4 + 1000)) + [10]:
            p, v1, v2 = seg[i, :2], seg[i, 2:4], seg[i, 4:6]
            assert out[0, i] == rgamma._compute_distance(p=p, vertices=[v1, v2]), i


@pytest.mark.parametrize("name", sorted(ERROR_CASES))
def test_argument_errors_are_the_reference_s(name):
    fn, ref, ev, rc, ec, kw = error_args(name)
    kind, msg = GOLDEN["error:" + name]
    with pytest.raises(Exception) as info:
        (G.gamma_geometric if fn == "geometric" else G.gamma_1d)(ref, ev, rc, ec, **kw)
    assert type(info.value).__name__ == kind and str(info.value) == msg


def test_float32_coordinates_are_refused():
    x = np.arange(10, dtype=np.float32)
    for f in (G.gamma_geometric, G.gamma_1d):
        with pytest.raises(TypeError, match="float64 or integer"):
            f(np.ones(10), np.ones(10), x, x)


def test_batch_checks_every_pair_before_the_device():
    good, bad = np.linspace(1, 2, 20), np.ones((2, 3))
    with pytest.raises(ValueError, match="must be 1D"):
        G.gamma_geometric_batch([good, bad], [good, good])
    with pytest.raises(ValueError, match="Resolution factor"):
        G.gamma_1d_batch([good], [good], resolution_factor=0)
    assert G.gamma_geometric_batch([], []) == [] and G.gamma_1d_batch(np.empty((0, 5)), np.empty((0, 5))) == []
