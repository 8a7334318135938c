"""GPU: core.gamma.gamma_geometric / gamma_1d and their batches against the reference's goldens and the oracle: gamma_geometric bit
for bit; gamma_1d's samples and positions bit for bit, its gamma bit for bit against the oracle and within 2 ulp of the reference
(whose squares are libm pow); ragged batches against pair-by-pair calls; the profile gamma methods against their goldens."""
import os

import numpy as np
import pytest

from oracle import gamma1d_oracle as O
from pylinac_b200.core import gamma as G
from pylinac_b200.core import profile as P
from tests.golden.gamma1d_cases import CASES, PROFILE_CASES, case_args, profile_signal
from tests.test_oracle_gamma1d import assert_gamma_1d_close

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "gamma1d_golden.npz"))
DTYPES = [np.float64, np.float32, np.uint16, np.int32]


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_reference(name):
    fn, ref, ev, rc, ec, kw = case_args(name)
    f = G.gamma_geometric if fn == "geometric" else G.gamma_1d
    if "error:" + name in GOLDEN:
        kind, msg = GOLDEN["error:" + name]
        with pytest.raises(Exception) as info:
            f(ref, ev, rc, ec, **kw)
        assert type(info.value).__name__ == kind and str(info.value) == msg
        return
    got = f(ref, ev, rc, ec, **kw)
    if fn == "geometric":
        assert got.dtype == GOLDEN[name].dtype
        np.testing.assert_array_equal(got, GOLDEN[name])
        return
    assert got[0].dtype == GOLDEN[name].dtype
    assert_gamma_1d_close(got[0], GOLDEN[name])
    np.testing.assert_array_equal(got[1], GOLDEN[name + ":samples"])
    np.testing.assert_array_equal(got[2], GOLDEN[name + ":x"])
    with np.errstate(all="ignore"):
        np.testing.assert_array_equal(got[0], O.gamma_1d(ref, ev, rc, ec, **kw)[0])


def _pair(rng, dtype):
    nr, ne = int(rng.integers(30, 700)), int(rng.integers(30, 700))
    pr, pe = float(rng.choice([0.1, 0.25, 0.392, 0.5, 1.0, 2.5])), float(rng.choice([0.1, 0.336, 0.5, 1.0]))
    rx = (np.arange(nr) - (nr - 1) / 2) * pr
    ex = (np.arange(ne) - (ne - 1) / 2) * pe
    ex = ex * max(1.0, (rx.max() + 2) / ex.max())
    w = (rx.max() - rx.min()) * 0.6
    shape = lambda x, c, s: s * (200 + 800 / (1 + np.exp(-(x - c + w / 2))) / (1 + np.exp(x - c - w / 2)))  # noqa: E731
    ref = shape(rx, 0.0, 1.0) + rng.normal(0, 3, nr)
    ev = shape(ex, rng.uniform(-1, 1), rng.uniform(0.97, 1.03)) + rng.normal(0, 3, ne)
    if np.issubdtype(dtype, np.integer):
        ref, ev = np.round(ref), np.round(ev)
    ref, ev = ref.astype(dtype), ev.astype(dtype)
    if rng.random() < 0.3:
        ex, ev = ex[::-1].copy(), ev[::-1].copy()
    if rng.random() < 0.2:
        rx, ref = rx[::-1].copy(), ref[::-1].copy()
    return ref, ev, rx, ex


@pytest.mark.parametrize("global_dose", [True, False])
def test_fuzz_against_the_oracle(global_dose):
    rng = np.random.default_rng(31 + global_dose)
    for trial in range(24):
        dtype = DTYPES[trial % 4]
        pairs = [_pair(rng, dtype) for _ in range(3)]
        kw = dict(dose_to_agreement=float(rng.choice([1, 2, 3])), distance_to_agreement=float(rng.choice([0.5, 1, 2, 3])),
                  gamma_cap_value=float(rng.choice([1, 2])), dose_threshold=float(rng.choice([0, 5, 50])))
        refs, evs, rcs, ecs = zip(*pairs)
        rf = int(rng.choice([1, 3, 5]))
        got1 = G.gamma_1d_batch(refs, evs, rcs, ecs, global_dose=global_dose, resolution_factor=rf, **kw)
        for k, (ref, ev, rc, ec) in enumerate(pairs):
            with np.errstate(all="ignore"):
                want = O.gamma_1d(ref, ev, rc, ec, global_dose=global_dose, resolution_factor=rf, **kw)
            for a, b in zip(got1[k], want):
                np.testing.assert_array_equal(a, b, err_msg=f"gamma_1d trial {trial} pair {k} {dtype}")
        if global_dose:
            got = G.gamma_geometric_batch(refs, evs, rcs, ecs, **kw)
            for k, (ref, ev, rc, ec) in enumerate(pairs):
                np.testing.assert_array_equal(got[k], O.gamma_geometric(ref, ev, rc, ec, **kw),
                                              err_msg=f"gamma_geometric trial {trial} pair {k} {dtype}")


def test_ragged_batches_equal_pair_by_pair_calls():
    rng = np.random.default_rng(9)
    pairs = [_pair(rng, DTYPES[k % 4]) for k in range(9)]
    refs, evs, rcs, ecs = zip(*pairs)
    kw = dict(dose_to_agreement=2, distance_to_agreement=2)
    for one, batch in ((G.gamma_geometric, G.gamma_geometric_batch), (G.gamma_1d, G.gamma_1d_batch)):
        got = batch(refs, evs, rcs, ecs, **kw)
        for k, p in enumerate(pairs):
            want = one(*p, **kw)
            for a, b in zip(got[k] if isinstance(got[k], tuple) else [got[k]], want if isinstance(want, tuple) else [want]):
                np.testing.assert_array_equal(a, b)
    rows = np.stack([np.linspace(1, 2, 50) + k for k in range(4)])
    assert [g.tolist() for g in G.gamma_geometric_batch(rows, rows)] == [G.gamma_geometric(r, r).tolist() for r in rows]


@pytest.mark.parametrize("name", sorted(PROFILE_CASES))
def test_profile_methods_equal_the_reference(name):
    method, nr, dr, ne, de, kw = PROFILE_CASES[name]
    rng = np.random.default_rng(4000 + sorted(PROFILE_CASES).index(name))
    a, b = profile_signal(nr, rng), profile_signal(ne, rng, centre=0.8)
    if method == "physical":
        r = P.FWXMProfilePhysical(a, dpmm=dr).gamma(P.FWXMProfilePhysical(b, dpmm=de), **kw)
        if kw.get("return_profiles"):
            r, pa, pb = r
            for tag, p in (("ref", pa), ("eval", pb)):
                for attr in ("values", "x_values", "physical_x_values"):
                    np.testing.assert_array_equal(np.asarray(getattr(p, attr)), GOLDEN[f"{name}:{tag}:{attr}"])
        np.testing.assert_array_equal(r, GOLDEN[name])
    else:
        pa, pb = P.SingleProfile(a, dpmm=dr), P.SingleProfile(b, dpmm=de)
        r = pa.gamma(pb, **kw)
        dta, dose = kw.get("distance_to_agreement", 1), kw.get("dose_to_agreement", 1)
        rest = {k: v for k, v in kw.items() if k not in ("distance_to_agreement", "dose_to_agreement")}
        np.testing.assert_array_equal(r, G.gamma_1d(pa.values, pb.values, pa.x_indices, pb.x_indices, dose, dta, **rest)[0])
        # the profiles' interpolated values come from the SingleProfile engine, which matches the reference to 1e-7 (DESIGN.md §1)
        np.testing.assert_array_equal(np.isnan(r), np.isnan(GOLDEN[name]))
        np.testing.assert_allclose(r, GOLDEN[name], rtol=1e-7, equal_nan=True)


def test_single_profile_needs_dpmm():
    a = profile_signal(101, np.random.default_rng(4100))
    kind, msg = GOLDEN["error:single_profile_no_dpmm"]
    with pytest.raises(ValueError) as info:
        P.SingleProfile(a, dpmm=None).gamma(P.SingleProfile(a, dpmm=2.0))
    assert str(info.value) == msg
