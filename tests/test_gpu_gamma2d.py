"""GPU: core.gamma.gamma_2d / gamma_2d_batch against the reference's goldens and the vectorised oracle, bit for bit (nan in the
same places), with and without the early exit, in batches across chunk boundaries, and the per-pair statistics."""
import os

import numpy as np
import pytest

from oracle import gamma2d_oracle
from pylinac_b200 import _native as nat
from pylinac_b200.core import gamma as G
from tests.golden.gamma2d_cases import CASES, case_pair

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "gamma2d_golden.npz"))
DTYPES = [np.uint16, np.int32, np.float32, np.float64, (np.float32, np.int32), (np.float32, np.uint16), (np.uint16, np.float32)]


def _pair(rng, shape, dtypes, eshape=None, special=True):
    rdt, edt = dtypes if isinstance(dtypes, tuple) else (dtypes, dtypes)
    eshape = eshape or shape
    yy, xx = np.mgrid[0:eshape[0], 0:eshape[1]].astype(np.float64)
    cy, cx = rng.uniform(0, eshape[0]), rng.uniform(0, eshape[1])
    s = rng.uniform(4, 30)
    base = 2000 * np.exp(-(((yy - cy) / s) ** 2 + ((xx - cx) / (1.3 * s)) ** 2)) + 50
    ev = base * rng.uniform(0.97, 1.03) + rng.normal(0, 15, eshape)
    ref = np.roll(base, (int(rng.integers(-2, 3)), int(rng.integers(-2, 3))), axis=(0, 1))[:shape[0], :shape[1]] + rng.normal(0, 15, shape)
    if special and np.issubdtype(edt, np.floating):
        ev[rng.random(eshape) < 0.01] = np.nan
        ev[rng.random(eshape) < 0.005] = np.inf

    def cast(a, dt):
        return np.round(a).clip(0, 60000).astype(dt) if np.issubdtype(dt, np.integer) else a.astype(dt)

    return cast(ref, rdt), cast(ev, edt)


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_reference_bit_for_bit(name):
    ref, ev, kw = case_pair(name)
    np.testing.assert_array_equal(G.gamma_2d(ref, ev, **kw), GOLDEN[name])
    np.testing.assert_array_equal(G.gamma_2d_batch(ref[None], ev[None], **kw, full_search=True)[0], GOLDEN[name])


@pytest.mark.parametrize("global_dose", [True, False])
def test_fuzz_every_dta_against_the_oracle(global_dose):
    rng = np.random.default_rng(7 + global_dose)
    for dta in range(1, 41):
        h, w = int(rng.integers(9, 75)), int(rng.integers(9, 75))
        if h % 8 == 0:
            h += 1
        if w % 32 == 0:
            w += 1
        dtypes = DTYPES[dta % len(DTYPES)]
        eshape = (h, w) if not global_dose or dta % 3 else (h + int(rng.integers(0, 9)), w + int(rng.integers(0, 9)))
        pairs = [_pair(rng, (h, w), dtypes, eshape) for _ in range(2)]
        kw = dict(dose_to_agreement=float(rng.choice([0.5, 1, 2, 3])), distance_to_agreement=dta,
                  gamma_cap_value=float(rng.choice([1, 1.5, 2])), global_dose=global_dose, dose_threshold=float(rng.choice([0, 5, 20])),
                  fill_value=float(rng.choice([np.nan, 0.0])))
        got = G.gamma_2d_batch(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), **kw)
        for k, (ref, ev) in enumerate(pairs):
            np.testing.assert_array_equal(got[k], gamma2d_oracle.gamma_2d(ref, ev, **kw), err_msg=f"dta {dta} pair {k} {dtypes}")


@pytest.mark.parametrize("dta", [1, 3, 10, 20, 40])
@pytest.mark.parametrize("global_dose", [True, False])
def test_early_exit_changes_nothing(dta, global_dose):
    rng = np.random.default_rng(dta)
    pairs = [_pair(rng, (131, 97), np.float64) for _ in range(3)] + [_pair(rng, (131, 97), np.float32) for _ in range(3)]
    for dt in (np.float64, np.float32):
        refs = np.stack([p[0] for p in pairs if p[0].dtype == dt])
        evs = np.stack([p[1] for p in pairs if p[1].dtype == dt])
        fast = G.gamma_2d_batch(refs, evs, distance_to_agreement=dta, global_dose=global_dose, dose_threshold=0)
        full = G.gamma_2d_batch(refs, evs, distance_to_agreement=dta, global_dose=global_dose, dose_threshold=0, full_search=True)
        np.testing.assert_array_equal(fast, full)


def test_batch_equals_pairs_one_by_one_across_chunks(monkeypatch):
    rng = np.random.default_rng(11)
    pairs = [_pair(rng, (45, 67), np.uint16, eshape=(50, 70)) for _ in range(7)]
    refs, evs = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    kw = dict(distance_to_agreement=4, dose_threshold=10)
    single = np.stack([G.gamma_2d(r, e, **kw) for r, e in pairs])
    monkeypatch.setattr(G, "_CHUNK_PIXELS", 3 * (45 * 67 + 50 * 70))      # chunks of 3, 3 and 1 pairs
    np.testing.assert_array_equal(G.gamma_2d_batch(refs, evs, **kw), single)
    ctx = nat.Context.default()
    with nat.Batch.upload(ctx, refs) as rb, nat.Batch.upload(ctx, evs) as eb:
        maps = G.gamma_2d_batch(rb, eb, **kw, device=True)
        with maps:
            np.testing.assert_array_equal(maps.download(), single)
        np.testing.assert_array_equal(G.gamma_2d_batch(rb, evs, **kw), single)


@pytest.mark.parametrize("fill_value", [np.nan, 0.0])
@pytest.mark.parametrize("device", [False, True])
def test_stats_equal_numpy_on_the_map(fill_value, device, monkeypatch):
    rng = np.random.default_rng(5)
    pairs = [_pair(rng, (83, 71), np.float64) for _ in range(5)]
    pairs[2][0][:] = 0                                          # nothing above the threshold: nothing evaluated
    refs, evs = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    monkeypatch.setattr(G, "_CHUNK_PIXELS", 2 * 2 * 83 * 71)
    maps, st = G.gamma_2d_batch(refs, evs, distance_to_agreement=3, fill_value=fill_value, stats=True, device=device)
    if device:
        with maps:
            maps = maps.download()
    for k in range(len(pairs)):
        g = maps[k]
        valid = g[~np.isnan(g)]
        assert st["evaluated"][k] == valid.size
        if valid.size:
            assert st["mean"][k] == pytest.approx(valid.mean(), rel=1e-12)
            assert st["pass_rate"][k] == np.count_nonzero(valid < 1) / valid.size * 100
        else:
            assert np.isnan(st["mean"][k]) and np.isnan(st["pass_rate"][k])


def test_float32_follows_numpy_promotion():
    """float32 pairs normalise, subtract and square in float32 (the reference under numpy 2); computing them in float64 differs."""
    rng = np.random.default_rng(3)
    ref, ev = _pair(rng, (97, 89), np.float32, special=False)
    for global_dose in (True, False):
        kw = dict(distance_to_agreement=3, global_dose=global_dose, dose_to_agreement=0.7, dose_threshold=0)
        got = G.gamma_2d(ref, ev, **kw)
        np.testing.assert_array_equal(got, gamma2d_oracle.gamma_2d(ref, ev, **kw))
        wide = G.gamma_2d(ref.astype(np.float64), ev.astype(np.float64), **kw)
        assert np.any(got != wide)
