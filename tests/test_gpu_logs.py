"""GPU: machine-log fluence maps (epid_log_fluence) bit-identical to the unmodified reference's goldens and to the numpy oracle,
the fluence gamma against the goldens, and batches of mixed trajectory logs / Dynalogs against the same logs alone."""
import hashlib
import os

import numpy as np
import pytest

from oracle import log_oracle
from pylinac_b200 import log_analyzer as la
from tests import log_writer as lw
from tests.golden.log_cases import CASES, GAMMA_SETTINGS, MAP_SETTINGS, SUB_COLS, SUB_ROWS, SUBBEAM_SETTINGS, write_case

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "log_golden.npz"))
FLUENCE_CASES = [c for c in CASES if c != "tlog_no_mu"]


def sha1(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(a, dtype=np.float64).tobytes()).digest(), np.uint8)


def check_map(key, a):
    assert tuple(G[f"{key}/shape"]) == a.shape, key
    assert np.array_equal(G[f"{key}/sub"], a[SUB_ROWS, SUB_COLS]), key
    assert np.array_equal(G[f"{key}/sha1"], sha1(a)), key


def same_float(a, b, rtol=1e-12):
    a, b = float(a), float(b)
    if np.isnan(a) or np.isnan(b):
        return np.isnan(a) and np.isnan(b)
    return abs(a - b) <= rtol * max(abs(b), 1e-300)


@pytest.mark.parametrize("name", FLUENCE_CASES)
def test_fluence_maps_match_reference(tmp_path, name):
    log = la.load_log(write_case(name, tmp_path))
    for res, eq in MAP_SETTINGS:
        for kind in ("actual", "expected"):
            check_map(f"{name}/map/{kind}/{res}/{int(eq)}", getattr(log.fluence, kind).calc_map(res, eq))


@pytest.mark.parametrize("name", [c for c in CASES if c.startswith("tlog")])
def test_subbeam_fluence_maps_match_reference(tmp_path, name):
    log = la.load_log(write_case(name, tmp_path))
    for k, s in enumerate(log.subbeams):
        for res, eq in SUBBEAM_SETTINGS:
            for kind in ("actual", "expected"):
                check_map(f"{name}/subbeam{k}/map/{kind}/{res}/{int(eq)}", getattr(s.fluence, kind).calc_map(res, eq))


@pytest.mark.parametrize("name", FLUENCE_CASES)
def test_gamma_matches_reference(tmp_path, name):
    log = la.load_log(write_case(name, tmp_path))
    for k, (doseTA, distTA, threshold, res) in enumerate(GAMMA_SETTINGS):
        log.fluence.actual.calc_map(res, False)
        log.fluence.expected.calc_map(res, False)
        g = log.fluence.gamma.calc_map(doseTA, distTA, threshold, res)
        key = f"{name}/gamma{k}"
        assert tuple(G[f"{key}/shape"]) == g.shape
        # epid_gamma's float32 gradient (hypotf) may differ from numpy's by an ulp: the tolerance of its own tests
        np.testing.assert_allclose(g[SUB_ROWS, SUB_COLS], G[f"{key}/sub"], rtol=1e-6, atol=1e-12)
        avg, pct = G[f"{key}/avg_pct"]
        assert same_float(log.fluence.gamma.avg_gamma, avg, 1e-6), (log.fluence.gamma.avg_gamma, avg)
        got_pct = float(log.fluence.gamma.pass_prcnt)
        assert (np.isnan(got_pct) and np.isnan(pct)) or abs(got_pct - pct) <= 100 * 2 / g.size, (got_pct, pct)   # <= 2 pixels
        assert np.abs(log.fluence.gamma.histogram()[0] - G[f"{key}/histogram"]).max() <= 2


def _mixed_dir(tmp_path):
    paths = []
    for name in ("tlog_v21_millennium", "dlog_regular", "tlog_v30_hd_subbeams", "dlog_vmat", "tlog_v40_metadata", "tlog_static",
                 "tlog_no_mu"):
        paths.append(write_case(name, tmp_path))
    return paths


def test_batch_of_mixed_logs_equals_each_log_alone(tmp_path):
    paths = _mixed_dir(tmp_path)
    rows = la.analyze_batch(paths, keep_maps=True)
    for p, r in zip(paths, rows):
        alone = la.load_log(p)
        assert r.treatment_type == alone.treatment_type
        if not hasattr(alone, "fluence"):
            assert r.avg_gamma is None and r.pass_prcnt is None
            continue
        alone.fluence.gamma.calc_map()
        assert np.array_equal(r.log.fluence.actual.array, alone.fluence.actual.array)
        assert np.array_equal(r.log.fluence.expected.array, alone.fluence.expected.array)
        assert np.array_equal(r.log.fluence.gamma.array, alone.fluence.gamma.array)
        assert same_float(r.avg_gamma, alone.fluence.gamma.avg_gamma) and same_float(r.pass_prcnt, alone.fluence.gamma.pass_prcnt)
        mlc = alone.axis_data.mlc
        assert (r.rms_avg, r.rms_max, r.error_p95) == (mlc.get_RMS_avg(), mlc.get_RMS_max(), mlc.get_error_percentile(95))


@pytest.mark.parametrize("names", [("tlog_v21_millennium", "tlog_v40_metadata", "tlog_static"),
                                   ("tlog_v21_millennium", "dlog_regular", "tlog_static")])
def test_machine_logs_average_the_golden_gammas(tmp_path, names):
    """MachineLogs(dir).avg_gamma() / avg_gamma_pct(): the mean of the reference's per-log values (dlog_regular's pass percent is
    nan in the reference -- every gamma pixel is nan -- and so is the mean)"""
    for name in names:
        write_case(name, tmp_path)
    logs = la.MachineLogs(str(tmp_path))
    n_d = sum(n.startswith("dlog") for n in names)
    assert (logs.num_logs, logs.num_tlogs, logs.num_dlogs) == (len(names), len(names) - n_d, n_d)
    want = np.array([G[f"{n}/gamma0/avg_pct"] for n in names])
    got_pct, got_avg = logs.avg_gamma_pct(), logs.avg_gamma()
    exp_avg, exp_pct = want[:, 0].mean(), want[:, 1].mean()
    assert same_float(got_avg, exp_avg, 1e-6), (got_avg, exp_avg)
    assert (np.isnan(got_pct) and np.isnan(exp_pct)) or abs(got_pct - exp_pct) <= 100 * 2 / (60 * 4000), (got_pct, exp_pct)


def test_spot_check_single_log_gamma(tmp_path):
    """load_log(path).fluence.gamma.calc_map() gives the golden pass percent"""
    log = la.load_log(write_case("tlog_v40_metadata", tmp_path))
    log.fluence.gamma.calc_map()
    assert abs(float(log.fluence.gamma.pass_prcnt) - G["tlog_v40_metadata/gamma0/avg_pct"][1]) <= 100 * 2 / (60 * 4000)


def test_seeded_fuzz_against_the_oracle(tmp_path):
    rng = np.random.default_rng(2026)
    paths = []
    for i in range(48):
        nsnap = int(rng.integers(40, 400))
        kw = dict(leaf_cm=float(rng.uniform(5, 24)), jaw_x=float(rng.uniform(1, 21)), jaw_y=float(rng.uniform(1, 12)),
                  static_pairs=tuple(rng.choice(60, int(rng.integers(0, 6)), replace=False)),
                  crossed_pairs=tuple(rng.choice(60, int(rng.integers(0, 4)), replace=False)), holds=int(rng.integers(0, 3)),
                  mu_total=float(rng.choice([0.2, 50.0, 300.0, 25000.0])))
        cols = lw.vmat_delivery(nsnap, 1000 + i, **kw)
        if i % 4 == 3:
            paths.append(lw.write_dlog_pair(tmp_path, f"F{i}_fz", cols, vmat=bool(i % 8 == 7))[0])
        else:
            nsub = int(rng.integers(1, 4))
            subs = tuple((int(c), f"S{c}") for c in sorted(rng.choice(50, nsub, replace=False)))
            paths.append(lw.write_tlog(os.path.join(tmp_path, f"F{i}_fz.bin"), cols, version=float(rng.choice([2.1, 3.0, 4.0])),
                                       mlc_model=int(rng.choice([2, 3])), subbeams=((0, "S0"),) + subs[1:]))
    res = float(rng.choice([0.1, 0.25, 0.5, 0.7]))
    logs = la._read_all(paths, True)
    with_fluence = [lg for lg in logs if hasattr(lg, "fluence")]
    a, e = la._compute_fluences([(lg.fluence, lg.fluence.actual._src()) for lg in with_fluence], res, False)
    ha, he = a.host(), e.host()
    for i, lg in enumerate(with_fluence):
        assert np.array_equal(ha[i], log_oracle.fluence_of(lg.fluence.actual, res)), paths[logs.index(lg)]
        assert np.array_equal(he[i], log_oracle.fluence_of(lg.fluence.expected, res)), paths[logs.index(lg)]
    # subbeam fluences of the same logs, one launch with equal_aspect (mixed MLC models -> one launch per map height)
    items = [(s.fluence, s.fluence.actual._src()) for lg in logs if isinstance(lg, la.TrajectoryLog) for s in lg.subbeams]
    for hd in (False, True):
        part = [it for it in items if it[0].actual._mlc.hdmlc == hd]
        if not part:
            continue
        a, e = la._compute_fluences(part, res, True)
        for i, (fs, _) in enumerate(part):
            assert np.array_equal(a.host()[i], log_oracle.fluence_of(fs.actual, res, True))
            assert np.array_equal(e.host()[i], log_oracle.fluence_of(fs.expected, res, True))


def test_long_logs_and_fine_resolution_against_the_oracle(tmp_path):
    """k_log_fluence stages beam-on snapshots 1024 at a time and covers 4096 columns per group: beam-on counts of exactly 1024 and
    2048, one past a chunk (1025) and several chunks (trajectory logs with beam holds, a Dynalog), at 0.08 mm (5000 columns: a
    second, partial column group) and with equal_aspect, bit for bit against the numpy oracle"""
    paths = []
    for i, (nsnap, holds) in enumerate(((1024, 0), (1025, 0), (2048, 0), (3000, 2), (2600, 1))):
        cols = lw.vmat_delivery(nsnap, 3000 + i, holds=holds, static_pairs=(5, 33), crossed_pairs=(20,), leaf_cm=22.0, jaw_x=20.5)
        if i == 4:
            paths.append(lw.write_dlog_pair(tmp_path, f"L{i}_long", cols, beam_off=range(100, 140))[0])
        else:
            paths.append(lw.write_tlog(os.path.join(tmp_path, f"L{i}_long.bin"), cols, version=3.0, mlc_model=2 + (i == 1)))
    logs = la._read_all(paths, True)
    nbeam = [len(lg.axis_data.mlc.snapshot_idx) for lg in logs]
    assert {1024, 1025, 2048} <= set(nbeam) and max(nbeam) > 2048, nbeam
    for res, eq in ((0.08, False), (0.3, True)):
        for hd in (False, True):
            part = [lg for lg in logs if lg.axis_data.mlc.hdmlc == hd]
            a, e = la._compute_fluences([(lg.fluence, lg.fluence.actual._src()) for lg in part], res, eq)
            for i, lg in enumerate(part):
                assert np.array_equal(a.host()[i], log_oracle.fluence_of(lg.fluence.actual, res, eq)), (lg.filename, res, eq)
                assert np.array_equal(e.host()[i], log_oracle.fluence_of(lg.fluence.expected, res, eq)), (lg.filename, res, eq)
            a.batch.free()
            e.batch.free()


def test_single_kind_map_whose_mu_stays_below_half_is_zero(tmp_path):
    """calc_map of the expected fluence when only the expected MU stays below 0.5 (the actual one does not): the reference's zero map"""
    cols = lw.vmat_delivery(300, 41)
    mu_e, mu_a = cols["mu"]
    cols["mu"] = (mu_e * 0.002, mu_a)
    log = la.load_log(lw.write_tlog(os.path.join(tmp_path, "P41_lowmu.bin"), cols, version=3.0))
    assert log.fluence.expected.calc_map(0.5).shape == (60, 800) and not log.fluence.expected.array.any()
    assert np.array_equal(log.fluence.actual.calc_map(0.5), log_oracle.fluence_of(log.fluence.actual, 0.5))


def test_batch_without_kept_maps_gives_the_same_numbers(tmp_path):
    paths = [write_case(n, tmp_path) for n in ("tlog_v21_millennium", "dlog_regular", "tlog_v40_metadata")]
    kept = la.analyze_batch(paths, keep_maps=True)
    freed = la.analyze_batch(paths)
    for k, f in zip(kept, freed):
        assert same_float(k.avg_gamma, f.avg_gamma) and same_float(k.pass_prcnt, f.pass_prcnt)
        assert not f.log.fluence.actual.is_map_calced() and not f.log.fluence.gamma.is_map_calced()
