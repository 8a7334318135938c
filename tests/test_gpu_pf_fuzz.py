"""GPU: PicketFence in CUDA against the oracle on seeded RANDOM frames and analyze() arguments (panel, orientation, picket count /
spacing / width, blur, noise, inversion, crop, pre-filter, separate leaves, sag, FWXM height, window width ratio, tolerance).
The oracle is bit-identical to the unmodified reference on the same generator (tests/test_oracle_vs_reference_live.py and a
40-case fuzz run against the live reference); here the CUDA path must agree with it: integers exactly, positions to 1e-6 px."""
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POS_TOL_PX = 1e-6
ERR_TOL_MM = 1e-6


def random_case(seed):
    from oracle import synth

    rng = np.random.default_rng(seed)
    panel = rng.choice(["epid1024", "as1200", "as1000"])
    fr = {"epid1024": synth.epid1024, "as1200": lambda: synth.as1200(1000.0), "as1000": lambda: synth.as1000(1000.0)}[panel]()
    a = synth.picketfence_frame(fr, pickets=int(rng.integers(4, 11)), picket_spacing_mm=int(rng.integers(15, 30)),
                                picket_width_mm=int(rng.integers(2, 6)), picket_offset_error=rng.uniform(-0.8, 0.8, 12),
                                noise_sigma=float(rng.uniform(0.0005, 0.006)), seed=seed,
                                orientation="left_right" if rng.random() < 0.4 else "up_down", blur_mm=float(rng.uniform(0.6, 2.0)))
    if rng.random() < 0.2:
        a = (a.max() - a + a.min()).astype(np.uint16)
    ak, ck = {}, {}
    if rng.random() < 0.3:
        ak["separate_leaves"] = True
        ak["nominal_gap_mm"] = float(rng.integers(2, 6))
    if rng.random() < 0.3:
        ak["sag_adjustment"] = float(rng.uniform(-2, 2))
    if rng.random() < 0.3:
        ak["fwxm"] = int(rng.integers(30, 80))
    if rng.random() < 0.3:
        ak["leaf_analysis_width_ratio"] = float(rng.uniform(0.3, 0.8))
    if rng.random() < 0.3:
        ak["tolerance"] = float(rng.uniform(0.1, 0.6))
    if rng.random() < 0.3:
        ck["crop_mm"] = int(rng.integers(0, 8))
    if rng.random() < 0.2:
        ck["filter"] = int(rng.choice([3, 5]))
    return a, 1 / fr.pixel_size, ck, ak


@pytest.mark.parametrize("seed", range(3000, 3024))
def test_pf_random_case_matches_oracle(seed):
    from oracle import pf_oracle
    from pylinac_b200 import picketfence as pf

    a, dpmm, ck, ak = random_case(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            o = pf_oracle.pf_analyze(a, dpmm, **ck, **ak)
        except (ValueError, TypeError, IndexError) as e:
            o = e
    r = pf.analyze_batch(a[None], dpmm, **ck, **ak)[0]
    if isinstance(o, Exception):
        assert r.status != 0
        with pytest.raises(type(o)) as ei:
            r.raise_for_status()
        assert type(ei.value) is type(o), (r.status, o)
        return
    assert r.status == 0, (r.status, ck, ak)
    assert int(r.s["orientation"]) == int(o["orientation"])
    assert sorted(int(v) for v in r.picket_idx) == sorted(int(v) for v in o["picket_idx"])
    assert int(r.s["n_meas"]) == o["n_meas"]
    assert np.array_equal(r.m["leaf_num"], o["meas_leaf"]) and np.array_equal(r.m["picket"], o["meas_picket"])
    npos = np.asarray(o["meas_position"]).shape[1]
    np.testing.assert_allclose(r.m["position"][:, :npos], o["meas_position"], rtol=0, atol=POS_TOL_PX)
    np.testing.assert_allclose(r.m["error"][:, :npos], o["meas_error"], rtol=0, atol=ERR_TOL_MM)
    assert bool(r.s["passed"]) == bool(o["passed"])
    np.testing.assert_allclose(float(r.s["max_error_mm"]), float(o["max_error"]), rtol=0, atol=ERR_TOL_MM)
    np.testing.assert_allclose(float(r.s["percent_passing"]), float(o["percent_passing"]), rtol=0, atol=1e-9)
    # everything else the oracle returns: the front end's decisions, the fits and the per-picket aggregates
    s = r.s
    npk = int(s["n_pickets"])
    assert npk == o["number_of_pickets"]
    assert int(s["noise_median_passes"]) == o["noise_median_passes"]
    assert bool(s["corner_inverted"]) == o["corner_inverted"]
    assert (int(s["height"]), int(s["width"])) == tuple(o["shape"])
    assert int(s["n_leaves_removed"]) == o["n_leaves_removed"]
    np.testing.assert_array_equal(s["picket_spacing_px"], o["picket_spacing"])
    np.testing.assert_allclose(r.m["width_mm"], o["meas_width_mm"], rtol=0, atol=ERR_TOL_MM)
    np.testing.assert_allclose(s["fit_slope"][:npk], o["fits"][:, 0], rtol=0, atol=1e-9)
    np.testing.assert_allclose(s["fit_intercept"][:npk], o["fits"][:, 1], rtol=0, atol=POS_TOL_PX)
    np.testing.assert_allclose(s["offsets_from_cax_mm"][:npk], o["offsets_from_cax_mm"], rtol=0, atol=ERR_TOL_MM)
    np.testing.assert_allclose(float(s["cax_px"]) / dpmm, o["cax_mm"], rtol=0, atol=1e-12)
    for key, ok in [("abs_median_error_mm", "abs_median_error"), ("mean_picket_spacing_mm", "mean_picket_spacing"), ("mlc_skew", "mlc_skew")]:
        np.testing.assert_allclose(float(s[key]), float(o[ok]), rtol=0, atol=ERR_TOL_MM, err_msg=key)
    pw = np.stack([s["picket_width_max"][:npk], s["picket_width_mean"][:npk], s["picket_width_median"][:npk], s["picket_width_min"][:npk]], axis=1)
    np.testing.assert_allclose(pw, o["picket_widths"], rtol=0, atol=ERR_TOL_MM)
    assert int(s["max_error_picket"]) == o["max_error_picket"]
    assert str(r.max_error_leaf) == str(o["max_error_leaf"])
    assert [str(x) for x in r.failed_leaves()] == [str(x) for x in o["failed_leaves"]]
