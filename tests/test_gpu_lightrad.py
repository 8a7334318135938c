"""Light / radiation field coincidence phantoms on the GPU (csrc/lightrad.cu, pylinac_b200/planar_imaging.py) against goldens of the
unmodified reference (tests/golden/lightrad_golden.npz, make_lightrad_golden.py) and against the synthetic frames' true geometry.

The near-edge BBs go through the restated equalize_adapthist of tests/golden/clahe_restated.py when the goldens are made: that operator's
parity with scikit-image itself is UNPINNED.  Their centres (1e-9 px) depend on every equalised pixel of the BB window, which is how
the device CLAHE is checked against the restatement here."""
import os

import numpy as np
import pytest

from pylinac_b200 import _native as nat
from pylinac_b200 import planar_imaging as pi
from pylinac_b200.contrib.quasar import QuasarLightRadScaling
from tests.golden.lightrad_cases import CASES, lightrad_case

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "lightrad_golden.npz"))
CLASSES = {"StandardImagingFC2": pi.StandardImagingFC2, "IMTLRad": pi.IMTLRad, "DoselabRLf": pi.DoselabRLf, "IsoAlign": pi.IsoAlign,
           "SNCFSQA": pi.SNCFSQA, "QuasarLightRadScaling": QuasarLightRadScaling}


def _golden(name):
    return {k.split("/", 1)[1]: G[k] for k in G.files if k.startswith(name + "/")}


def _check_frame(name, fr, g):
    if "error_type" in g:
        with pytest.raises(Exception) as ei:
            fr.raise_for_status()
            fr.bb_centers
        assert type(ei.value).__name__ == str(g["error_type"]), (name, ei.value)
        assert str(ei.value) == str(g["error_message"]), name
        return
    fr.raise_for_status()
    np.testing.assert_allclose([fr.field_center.x, fr.field_center.y], g["field_center"], rtol=0, atol=1e-7, err_msg=name)
    np.testing.assert_allclose([fr.field_width_x, fr.field_width_y], g["field_width"], rtol=0, atol=1e-7, err_msg=name)
    assert list(fr.bb_centers) == [str(k) for k in g["bb_keys"]], name
    np.testing.assert_allclose([[p.x, p.y] for p in fr.bb_centers.values()], g["bb_centers"], rtol=0, atol=1e-9, err_msg=name)
    np.testing.assert_allclose([fr.bb_center.x, fr.bb_center.y], g["bb_center"], rtol=0, atol=1e-9, err_msg=name)
    assert fr.near_edge == list(g["near_edge"]), name
    if "scaling_centers" in g:
        np.testing.assert_allclose([[p.x, p.y] for p in fr.scaling_centers], g["scaling_centers"], rtol=0, atol=1e-9, err_msg=name)


@pytest.mark.parametrize("name", CASES)
def test_lightrad_batch_matches_reference_golden(name):
    c = lightrad_case(name)
    g = _golden(name)
    res = pi.analyze_batch(c["frame"][None], float(g["dpmm"]), CLASSES[c["cls"]], **c["ctor"], **c["analyze"])
    _check_frame(name, res[0], g)


@pytest.mark.parametrize("name", CASES)
def test_lightrad_class_matches_reference_golden(name):
    c = lightrad_case(name)
    g = _golden(name)
    ph = CLASSES[c["cls"]](c["frame"], image_kwargs=dict(dpi=25.4 * c["dpmm"]), **c["ctor"])
    assert ph.image.dpmm == float(g["dpmm"])
    if "error_type" in g:
        with pytest.raises(Exception) as ei:
            ph.analyze(**c["analyze"])
        assert type(ei.value).__name__ == str(g["error_type"]) and str(ei.value) == str(g["error_message"])
        return
    ph.analyze(**c["analyze"])
    np.testing.assert_allclose([ph.field_center.x, ph.field_center.y], g["field_center"], rtol=0, atol=1e-7)
    np.testing.assert_allclose([ph.field_width_x, ph.field_width_y], g["field_width"], rtol=0, atol=1e-7)
    np.testing.assert_allclose([ph.epid_center.x, ph.epid_center.y], g["epid_center"], rtol=0, atol=0)
    np.testing.assert_allclose([ph.field_epid_offset_mm.x, ph.field_epid_offset_mm.y], g["field_epid_offset_mm"], rtol=0, atol=1e-7)
    np.testing.assert_allclose([ph.field_bb_offset_mm.x, ph.field_bb_offset_mm.y], g["field_bb_offset_mm"], rtol=0, atol=1e-7)
    np.testing.assert_allclose([[p.x, p.y] for p in ph.bb_centers.values()], g["bb_centers"], rtol=0, atol=1e-9)
    lines = ph.results(as_list=True)
    ref = [str(s) for s in g["results"]]
    assert lines[0] == ref[0] and lines[2:] == ref[2:]
    rd = ph.results_data()
    np.testing.assert_allclose([rd.field_size_x_mm, rd.field_size_y_mm, rd.field_epid_offset_x_mm, rd.field_epid_offset_y_mm,
                                rd.field_bb_offset_x_mm, rd.field_bb_offset_y_mm], g["results_data"], rtol=0, atol=1e-7)
    if "scaling_centers" in g:
        np.testing.assert_allclose([[p.x, p.y] for p in ph.scaling_centers], g["scaling_centers"], rtol=0, atol=1e-9)


@pytest.mark.parametrize("name", [n for n in CASES if "error_type" not in _golden(n)])
def test_lightrad_matches_synthetic_ground_truth(name):
    """the reference's own deltas (tests_basic/test_planar_imaging.py:1042-1067): field size 0.3 mm, BB-to-field offset 0.2 mm"""
    c = lightrad_case(name)
    t = c["truth"]
    fr = pi.analyze_batch(c["frame"][None], c["dpmm"], CLASSES[c["cls"]], **c["ctor"], **c["analyze"])[0]
    np.testing.assert_allclose([fr.field_width_x, fr.field_width_y], t["field_size_mm"], atol=0.3)
    nbb = len(fr.bb_centers) - (1 if CLASSES[c["cls"]]._virtual_center else 0)
    bb = t["bb_px"][:nbb]
    true_bb_center = bb.mean(axis=0)
    if CLASSES[c["cls"]]._virtual_center:
        true_bb_center = bb[0] - np.array([40 * c["dpmm"], -40 * c["dpmm"]])
    true_offset = (true_bb_center - t["field_center_px"]) / c["dpmm"]
    off = fr.field_bb_offset_mm
    np.testing.assert_allclose([off.x, off.y], true_offset, atol=0.2)


def test_lightrad_mixed_batch_equals_single_frames():
    """FC-2 frames of one shape in one batch: 10x10 and 15x15, near-edge and not, inverted, mismatched, without BBs"""
    names = [n for n in CASES if lightrad_case(n)["cls"] == "StandardImagingFC2" and lightrad_case(n)["frame"].shape == (1280, 1280)
             and not lightrad_case(n)["ctor"] and not lightrad_case(n)["analyze"]]
    assert len(names) >= 6
    frames = np.stack([lightrad_case(n)["frame"] for n in names])
    dpmm = float(_golden(names[0])["dpmm"])
    batch = pi.analyze_batch(frames, dpmm)
    for i, n in enumerate(names):
        one = pi.analyze_batch(frames[i:i + 1], dpmm)
        assert batch.rows[i].tobytes() == one.rows[0].tobytes(), n
        _check_frame(n, batch[i], _golden(n))


def test_lightrad_device_resident_batch():
    names = ["fc2_10_near", "fc2_10_far", "fc2_inverted", "fc2_15_near"]
    frames = np.stack([lightrad_case(n)["frame"] for n in names])
    dpmm = float(_golden(names[0])["dpmm"])
    ctx = nat.Context.default()
    b = nat.Batch.upload(ctx, frames)
    try:
        res = pi.analyze_batch(b, dpmm)
    finally:
        b.free()
    for i, n in enumerate(names):
        _check_frame(n, res[i], _golden(n))


def test_lightrad_batch_larger_than_one_chunk():
    """more frames than one device chunk (64): every frame equals its own one-frame call"""
    names = ["fc2_10_near", "fc2_10_far", "fc2_15", "fc2_no_bb"]
    frames = np.stack([lightrad_case(names[i % len(names)])["frame"] for i in range(70)])
    dpmm = float(_golden(names[0])["dpmm"])
    res = pi.analyze_batch(frames, dpmm)
    singles = {n: pi.analyze_batch(lightrad_case(n)["frame"][None], dpmm).rows[0].tobytes() for n in names}
    for i in range(70):
        assert res.rows[i].tobytes() == singles[names[i % len(names)]], i
