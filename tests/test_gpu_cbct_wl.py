"""GPU: WinstonLutz.from_cbct -- the stack projection (epid_stack_mip), the slice-axis zoom (epid_zoom) and the four views
(epid_cbct_views) bit-identical to the frames the UNMODIFIED reference builds (tests/golden/cbct_wl_golden.npz), and the set
analysis of those frames against the reference's results at the tolerances of test_gpu_wl.py / test_wlset_host.py."""
import hashlib
import os
import zipfile

import numpy as np
import pytest

from tests import ct_writer
from tests.dicom_writer import write_dicom
from tests.golden.cbct_wl_cases import CASES, SPHERE_EXPECT, case_volume
from tests.golden.make_wlset_golden import SCALARS

pytestmark = pytest.mark.gpu

GOLD = np.load("tests/golden/cbct_wl_golden.npz")
POS_TOL_PX = 1e-9
GANTRY_ORDER = (0, 180, 270, 90)      # set order: the reference's file names G=0, G=180, G=270, G=90 sorted


def _series(tmp_path, name, **kw):
    vol, st_mm, ps = case_volume(name)
    order = np.random.default_rng(7).permutation(len(vol))
    ct_writer.write_series(tmp_path / name, vol, slice_thickness=st_mm, pixel_spacing=ps, order=order, z0=-40.0, **kw)
    return tmp_path / name


@pytest.mark.parametrize("shape", [(3, 7, 5), (4, 64, 512), (2, 40, 1024), (2, 33, 2048), (1, 300, 8), (200, 16, 16), (2, 1000, 24),
                                   (3, 130, 250)])
@pytest.mark.parametrize("dtype", [np.int16, np.uint16])
def test_stack_mip_equals_numpy(shape, dtype):
    from pylinac_b200 import _native as nat

    info = np.iinfo(dtype)
    rng = np.random.default_rng(sum(shape))
    vol = rng.integers(info.min, info.max + 1, size=shape).astype(dtype)
    ctx = nat.Context.default()
    b = nat.Batch.upload(ctx, vol)
    colmax, rowmax = nat.stack_mip(ctx, b)
    stack = np.moveaxis(vol, 0, -1)
    c, r = colmax.download(), rowmax.download()
    assert c.dtype == dtype and c.shape == (shape[2], 1, shape[0]) and r.shape == (shape[1], 1, shape[0])
    np.testing.assert_array_equal(c[:, 0], stack.max(axis=0))
    np.testing.assert_array_equal(r[:, 0], stack.max(axis=1))
    for x in (b, colmax, rowmax):
        x.free()


def test_stack_mip_refuses_other_dtypes_and_widths():
    from pylinac_b200 import _native as nat

    ctx = nat.Context.default()
    for vol in (np.zeros((2, 4, 8), np.int32), np.zeros((2, 4, 8), np.float64), np.zeros((1, 2, 2056), np.uint16)):
        b = nat.Batch.upload(ctx, vol)
        with pytest.raises(NotImplementedError):
            nat.stack_mip(ctx, b)
        b.free()


@pytest.mark.parametrize("name", CASES)
def test_projections_and_frames_are_bit_identical_to_reference(name):
    from pylinac_b200 import _native as nat
    from pylinac_b200 import winston_lutz as wl

    vol, st_mm, ps = case_volume(name)
    ctx = nat.Context.default()
    b = nat.Batch.upload(ctx, vol)
    colmax, rowmax = nat.stack_mip(ctx, b)
    np.testing.assert_array_equal(colmax.download()[:, 0], GOLD[f"{name}/colmax"])
    np.testing.assert_array_equal(rowmax.download()[:, 0], GOLD[f"{name}/rowmax"])
    for x in (b, colmax, rowmax):
        x.free()
    groups = wl.cbct_frames(vol, st_mm / ps)
    assert len(groups) == (1 if vol.shape[1] == vol.shape[2] else 2)
    seen = set()
    for batch, idx in groups:
        frames = batch.download()
        batch.free()
        for f, k in zip(frames, idx):
            g = GANTRY_ORDER[k]
            seen.add(g)
            assert list(f.shape) == GOLD[f"{name}/frame_{g}_shape"].tolist()
            assert hashlib.sha1(f.tobytes()).digest() == GOLD[f"{name}/frame_{g}_sha1"].tobytes(), g
    assert seen == set(GANTRY_ORDER)


def _check_against_golden(st, name, tol=1e-7):
    rd = st.results_data()
    for k in SCALARS:
        np.testing.assert_allclose(getattr(rd, k), GOLD[f"{name}/{k}"], rtol=0, atol=tol, err_msg=k)
    sv = st.bb_shift_vector
    np.testing.assert_allclose([sv.x, sv.y, sv.z], GOLD[f"{name}/bb_shift_vector"], rtol=0, atol=tol)
    assert st.dpmm == float(GOLD[f"{name}/dpmm"])
    for im in st.images:
        g = int(round(im.gantry_angle))
        np.testing.assert_allclose([im.bb.x, im.bb.y], GOLD[f"{name}/bb_{g}"], rtol=0, atol=POS_TOL_PX)
        np.testing.assert_allclose([im.field_cax.x, im.field_cax.y], GOLD[f"{name}/field_{g}"], rtol=0, atol=POS_TOL_PX)
        np.testing.assert_allclose([im.epid.x, im.epid.y], GOLD[f"{name}/epid_{g}"], rtol=0, atol=0)
        np.testing.assert_allclose(im.cax2bb_distance, float(GOLD[f"{name}/cax2bb_distance_{g}"]), rtol=0, atol=POS_TOL_PX)


@pytest.mark.parametrize("name", CASES)
def test_from_cbct_matches_reference(tmp_path, name):
    from pylinac_b200 import winston_lutz as wl

    st = wl.WinstonLutz.from_cbct(_series(tmp_path, name), raw_pixels=True)
    assert st.is_from_cbct and [a[0] for a in st._axes] == list(GANTRY_ORDER)
    st.analyze(bb_size_mm=5)            # low_density_bb / open_field forced on, as in the reference
    _check_against_golden(st, name)


@pytest.mark.parametrize("name", list(SPHERE_EXPECT))
def test_sphere_cases_meet_the_reference_expectations(tmp_path, name):
    """TestPerfectCBCT / TestOffset{Left,Down,In}CBCT (tests_basic/test_winstonlutz.py:2186-2218) and the deltas of their mixin
    (:1186-1212)."""
    from pylinac_b200 import winston_lutz as wl

    mx, med, mean, epid_max, shift = SPHERE_EXPECT[name]
    st = wl.WinstonLutz.from_cbct(_series(tmp_path, name), raw_pixels=False)      # no rescale tags: the stored integers
    st.analyze(bb_size_mm=5)
    assert len(st.images) == 4
    assert abs(st.cax2bb_distance("max") - mx) <= 0.15
    assert abs(st.cax2bb_distance("median") - med) <= 0.1
    assert abs(st.cax2bb_distance("mean") - mean) <= 0.1
    assert abs(st.cax2epid_distance("max") - epid_max) <= 0.1
    sv = st.bb_shift_vector
    assert all(abs(a - b) <= 0.15 for a, b in zip((sv.x, sv.y, sv.z), shift)), (sv, shift)
    assert st.gantry_iso_size == pytest.approx(0, abs=0.15) and st.collimator_iso_size == 0 and st.couch_iso_size == 0


def _undated(d):
    if isinstance(d, dict):
        return {k: _undated(v) for k, v in d.items() if k != "date_of_analysis"}
    if isinstance(d, list):
        return [_undated(v) for v in d]
    return d


@pytest.mark.parametrize("name", ["sphere_left5", "int16_negative", "ratio_2p0_0p9"])
def test_from_cbct_equals_winston_lutz_on_the_written_frames(tmp_path, name):
    """The frames written as the DICOM files the reference writes (G=<angle>, ImagePlanePixelSpacing 25.4 / dpi, SID / SAD 1000)
    and loaded with WinstonLutz(directory) give the same set, including the axes that kwargs resolve."""
    from pylinac_b200 import winston_lutz as wl

    vol, st_mm, ps = case_volume(name)
    dpi = 25.4 / ps
    d = tmp_path / "frames"
    d.mkdir()
    groups = wl.cbct_frames(vol, st_mm / ps)
    for batch, idx in groups:
        for f, k in zip(batch.download(), idx):
            g = GANTRY_ORDER[k]
            write_dicom(d / f"G={g}", f, pixel_spacing_mm=25.4 / dpi, sid=1000, sad=1000.0, gantry=float(f"{g:.2f}"), coll=0.0, couch=0.0)
        batch.free()
    series = _series(tmp_path, name)
    for kwargs in ({}, {"axis_mapping": {"G=90": (90, 0, 45)}}, {"use_filenames": True}, {"axes_precision": 0}):
        a = wl.WinstonLutz.from_cbct(series, raw_pixels=True, **kwargs)
        b = wl.WinstonLutz(str(d), **kwargs)
        assert a._axes == b._axes and a.dpmm == b.dpmm, kwargs
        if kwargs.get("use_filenames"):
            continue            # every gantry resolves to missing_axis_value: not a set the solve can place
        a.analyze(bb_size_mm=5)
        b.analyze(bb_size_mm=5, low_density_bb=True, open_field=True)
        assert _undated(a.results_data(as_dict=True)) == _undated(b.results_data(as_dict=True)), kwargs


def test_from_cbct_zip(tmp_path):
    from pylinac_b200 import winston_lutz as wl

    series = _series(tmp_path, "sphere_in5")
    zpath = tmp_path / "cbct.zip"
    with zipfile.ZipFile(zpath, "w") as z:
        for f in sorted(os.listdir(series)):
            z.write(series / f, arcname=f"scan/{f}")
    st = wl.WinstonLutz.from_cbct_zip(zpath, raw_pixels=True)
    st.analyze(bb_size_mm=5)
    _check_against_golden(st, "sphere_in5")
