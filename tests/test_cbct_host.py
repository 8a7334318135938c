"""CPU: the CT series reader (core.image.DicomImageStack: discovery, filtering, series choice, sorting, one volume), the host-side
refusals of WinstonLutz.from_cbct, and the numpy oracle of its frames (oracle/cbct_oracle.py) against goldens produced by the
UNMODIFIED reference from_cbct (tests/golden/make_cbct_wl_golden.py)."""
import hashlib
import os
import zipfile

import numpy as np
import pytest

from oracle import cbct_oracle
from pylinac_b200 import dicom
from pylinac_b200 import winston_lutz as wl
from pylinac_b200.core import image
from tests import ct_writer
from tests.golden.cbct_wl_cases import CASES, case_volume

GOLD = np.load("tests/golden/cbct_wl_golden.npz")


def _volume(n=12, h=6, w=10, dtype=np.int16, seed=0):
    rng = np.random.default_rng(seed)
    lo, hi = (-1200, 1500) if dtype == np.int16 else (0, 4000)
    return rng.integers(lo, hi, size=(n, h, w)).astype(dtype)


def test_stack_discovery_filters_sorts_and_views_one_volume(tmp_path):
    vol = _volume()
    order = np.random.default_rng(1).permutation(len(vol))           # files written in shuffled slice order
    top = tmp_path / "series"
    ct_writer.write_series(top, vol[:6], slice_thickness=2.5, pixel_spacing=0.75, order=order[order < 6])
    sub = top / "nested" / "deeper"                                 # the rest one level down: os.walk is recursive
    ct_writer.write_series(sub, vol, slice_thickness=2.5, pixel_spacing=0.75, order=[n for n in order if n >= 6])
    os.rename(sub / "CT0000.dcm", sub / "A.dcm")                    # names do not matter
    # distractors: a text file, a second (smaller) series, a non-image SOP class, a file without a SOP Class UID
    (top / "notes.txt").write_text("not a DICOM file")
    other = _volume(n=3, seed=5)
    ct_writer.write_series(top / "other", other, slice_thickness=1.0, pixel_spacing=1.0, series_uid="1.2.3.999")
    ct_writer.write_ct_slice(top / "rtss.dcm", vol[0], series_uid="1.2.826.0.1.3680043.2.1", z=-50.0, slice_thickness=2.5,
                             pixel_spacing=0.75, sop_class=ct_writer.RT_STRUCTURE_SET_STORAGE)
    ct_writer.write_ct_slice(top / "nosop.dcm", vol[0], series_uid="1.2.826.0.1.3680043.2.1", z=-60.0, slice_thickness=2.5,
                             pixel_spacing=0.75, sop_class=None)
    st = image.DicomImageStack(top, min_number=10, raw_pixels=True)
    assert len(st) == len(vol) and st.volume.shape == vol.shape and st.volume.dtype == np.int16
    np.testing.assert_array_equal(st.volume, vol)
    assert [m.ImagePositionPatient[-1] for m in st.metadatas] == [n * 2.5 for n in range(len(vol))]
    for k in range(len(vol)):
        assert isinstance(st[k], image.DicomImage) and st[k] is st.images[k]
        assert st[k].array.dtype == np.int16 and np.shares_memory(st[k].array, st.volume)
        np.testing.assert_array_equal(st[k].array, vol[k])
    assert st.metadata is st.metadatas[0] and st.metadata.SliceThickness == 2.5 and st.metadata.PixelSpacing == [0.75, 0.75]
    assert st.slice_spacing == 2.5
    # check_uid=False keeps the second series too (sorted into one list by position; every slice has the same shape)
    both = image.DicomImageStack(top, min_number=10, check_uid=False, raw_pixels=True)
    assert len(both) == len(vol) + len(other)


def test_stack_ties_fall_like_numpy_argsort(tmp_path):
    vol = _volume(n=4)
    for k in range(4):       # two slices at every position: np.argsort's (quicksort) order of the equal keys decides
        ct_writer.write_ct_slice(tmp_path / f"s{k}.dcm", vol[k], series_uid="1.2.3", z=float(k // 2), slice_thickness=1.0,
                                 pixel_spacing=1.0)
    paths = [str(tmp_path / f"s{k}.dcm") for k in (3, 1, 2, 0)]
    st = image.DicomImageStack(paths, min_number=1, raw_pixels=True)
    order = np.argsort([float(k // 2) for k in (3, 1, 2, 0)])
    np.testing.assert_array_equal(st.volume, vol[[(3, 1, 2, 0)[i] for i in order]])


def test_stack_rescale_and_dtype_follow_dicom_image(tmp_path):
    vol = _volume(n=3, dtype=np.uint16)
    paths = ct_writer.write_series(tmp_path, vol, slice_thickness=1.0, pixel_spacing=1.0, slope=1.0, intercept=-1024.0)
    st = image.DicomImageStack(paths, min_number=3)
    assert st[1].array.dtype == np.float64
    np.testing.assert_array_equal(st[1].array, vol[1].astype(np.float64) - 1024.0)
    raw = image.DicomImageStack(paths, min_number=3, raw_pixels=True, dtype=np.int32)
    assert raw[2].array.dtype == np.int32
    np.testing.assert_array_equal(raw[2].array, vol[2])


def test_stack_errors(tmp_path):
    (tmp_path / "a.txt").write_text("nothing here")
    with pytest.raises(FileNotFoundError):
        image.DicomImageStack(tmp_path)
    with pytest.raises(FileNotFoundError):
        image.DicomImageStack(tmp_path / "does-not-exist")
    ct_writer.write_series(tmp_path / "s", _volume(n=5), slice_thickness=1.0, pixel_spacing=1.0)
    with pytest.raises(ValueError, match="The minimum number images from the same study were not found"):
        image.DicomImageStack(tmp_path, min_number=6)
    assert len(image.DicomImageStack(tmp_path, min_number=5)) == 5


def test_stack_from_zip(tmp_path):
    vol = _volume(n=4)
    paths = ct_writer.write_series(tmp_path / "s", vol, slice_thickness=1.0, pixel_spacing=1.0, order=[2, 0, 3, 1])
    zpath = tmp_path / "series.zip"
    with zipfile.ZipFile(zpath, "w") as z:
        for p in paths:
            z.write(p, arcname=os.path.join("export", os.path.basename(p)))
    st = image.DicomImageStack.from_zip(zpath, min_number=4, raw_pixels=True)
    np.testing.assert_array_equal(st.volume, vol)


def test_image_storage_table_names_image_classes_only():
    for uid in ("1.2.840.10008.5.1.4.1.1.2", "1.2.840.10008.5.1.4.1.1.2.1", "1.2.840.10008.5.1.4.1.1.4", "1.2.840.10008.5.1.4.1.1.481.1",
                "1.2.840.10008.5.1.4.1.1.7"):
        assert uid in dicom.IMAGE_STORAGE_UIDS
    assert all("Image Storage" in name for name in dicom.IMAGE_STORAGE_UIDS.values())
    for uid in ("1.2.840.10008.5.1.4.1.1.481.3", "1.2.840.10008.5.1.4.1.1.481.2", "1.2.840.10008.5.1.4.1.1.66"):
        assert uid not in dicom.IMAGE_STORAGE_UIDS


def test_from_cbct_refuses_float_hounsfield_frames_before_device_work(tmp_path):
    vol = _volume(n=10, dtype=np.uint16)
    ct_writer.write_series(tmp_path, vol, slice_thickness=1.0, pixel_spacing=1.0, slope=1.0, intercept=-1024.0)
    with pytest.raises(NotImplementedError, match="raw_pixels=True"):
        wl.WinstonLutz.from_cbct(tmp_path)
    ct_writer.write_series(tmp_path / "short", vol[:9], slice_thickness=1.0, pixel_spacing=1.0)
    with pytest.raises(ValueError, match="minimum number"):     # from_cbct asks for at least 10 slices of one series
        wl.WinstonLutz.from_cbct(tmp_path / "short", raw_pixels=True)


@pytest.mark.parametrize("name", CASES)
def test_oracle_frames_match_reference_golden(name):
    vol, st_mm, ps = case_volume(name)
    assert hashlib.sha1(vol.tobytes()).digest() == GOLD[f"{name}/volume_sha1"].tobytes()
    colmax, rowmax = cbct_oracle.projections(vol)
    np.testing.assert_array_equal(colmax, GOLD[f"{name}/colmax"])
    np.testing.assert_array_equal(rowmax, GOLD[f"{name}/rowmax"])
    frames = cbct_oracle.cbct_frames(vol, st_mm, ps)
    for g, f in frames.items():
        assert f.dtype == np.uint16 and list(f.shape) == GOLD[f"{name}/frame_{g}_shape"].tolist()
        assert hashlib.sha1(f.tobytes()).digest() == GOLD[f"{name}/frame_{g}_sha1"].tobytes(), g
