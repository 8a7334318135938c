"""CPU: the ACR CT host logic -- the epid_ct_region layout, region objects and the roll's sorting, eccentricity from exact moments,
the relative MTF against scipy's interp1d, z_position and the scan-extent check, and the shared roi_settings."""
import os
import subprocess
import types
import warnings

import numpy as np
import pytest
from scipy.interpolate import interp1d

from pylinac_b200 import _native as nat
from pylinac_b200 import acr, ct
from pylinac_b200.core.mtf import MTF

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "epid.h")


def test_ct_region_layout_matches_header(tmp_path):
    d = nat.CT_REGION_DTYPE
    prints = ['std::printf("sizeof %zu\\n", sizeof(epid_ct_region));']
    prints += [f'std::printf("{m} %zu %zu\\n", offsetof(epid_ct_region, {m}), sizeof(epid_ct_region::{m}));' for m in d.names]
    src = tmp_path / "region_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "region_layout")], check=True)
    out = subprocess.run([str(tmp_path / "region_layout")], check=True, capture_output=True, text=True).stdout
    header = {m: tuple(int(v) for v in vals) for m, *vals in (line.split() for line in out.splitlines())}
    assert header.pop("sizeof") == (d.itemsize,)
    assert header == {m: (d.fields[m][1], d.fields[m][0].itemsize) for m in d.names}


def _row(mask, label=1):
    """the epid_ct_region row of a boolean mask (one region)"""
    rr, cc = np.nonzero(mask)
    r0, c0 = rr.min(), cc.min()
    row = np.zeros((), nat.CT_REGION_DTYPE)
    row["label"], row["first"], row["area"], row["filled_area"] = label, rr[0] * mask.shape[1] + cc[0], len(rr), len(rr)
    row["bbox"] = (r0, c0, rr.max() + 1, cc.max() + 1)
    row["sum_r"], row["sum_c"] = rr.sum(), cc.sum()
    row["m_rr"], row["m_cc"], row["m_rc"] = ((rr - r0) ** 2).sum(), ((cc - c0) ** 2).sum(), ((rr - r0) * (cc - c0)).sum()
    return row


@pytest.mark.parametrize("seed", range(8))
def test_eccentricity_and_centroid_from_exact_moments(seed):
    from oracle import acr_oracle

    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:60, 0:70]
    a, b, t = rng.uniform(3, 20), rng.uniform(3, 20), rng.uniform(0, np.pi)
    u, v = (xx - 35) * np.cos(t) + (yy - 30) * np.sin(t), -(xx - 35) * np.sin(t) + (yy - 30) * np.cos(t)
    mask = (u / a) ** 2 + (v / b) ** 2 < 1
    reg = ct.Region(_row(mask))
    lab = mask.astype(int)
    ref = acr_oracle.regionprops(lab)[0]
    assert reg.centroid == ref.centroid and reg.bbox == ref.bbox and reg.bbox_area == ref.bbox_area
    assert abs(reg.eccentricity - ref.eccentricity) <= 1e-9


def test_roll_sorts_regions_with_a_custom_key(monkeypatch):
    """find_phantom_roll keeps the reference's filters and stable sorts: func picks two, the top one comes first"""
    regions = []
    for label, (cy, cx, box) in enumerate([(10.0, 50.0, 200), (40.0, 52.0, 150), (70.0, 49.0, 150), (90.0, 90.0, 100)], start=1):
        regions.append(types.SimpleNamespace(label=label, filled_area=400, eccentricity=0.1, centroid=(cy, cx), bbox_area=box))
    regions[3].eccentricity = 0.7                               # excluded
    ph = object.__new__(acr.ACRCT)
    ph.origin_slice, ph.roll_slice_offset = 5, 0
    ph.dicom_stack = types.SimpleNamespace(slice_spacing=1.0)
    monkeypatch.setattr(acr.ACRCT, "mm_per_pixel", property(lambda self: 1.0))
    monkeypatch.setattr(ct, "Slice", lambda *a, **k: types.SimpleNamespace(phan_center=types.SimpleNamespace(x=50.0)))
    monkeypatch.setattr(acr.ACRCT, "get_regions", lambda self, z: regions)
    # bbox_area: labels 2 and 3 (150, 150) in label order, top first
    assert ph.find_phantom_roll() == np.rad2deg(np.arctan2(30.0, -3.0)) - 90
    # the default key: closest to the centre in x, labels 3 then 1
    assert ct.CatPhanBase.find_phantom_roll(ph) == np.rad2deg(np.arctan2(60.0, -1.0)) - 90
    regions[1].filled_area = regions[2].filled_area = 10    # too small: one bubble left
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        assert ph.find_phantom_roll() == 0.0
    assert [str(w.message) for w in caught] == ["Could not determine phantom roll. Setting roll to 0."]


def _scipy_mtf50(norm, x):
    return float(interp1d(list(norm.values()), list(norm.keys()), fill_value="extrapolate")(x / 100))


@pytest.mark.parametrize("seed", range(10))
def test_mtf_matches_scipy(seed):
    rng = np.random.default_rng(seed)
    n = rng.integers(2, 9)
    spacings = list(rng.permutation(np.round(rng.uniform(0.1, 2.0, n), 2)))
    maxima = list(rng.uniform(500, 1500, n))
    minima = list(rng.uniform(-500, 400, n))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        m = MTF(spacings, maxima, minima)
        for x in (10, 30, 50, 80, 100):
            assert m.relative_resolution(x) == _scipy_mtf50(m.norm_mtfs, x)
    assert list(m.norm_mtfs) == sorted(spacings)
    rising = np.max(np.diff(list(m.norm_mtfs.values()))) > 0
    assert any("does not drop monotonically" in str(w.message) for w in caught) == rising


def test_mtf_extrapolation_warning_and_bounds():
    m = MTF([0.1, 0.2, 0.3], [100.0, 100.0, 100.0], [0.0, 30.0, 60.0])
    with pytest.warns(UserWarning, match="MTF resolution wasn't calculated for 5%"):
        assert m.relative_resolution(5) > 0.3
    with pytest.raises(ValueError):
        m.relative_resolution(101)
    with pytest.raises(ValueError, match="greater than 1"):
        MTF([0.1], [1.0], [0.0])


def test_z_position_and_scan_extent():
    assert ct.z_position(types.SimpleNamespace(ImagePositionPatient=[0, 0, -12.5])) == -12.5
    assert ct.z_position(types.SimpleNamespace(SliceLocation=3.0)) == 3.0
    ph = object.__new__(acr.ACRCT)
    ph.dicom_stack = types.SimpleNamespace(metadatas=[types.SimpleNamespace(ImagePositionPatient=[0, 0, z * 2.5]) for z in range(45)])
    ph.origin_slice = 4                                          # z 10: modules up to 110, scan to 110
    assert ph._ensure_physical_scan_extent()
    ph.origin_slice = 5                                          # up to 112.5
    assert not ph._ensure_physical_scan_extent()
    ph.dicom_stack.metadatas[-1].ImagePositionPatient[-1] = 112.46     # rounds to 112.5
    assert ph._ensure_physical_scan_extent()


def test_results_formatting():
    ph = object.__new__(acr.ACRCT)
    roi = lambda v, s=1.0: types.SimpleNamespace(pixel_value=v, std=s)  # noqa: E731
    ph.ct_calibration_module = types.SimpleNamespace(roi_vals_as_str="Air: -1000.0")
    ph.low_contrast_module = types.SimpleNamespace(cnr=lambda: 1.23456)
    ph.uniformity_module = types.SimpleNamespace(roi_vals_as_str="Top: 0.0", rois={"Center": roi(0.0, 4.567)})
    ph.spatial_resolution_module = types.SimpleNamespace(mtf=types.SimpleNamespace(relative_resolution=lambda x: 0.905))
    assert ph.results() == ("\n - ACR CT 464 QA Test - \nHU ROIs: Air: -1000.0\nContrast to Noise Ratio: 1.23\nUniformity ROIs: Top: 0.0\n"
                            "Uniformity Center ROI standard deviation: 4.57\nMTF 50% (lp/mm): 0.91\n")
