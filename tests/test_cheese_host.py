"""CPU: the cheese phantoms' series reading and argument errors, the unbuilt localization branch, and the epid_ct_slice layout."""
import os
import subprocess

import numpy as np
import pytest

from pylinac_b200 import _native as nat
from pylinac_b200 import cheese

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "epid.h")


def test_ct_slice_layout_matches_header(tmp_path):
    d = nat.CT_SLICE_DTYPE
    prints = ['std::printf("sizeof %zu\\n", sizeof(epid_ct_slice));']
    prints += [f'std::printf("{m} %zu %zu\\n", offsetof(epid_ct_slice, {m}), sizeof(epid_ct_slice::{m}));' for m in d.names]
    src = tmp_path / "ct_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "epid.h"\nint main() {\n' + "\n".join(prints) + "\nreturn 0;\n}\n")
    subprocess.run(["c++", "-std=c++17", "-I", os.path.dirname(HEADER), str(src), "-o", str(tmp_path / "ct_layout")], check=True)
    out = subprocess.run([str(tmp_path / "ct_layout")], check=True, capture_output=True, text=True).stdout
    header = {m: tuple(int(v) for v in vals) for m, *vals in (line.split() for line in out.splitlines())}
    assert header.pop("sizeof") == (d.itemsize,)
    assert header == {m: (d.fields[m][1], d.fields[m][0].itemsize) for m in d.names}


def test_not_a_directory(tmp_path):
    with pytest.raises(NotADirectoryError, match="Path given was not a Directory/Folder"):
        cheese.TomoCheese(str(tmp_path / "missing"))


def test_memory_efficient_mode_is_not_implemented(tmp_path):
    with pytest.raises(NotImplementedError, match="memory_efficient_mode"):
        cheese.CIRS062M(str(tmp_path), memory_efficient_mode=True)


def test_too_few_images(tmp_path):
    from tests.ct_writer import write_series

    write_series(tmp_path, np.zeros((3, 16, 16), np.int16), slice_thickness=1.0, pixel_spacing=1.0)
    with pytest.raises(ValueError, match="minimum number images"):
        cheese.TomoCheese(str(tmp_path))


def test_series_is_read_in_z_order(tmp_path):
    from tests.ct_writer import write_series

    vol = (np.arange(12)[:, None, None] * np.ones((1, 8, 8))).astype(np.int16)
    write_series(tmp_path, vol, slice_thickness=2.0, pixel_spacing=0.5, order=[3, 1, 0, 2, 11, 9, 8, 10, 4, 5, 7, 6], slope=1.0,
                 intercept=-1024.0)
    ph = cheese.TomoCheese(str(tmp_path))
    assert ph.num_images == 12 and ph.mm_per_pixel == 0.5
    assert ph.catphan_size == np.pi * 150.0**2 / 0.25
    assert [float(ph.dicom_stack[k].array[0, 0]) for k in range(12)] == [k - 1024.0 for k in range(12)]


def test_unclipped_localization_is_not_implemented():
    if nat.device_count() == 0:
        pytest.skip("the entry point is reached on a device")
    with pytest.raises(NotImplementedError, match="without clipping"):
        nat.ct_localize(nat.Context.default(), np.zeros((1, 8, 8), np.int16), 1.0, 0.0, [0], 10.0, True, clip_in_localization=False)


def test_roll_messages(capsys, monkeypatch):
    """find_phantom_roll's two printed messages, on a profile with no peak and one whose peak is far from every insert"""

    class FakeProfile:
        def __init__(self, values):
            self.values = values

        def find_fwxm_peaks(self, max_number=None):
            return self.peaks, None

    ph = object.__new__(cheese.TomoCheese)
    ph.origin_slice, ph.localization_radius = 0, 110
    monkeypatch.setattr(cheese.TomoCheese, "mm_per_pixel", property(lambda self: 1.0))
    monkeypatch.setattr(cheese, "Slice", lambda *a, **k: type("S", (), {"phan_center": (0, 0), "image": type("I", (), {"array": None})})())
    for peaks, text in (([], "No low-HU regions found"), ([100], "Detected shift of ")):
        prof = FakeProfile(np.zeros(3600))
        prof.peaks = peaks
        monkeypatch.setattr(cheese, "CollapsedCircleProfile", lambda *a, **k: prof)
        assert ph.find_phantom_roll() == 0
        assert text in capsys.readouterr().out


def test_inverted_series_is_not_localized(tmp_path):
    """PixelIntensityRelationshipSign -1 inverts the images after the rescale, which the localization does not; such a series is
    refused before anything reaches the device"""
    from tests.ct_writer import write_series

    write_series(tmp_path, np.zeros((10, 8, 8), np.int16), slice_thickness=1.0, pixel_spacing=1.0, slope=1.0, intercept=-1024.0)
    ph = cheese.TomoCheese(str(tmp_path))
    ph.dicom_stack.metadatas[3]["PixelIntensityRelationshipSign"] = -1
    with pytest.raises(NotImplementedError, match="PixelIntensityRelationshipSign"):
        ph.localization(True)
