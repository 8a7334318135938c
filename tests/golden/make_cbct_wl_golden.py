"""Generate tests/golden/cbct_wl_golden.npz: the UNMODIFIED reference ``WinstonLutz.from_cbct`` (winston_lutz.py:1444-1509,
stub-imported; skimage served by oracle/skimage_shim.py) on the seeded volumes of cbct_wl_cases.py.

pydicom is not installed here, so the two file boundaries of from_cbct are served in memory:
* ``DicomImageStack`` is a fake holding the slices and the SliceThickness / PixelSpacing tags;
* ``array_to_dicom`` is intercepted: each frame, its gantry and its dpi are captured (``save_as`` writes nothing), and the
  ``cls(dicom_dir)`` that would read the files back builds its images from the captured frames, read back as the uint16 bits
  array_to_dicom writes (PixelRepresentation 0), with ImagePlanePixelSpacing 25.4 / dpi, SID 1000 and SAD 1000.
The set is then analysed by the reference (``analyze(bb_size_mm=5)``; is_from_cbct forces low_density_bb / open_field).

Run here (the container that has /root/reference):  python -m tests.golden.make_cbct_wl_golden
"""
from __future__ import annotations

import hashlib
import shutil
import tempfile
import threading
import types
import warnings

import numpy as np

from tests.golden.cbct_wl_cases import CASES, case_volume
from tests.golden.make_wlset_golden import SCALARS


def _sha(a):
    return np.frombuffer(hashlib.sha1(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def reference_from_cbct(volume, slice_thickness, pixel_spacing):
    from oracle import skimage_shim
    from oracle.refstub import reference_image_from_array

    skimage_shim.install()
    from pylinac import winston_lutz as wl

    captured = []

    class FakeStack:
        def __init__(self, folder, min_number=39, raw_pixels=False, **kwargs):
            self.images = [np.array(s) for s in volume]
            self.metadata = types.SimpleNamespace(SliceThickness=slice_thickness, PixelSpacing=[pixel_spacing, pixel_spacing])

    def fake_array_to_dicom(array, sid, gantry, coll, couch, dpi, extra_tags=None):
        captured.append((np.array(array), gantry, dpi, sid))
        return types.SimpleNamespace(save_as=lambda *a, **k: None)

    class CapturedWL(wl.WinstonLutz):
        def __init__(self, directory, **kwargs):
            self._captured_warnings, self._warnings_lock = [], threading.Lock()
            self.images = [reference_image_from_array(wl.WinstonLutz2D, a.view(np.uint16) if a.dtype == np.int16 else a, 25.4 / dpi,
                                                      sid=sid, gantry=float(f"{g:.2f}"), coll=0.0, couch=0.0)
                           for a, g, dpi, sid in captured]
            self.images.sort(key=lambda i: (i.gantry_angle, i.collimator_angle, i.couch_angle))
            self._is_analyzed = False

    old = wl.DicomImageStack, wl.array_to_dicom, wl.tempfile
    tmp = tempfile.mkdtemp()
    wl.DicomImageStack, wl.array_to_dicom = FakeStack, fake_array_to_dicom
    wl.tempfile = types.SimpleNamespace(mkdtemp=lambda: tmp)
    try:
        st = CapturedWL.from_cbct("unused", raw_pixels=True)
    finally:
        wl.DicomImageStack, wl.array_to_dicom, wl.tempfile = old
        shutil.rmtree(tmp, ignore_errors=True)
    assert st.is_from_cbct
    st.analyze(bb_size_mm=5)
    out = {}
    for a, g, dpi, _ in captured:
        out[f"frame_{g}_sha1"] = _sha(a.view(np.uint16) if a.dtype == np.int16 else a)
        out[f"frame_{g}_shape"] = np.array(a.shape)
        out[f"frame_{g}_dtype"] = np.array(str(a.dtype))
        out["dpi"] = np.array(dpi)
    rd = st.results_data()
    for k in SCALARS:
        out[k] = np.asarray(getattr(rd, k))
    sv = st.bb_shift_vector
    out["bb_shift_vector"] = np.array([sv.x, sv.y, sv.z], dtype=float)
    for im in st.images:
        g = int(round(im.gantry_angle))
        out[f"bb_{g}"] = np.array([im.bb.x, im.bb.y])
        out[f"field_{g}"] = np.array([im.field_cax.x, im.field_cax.y])
        out[f"epid_{g}"] = np.array([im.epid.x, im.epid.y])
        out[f"cax2bb_distance_{g}"] = np.array(im.cax2bb_distance)
    out["dpmm"] = np.array(st.images[0].dpmm)
    out["cax2epid_max"] = np.array(st.cax2epid_distance("max"))
    return out, captured


def main():
    from oracle import cbct_oracle
    from oracle.refstub import import_reference

    import_reference()
    warnings.simplefilter("ignore")
    store = {}
    for name in CASES:
        vol, st_mm, ps = case_volume(name)
        store[f"{name}/volume_sha1"] = _sha(vol)
        colmax, rowmax = cbct_oracle.projections(vol)
        store[f"{name}/colmax"], store[f"{name}/rowmax"] = colmax, rowmax
        ref, captured = reference_from_cbct(vol, st_mm, ps)
        oracle_frames = cbct_oracle.cbct_frames(vol, st_mm, ps)
        for a, g, _, _ in captured:
            assert np.array_equal(oracle_frames[g], a.view(np.uint16) if a.dtype == np.int16 else a), (name, g)
        for k, v in ref.items():
            store[f"{name}/{k}"] = v
        print(name, vol.dtype, vol.shape, ref["frame_0_shape"].tolist(), ref["frame_270_shape"].tolist(), "shift",
              np.round(ref["bb_shift_vector"], 3).tolist(), "cax2bb max", float(ref["max_2d_cax_to_bb_mm"]))
    np.savez_compressed("tests/golden/cbct_wl_golden.npz", **store)


if __name__ == "__main__":
    main()
