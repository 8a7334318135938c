"""Test helper: write uncompressed multi-frame nuclear medicine (NM) DICOM files without pydicom, so the NM ingest
(dicom.read_nm_frames, core.image.NMImageStack) and the nuclear classes can be tested from files: implicit or explicit VR, 1 or N
frames, uint8 or uint16 pixels."""
from __future__ import annotations

import struct

import numpy as np

from tests.dicom_writer import _ds, _elem, _str, _uid

NM_SOP_CLASS = "1.2.840.10008.5.1.4.1.1.20"


def write_nm(path, frames: np.ndarray, *, pixel_spacing_mm=4.8, modality="NM", explicit=True, preamble=True):
    """frames: [n, h, w] or [h, w] uint8 / uint16.  Returns the path."""
    a = np.ascontiguousarray(frames)
    if a.ndim == 2:
        a = a[None]
    assert a.ndim == 3 and a.dtype in (np.uint16, np.uint8)
    bits = 8 * a.dtype.itemsize
    ex = explicit
    body = [
        _elem(0x0008, 0x0016, b"UI", _uid(NM_SOP_CLASS), ex),
        _elem(0x0008, 0x0060, b"CS", _str(modality), ex),
        _elem(0x0028, 0x0002, b"US", struct.pack("<H", 1), ex),
        _elem(0x0028, 0x0008, b"IS", _str(str(a.shape[0])), ex),
        _elem(0x0028, 0x0010, b"US", struct.pack("<H", a.shape[1]), ex),
        _elem(0x0028, 0x0011, b"US", struct.pack("<H", a.shape[2]), ex),
        _elem(0x0028, 0x0030, b"DS", _ds([pixel_spacing_mm, pixel_spacing_mm]), ex),
        _elem(0x0028, 0x0100, b"US", struct.pack("<H", bits), ex),
        _elem(0x0028, 0x0101, b"US", struct.pack("<H", bits), ex),
        _elem(0x0028, 0x0103, b"US", struct.pack("<H", 0), ex),
    ]
    pixels = a.astype(a.dtype.newbyteorder("<")).tobytes()
    pixels += b"\x00" * (len(pixels) & 1)
    body.append(_elem(0x7FE0, 0x0010, b"OB" if bits == 8 else b"OW", pixels, ex))
    out = b""
    if preamble:
        ts = "1.2.840.10008.1.2.1" if explicit else "1.2.840.10008.1.2"
        meta = _elem(0x0002, 0x0002, b"UI", _uid(NM_SOP_CLASS), True) + _elem(0x0002, 0x0010, b"UI", _uid(ts), True)
        meta = _elem(0x0002, 0x0000, b"UL", struct.pack("<I", len(meta)), True) + meta
        out = b"\x00" * 128 + b"DICM" + meta
    out += b"".join(body)
    with open(path, "wb") as f:
        f.write(out)
    return str(path)
