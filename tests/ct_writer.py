"""Test helper: write CT slices and series as uncompressed DICOM (what a CT / CBCT console exports, restated from the tags the
reference's DicomImageStack reads: SOP Class UID, SeriesInstanceUID, ImagePositionPatient, SliceThickness, PixelSpacing, the pixel
module and optional rescale tags), without pydicom."""
from __future__ import annotations

import os
import struct

import numpy as np

from tests.dicom_writer import _ds, _elem, _str, _uid

CT_IMAGE_STORAGE = "1.2.840.10008.5.1.4.1.1.2"
RT_STRUCTURE_SET_STORAGE = "1.2.840.10008.5.1.4.1.1.481.3"


def write_ct_slice(path, array: np.ndarray, *, series_uid: str, z: float, slice_thickness: float, pixel_spacing: float,
                   sop_class: str = CT_IMAGE_STORAGE, slope=None, intercept=None, explicit: bool = True):
    """array: 2-D int16 (PixelRepresentation 1) or uint16 (0).  sop_class None: no SOP Class UID element.  Returns the path."""
    a = np.ascontiguousarray(array)
    assert a.ndim == 2 and a.dtype in (np.int16, np.uint16)
    ex = explicit
    body = []
    if sop_class is not None:
        body.append(_elem(0x0008, 0x0016, b"UI", _uid(sop_class), ex))
    body.append(_elem(0x0008, 0x0060, b"CS", _str("CT"), ex))
    body.append(_elem(0x0018, 0x0050, b"DS", _ds(slice_thickness), ex))
    body.append(_elem(0x0020, 0x000E, b"UI", _uid(series_uid), ex))
    body.append(_elem(0x0020, 0x0032, b"DS", _ds([0.0, 0.0, z]), ex))
    body.append(_elem(0x0028, 0x0002, b"US", struct.pack("<H", 1), ex))
    body.append(_elem(0x0028, 0x0010, b"US", struct.pack("<H", a.shape[0]), ex))
    body.append(_elem(0x0028, 0x0011, b"US", struct.pack("<H", a.shape[1]), ex))
    body.append(_elem(0x0028, 0x0030, b"DS", _ds([pixel_spacing, pixel_spacing]), ex))
    body.append(_elem(0x0028, 0x0100, b"US", struct.pack("<H", 16), ex))
    body.append(_elem(0x0028, 0x0101, b"US", struct.pack("<H", 16), ex))
    body.append(_elem(0x0028, 0x0103, b"US", struct.pack("<H", 1 if a.dtype == np.int16 else 0), ex))
    if intercept is not None:
        body.append(_elem(0x0028, 0x1052, b"DS", _ds(intercept), ex))
    if slope is not None:
        body.append(_elem(0x0028, 0x1053, b"DS", _ds(slope), ex))
    body.append(_elem(0x7FE0, 0x0010, b"OW", a.astype(a.dtype.newbyteorder("<")).tobytes(), ex))
    ts = "1.2.840.10008.1.2.1" if explicit else "1.2.840.10008.1.2"
    meta = _elem(0x0002, 0x0002, b"UI", _uid(sop_class or CT_IMAGE_STORAGE), True) + _elem(0x0002, 0x0010, b"UI", _uid(ts), True)
    meta = _elem(0x0002, 0x0000, b"UL", struct.pack("<I", len(meta)), True) + meta
    with open(path, "wb") as f:
        f.write(b"\x00" * 128 + b"DICM" + meta + b"".join(body))
    return str(path)


def write_series(directory, volume: np.ndarray, *, slice_thickness: float, pixel_spacing: float, series_uid: str = "1.2.826.0.1.3680043.2.1",
                 order=None, z0: float = 0.0, **kwargs) -> list[str]:
    """volume [N, H, W]: slice n at z = z0 + n * slice_thickness, written as ``CT<k>.dcm`` in the order `order` (a permutation of
    range(N); default: the slices' own order), so that the file names say nothing about the slice position."""
    os.makedirs(directory, exist_ok=True)
    order = range(len(volume)) if order is None else order
    paths = []
    for k, n in enumerate(order):
        paths.append(write_ct_slice(os.path.join(directory, f"CT{k:04d}.dcm"), volume[n], series_uid=series_uid,
                                    z=z0 + n * slice_thickness, slice_thickness=slice_thickness, pixel_spacing=pixel_spacing, **kwargs))
    return paths
