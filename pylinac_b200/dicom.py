"""Minimal DICOM Part-10 reader for uncompressed EPID RT-Images (host-side ingest).

The reference reads files with ``pydicom.dcmread`` (core/io.py:73-84) and then only touches a handful of tags
(core/image.py:363-389, 1431-1444, 1509-1580, 1612-1730).  pydicom is not a dependency here; this parser handles
what linac EPIDs write: explicit- or implicit-VR little endian, native (uncompressed) PixelData.

Only the tags the hot path consumes are decoded into Python values; everything else is skipped.
"""
from __future__ import annotations

import io
import struct

import numpy as np

_EXPLICIT_LONG_VR = {b"OB", b"OW", b"OF", b"OD", b"OL", b"OV", b"SQ", b"UC", b"UN", b"UR", b"UT"}

# (group, element) -> (keyword, kind)
_TAGS = {
    (0x0002, 0x0010): ("TransferSyntaxUID", "str"),
    (0x0008, 0x0016): ("SOPClassUID", "str"),
    (0x0008, 0x0060): ("Modality", "str"),
    (0x0008, 0x0070): ("Manufacturer", "str"),
    (0x0008, 0x0012): ("InstanceCreationDate", "str"),
    (0x0008, 0x0013): ("InstanceCreationTime", "str"),
    (0x0008, 0x0023): ("ContentDate", "str"),
    (0x0008, 0x0033): ("ContentTime", "str"),
    (0x0018, 0x0050): ("SliceThickness", "ds"),
    (0x0018, 0x1110): ("DistanceSourceToDetector", "ds"),
    (0x0018, 0x1164): ("ImagerPixelSpacing", "ds"),
    (0x0020, 0x000E): ("SeriesInstanceUID", "str"),
    (0x0020, 0x0032): ("ImagePositionPatient", "ds"),
    (0x0028, 0x0002): ("SamplesPerPixel", "us"),
    (0x0028, 0x0008): ("NumberOfFrames", "is"),
    (0x0028, 0x0010): ("Rows", "us"),
    (0x0028, 0x0011): ("Columns", "us"),
    (0x0028, 0x0030): ("PixelSpacing", "ds"),
    (0x0028, 0x0100): ("BitsAllocated", "us"),
    (0x0028, 0x0101): ("BitsStored", "us"),
    (0x0028, 0x0103): ("PixelRepresentation", "us"),
    (0x0028, 0x1040): ("PixelIntensityRelationship", "str"),
    (0x0028, 0x1041): ("PixelIntensityRelationshipSign", "ss"),
    (0x0028, 0x1052): ("RescaleIntercept", "ds"),
    (0x0028, 0x1053): ("RescaleSlope", "ds"),
    (0x3002, 0x0011): ("ImagePlanePixelSpacing", "ds"),
    (0x3002, 0x000D): ("XRayImageReceptorTranslation", "ds"),
    (0x3002, 0x0022): ("RadiationMachineSAD", "ds"),
    (0x3002, 0x0026): ("RTImageSID", "ds"),
    (0x300A, 0x011E): ("GantryAngle", "ds"),
    (0x300A, 0x0120): ("BeamLimitingDeviceAngle", "ds"),
    (0x300A, 0x0122): ("PatientSupportAngle", "ds"),
}
_PIXEL_DATA = (0x7FE0, 0x0010)

# The standard storage SOP classes (DICOM PS3.6 annex A) whose names contain "Image Storage": LazyDicomImageStack keeps a file when
# ``"Image Storage" in ds.SOPClassUID.name`` (core/image.py:1961); pydicom's UID names are restated here as a table.
IMAGE_STORAGE_UIDS = {
    "1.2.840.10008.5.1.4.1.1.1": "Computed Radiography Image Storage",
    "1.2.840.10008.5.1.4.1.1.1.1": "Digital X-Ray Image Storage - For Presentation",
    "1.2.840.10008.5.1.4.1.1.1.1.1": "Digital X-Ray Image Storage - For Processing",
    "1.2.840.10008.5.1.4.1.1.1.2": "Digital Mammography X-Ray Image Storage - For Presentation",
    "1.2.840.10008.5.1.4.1.1.1.2.1": "Digital Mammography X-Ray Image Storage - For Processing",
    "1.2.840.10008.5.1.4.1.1.1.3": "Digital Intra-Oral X-Ray Image Storage - For Presentation",
    "1.2.840.10008.5.1.4.1.1.1.3.1": "Digital Intra-Oral X-Ray Image Storage - For Processing",
    "1.2.840.10008.5.1.4.1.1.2": "CT Image Storage",
    "1.2.840.10008.5.1.4.1.1.2.1": "Enhanced CT Image Storage",
    "1.2.840.10008.5.1.4.1.1.2.2": "Legacy Converted Enhanced CT Image Storage",
    "1.2.840.10008.5.1.4.1.1.3.1": "Ultrasound Multi-frame Image Storage",
    "1.2.840.10008.5.1.4.1.1.4": "MR Image Storage",
    "1.2.840.10008.5.1.4.1.1.4.1": "Enhanced MR Image Storage",
    "1.2.840.10008.5.1.4.1.1.4.3": "Enhanced MR Color Image Storage",
    "1.2.840.10008.5.1.4.1.1.4.4": "Legacy Converted Enhanced MR Image Storage",
    "1.2.840.10008.5.1.4.1.1.6.1": "Ultrasound Image Storage",
    "1.2.840.10008.5.1.4.1.1.7": "Secondary Capture Image Storage",
    "1.2.840.10008.5.1.4.1.1.7.1": "Multi-frame Single Bit Secondary Capture Image Storage",
    "1.2.840.10008.5.1.4.1.1.7.2": "Multi-frame Grayscale Byte Secondary Capture Image Storage",
    "1.2.840.10008.5.1.4.1.1.7.3": "Multi-frame Grayscale Word Secondary Capture Image Storage",
    "1.2.840.10008.5.1.4.1.1.7.4": "Multi-frame True Color Secondary Capture Image Storage",
    "1.2.840.10008.5.1.4.1.1.12.1": "X-Ray Angiographic Image Storage",
    "1.2.840.10008.5.1.4.1.1.12.1.1": "Enhanced XA Image Storage",
    "1.2.840.10008.5.1.4.1.1.12.2": "X-Ray Radiofluoroscopic Image Storage",
    "1.2.840.10008.5.1.4.1.1.12.2.1": "Enhanced XRF Image Storage",
    "1.2.840.10008.5.1.4.1.1.13.1.1": "X-Ray 3D Angiographic Image Storage",
    "1.2.840.10008.5.1.4.1.1.13.1.2": "X-Ray 3D Craniofacial Image Storage",
    "1.2.840.10008.5.1.4.1.1.13.1.3": "Breast Tomosynthesis Image Storage",
    "1.2.840.10008.5.1.4.1.1.20": "Nuclear Medicine Image Storage",
    "1.2.840.10008.5.1.4.1.1.77.1.1": "VL Endoscopic Image Storage",
    "1.2.840.10008.5.1.4.1.1.77.1.2": "VL Microscopic Image Storage",
    "1.2.840.10008.5.1.4.1.1.77.1.3": "VL Slide-Coordinates Microscopic Image Storage",
    "1.2.840.10008.5.1.4.1.1.77.1.4": "VL Photographic Image Storage",
    "1.2.840.10008.5.1.4.1.1.128": "Positron Emission Tomography Image Storage",
    "1.2.840.10008.5.1.4.1.1.128.1": "Legacy Converted Enhanced PET Image Storage",
    "1.2.840.10008.5.1.4.1.1.130": "Enhanced PET Image Storage",
    "1.2.840.10008.5.1.4.1.1.481.1": "RT Image Storage",
}


class InvalidDicomError(Exception):
    pass


class Dataset(dict):
    """Decoded tags by keyword, plus ``pixel_array``."""

    pixel_array: np.ndarray

    def __getattr__(self, item):
        try:
            return self[item]
        except KeyError:
            raise AttributeError(item)


def _decode(kind, raw: bytes):
    if kind == "us":
        vals = struct.unpack("<%dH" % (len(raw) // 2), raw)
    elif kind == "ss":
        vals = struct.unpack("<%dh" % (len(raw) // 2), raw)
    elif kind in ("ds", "is"):
        txt = raw.decode("ascii", "ignore").strip(" \x00")
        if not txt:
            return None
        parts = txt.split("\\")
        vals = [float(p) if kind == "ds" else int(float(p)) for p in parts if p.strip()]
    else:
        return raw.decode("ascii", "ignore").strip(" \x00")
    if len(vals) == 1:
        return vals[0]
    return list(vals)


def _read_elements(buf: memoryview, pos: int, end: int, explicit: bool, ds: Dataset, depth=0):
    n = len(buf)
    while pos + 8 <= min(end, n):
        group, elem = struct.unpack_from("<HH", buf, pos)
        if (group, elem) == (0xFFFE, 0xE00D) or (group, elem) == (0xFFFE, 0xE0DD):  # item / sequence delimiters
            return pos + 8
        is_explicit = explicit or group == 0x0002
        if group == 0xFFFE:  # item start
            length = struct.unpack_from("<I", buf, pos + 4)[0]
            pos += 8
            if length == 0xFFFFFFFF:
                pos = _read_elements(buf, pos, n, explicit, Dataset(), depth + 1)
            else:
                pos += length
            continue
        if is_explicit:
            vr = bytes(buf[pos + 4 : pos + 6])
            if vr in _EXPLICIT_LONG_VR:
                length = struct.unpack_from("<I", buf, pos + 8)[0]
                hdr = 12
            else:
                length = struct.unpack_from("<H", buf, pos + 6)[0]
                hdr = 8
        else:
            vr = b""
            length = struct.unpack_from("<I", buf, pos + 4)[0]
            hdr = 8
        pos += hdr
        if length == 0xFFFFFFFF:  # undefined length: sequence (or encapsulated pixel data)
            if (group, elem) == _PIXEL_DATA:
                raise InvalidDicomError("compressed (encapsulated) pixel data is not supported")
            pos = _read_sequence(buf, pos, explicit, depth)
            continue
        if depth == 0:
            if (group, elem) == _PIXEL_DATA:
                ds["_pixel_offset"] = pos
                ds["_pixel_length"] = length
            elif (group, elem) in _TAGS:
                key, kind = _TAGS[(group, elem)]
                ds[key] = _decode(kind, bytes(buf[pos : pos + length]))
        pos += length
    return pos


def _read_sequence(buf, pos, explicit, depth):
    n = len(buf)
    while pos + 8 <= n:
        group, elem, length = struct.unpack_from("<HHI", buf, pos)
        pos += 8
        if (group, elem) == (0xFFFE, 0xE0DD):
            return pos
        if (group, elem) == (0xFFFE, 0xE000):
            if length == 0xFFFFFFFF:
                pos = _read_elements(buf, pos, n, explicit, Dataset(), depth + 1)
            else:
                pos += length
        else:
            raise InvalidDicomError("malformed sequence")
    return pos


def dcmread(source, pixels: bool = True) -> Dataset:
    """Parse a DICOM file (path, bytes or binary stream).  pixels=False: header only -- `source` may be the leading part of a file;
    the dataset then carries PixelOffset / PixelLength / PixelDtype (file position, byte count and dtype of the pixel data) instead of
    ``pixel_array``."""
    if isinstance(source, (bytes, bytearray)):
        data = bytes(source)
    elif hasattr(source, "read"):
        source.seek(0)
        data = source.read()
    else:
        with open(source, "rb") as f:
            data = f.read()
    buf = memoryview(data)
    ds = Dataset()
    pos = 0
    explicit = False
    if len(data) >= 132 and data[128:132] == b"DICM":
        pos = 132
        # file meta group 0002 is always explicit VR LE
        meta = Dataset()
        p = pos
        while p + 8 <= len(buf):
            group = struct.unpack_from("<H", buf, p)[0]
            if group != 0x0002:
                break
            elem = struct.unpack_from("<H", buf, p + 2)[0]
            vr = bytes(buf[p + 4 : p + 6])
            if vr in _EXPLICIT_LONG_VR:
                length = struct.unpack_from("<I", buf, p + 8)[0]
                hdr = 12
            else:
                length = struct.unpack_from("<H", buf, p + 6)[0]
                hdr = 8
            if (group, elem) in _TAGS:
                key, kind = _TAGS[(group, elem)]
                meta[key] = _decode(kind, bytes(buf[p + hdr : p + hdr + length]))
            p += hdr + length
        pos = p
        ts = meta.get("TransferSyntaxUID", "1.2.840.10008.1.2")
        ds["TransferSyntaxUID"] = ts
        if ts == "1.2.840.10008.1.2":
            explicit = False
        elif ts in ("1.2.840.10008.1.2.1",):
            explicit = True
        elif ts == "1.2.840.10008.1.2.2":
            raise InvalidDicomError("big-endian transfer syntax is not supported")
        else:
            raise InvalidDicomError(f"compressed transfer syntax {ts} is not supported")
    else:
        # no preamble: assume implicit VR little endian (the reference forces this too, core/io.py:81-83),
        # unless the first element carries a plausible explicit VR
        if len(data) < 8:
            raise InvalidDicomError("not a DICOM file")
        vr = data[4:6]
        explicit = vr.isalpha() and vr.isupper()
    _read_elements(buf, pos, len(buf), explicit, ds)
    if "_pixel_offset" not in ds or "Rows" not in ds or "Columns" not in ds:
        raise InvalidDicomError("no pixel data found")
    rows, cols = int(ds["Rows"]), int(ds["Columns"])
    bits = int(ds.get("BitsAllocated", 16))
    signed = int(ds.get("PixelRepresentation", 0)) == 1
    if bits == 8:
        dt = np.int8 if signed else np.uint8
    elif bits == 16:
        dt = np.dtype("<i2") if signed else np.dtype("<u2")
    elif bits == 32:
        dt = np.dtype("<i4") if signed else np.dtype("<u4")
    else:
        raise InvalidDicomError(f"BitsAllocated={bits} is not supported")
    frames = int(ds.get("NumberOfFrames", 1) or 1)
    count = rows * cols * frames
    off = ds.pop("_pixel_offset")
    plen = ds.pop("_pixel_length")
    if not pixels:
        ds["PixelOffset"], ds["PixelLength"], ds["PixelDtype"], ds["PixelCount"] = off, plen, np.dtype(dt), count
        return ds
    arr = np.frombuffer(data, dtype=dt, count=count, offset=off)
    ds.pixel_array = arr.reshape((frames, rows, cols) if frames > 1 else (rows, cols))
    return ds


def is_dicom(source) -> bool:
    try:
        dcmread(source)
        return True
    except Exception:
        return False


# ------------------------------------------------------------------------------------------------ batched ingest
def read_header(path, head_bytes: int = 1 << 18) -> Dataset:
    """Header of one file without touching its pixel data: the first `head_bytes` are parsed (EPID headers are a few KB); a file
    whose pixel element starts later is parsed again in full."""
    import os

    size = os.path.getsize(path)
    with open(path, "rb") as f:
        head = f.read(min(size, head_bytes))
        try:
            ds = dcmread(head, pixels=False)
        except InvalidDicomError:
            if size <= head_bytes:
                raise
            ds = dcmread(head + f.read(), pixels=False)
    if ds["PixelOffset"] + ds["PixelCount"] * ds["PixelDtype"].itemsize > size:
        raise InvalidDicomError(f"{path}: pixel data is truncated")
    return ds


def read_frames(paths, out=None, threads: int = 8, headers=None):
    """Batched ingest (the reference reads one file at a time: core/io.py:73-84 + core/image.py:1431-1444): parse the headers, then
    read every file's pixel bytes with ``readinto`` STRAIGHT into its slot of one [n, rows, cols] array -- pass a page-locked array
    (``_native.pinned_empty``) as `out` and the bytes go page cache -> pinned memory -> HBM with no intermediate copy.  All files
    must share rows / columns / stored dtype.  `headers`: the files' ``read_header`` datasets when the caller already has them.
    Returns (frames, headers)."""
    from concurrent.futures import ThreadPoolExecutor

    paths = [str(p) for p in paths]
    if not paths:
        raise ValueError("no files")
    with ThreadPoolExecutor(max(1, min(threads, len(paths)))) as pool:
        headers = list(pool.map(read_header, paths)) if headers is None else list(headers)
        h0 = headers[0]
        shape = (int(h0["Rows"]), int(h0["Columns"]))
        dt = h0["PixelDtype"]
        for pth, h in zip(paths, headers):
            if (int(h["Rows"]), int(h["Columns"])) != shape or h["PixelDtype"] != dt or int(h.get("NumberOfFrames", 1) or 1) != 1:
                raise ValueError(f"{pth}: {h['Rows']} x {h['Columns']} {h['PixelDtype']} differs from the first file's {shape} {dt}")
        if out is None:
            out = np.empty((len(paths),) + shape, dt)
        if out.shape != (len(paths),) + shape or out.dtype != dt or not out.flags.c_contiguous:
            raise ValueError(f"out must be a C-contiguous {(len(paths),) + shape} array of {dt}")

        list(pool.map(lambda i: _read_pixels(paths[i], headers[i], out[i]), range(len(paths))))
    return out, headers


def _read_pixels(path, header, dst: np.ndarray) -> None:
    """``readinto`` the pixel bytes of `path` (located by its `header`) straight into the C-contiguous `dst`"""
    with open(path, "rb", buffering=0) as f:
        f.seek(header["PixelOffset"])
        mv = memoryview(dst).cast("B")
        got = 0
        while got < len(mv):
            k = f.readinto(mv[got:])
            if not k:
                raise InvalidDicomError(f"{path}: pixel data is truncated")
            got += k


def read_nm_frames(paths, out=None, threads: int = 8):
    """Batched ingest of multi-frame files (nuclear medicine stacks): every frame of every file, in file then frame order, read with
    ``readinto`` straight into one [n, rows, cols] array, where n is the files' total NumberOfFrames.  Pass a page-locked array
    (``_native.pinned_empty``) as `out` for a direct H2D copy.  All files must share rows / columns / stored dtype.  Returns
    (frames, headers)."""
    from concurrent.futures import ThreadPoolExecutor

    paths = [str(p) for p in paths]
    if not paths:
        raise ValueError("no files")
    with ThreadPoolExecutor(max(1, min(threads, len(paths)))) as pool:
        headers = list(pool.map(read_header, paths))
        h0 = headers[0]
        shape = (int(h0["Rows"]), int(h0["Columns"]))
        dt = h0["PixelDtype"]
        for pth, h in zip(paths, headers):
            if (int(h["Rows"]), int(h["Columns"])) != shape or h["PixelDtype"] != dt:
                raise ValueError(f"{pth}: {h['Rows']} x {h['Columns']} {h['PixelDtype']} differs from the first file's {shape} {dt}")
        counts = [int(h.get("NumberOfFrames", 1) or 1) for h in headers]
        starts = np.concatenate([[0], np.cumsum(counts)])
        if out is None:
            out = np.empty((int(starts[-1]),) + shape, dt)
        if out.shape != (int(starts[-1]),) + shape or out.dtype != dt or not out.flags.c_contiguous:
            raise ValueError(f"out must be a C-contiguous {(int(starts[-1]),) + shape} array of {dt}")
        list(pool.map(lambda i: _read_pixels(paths[i], headers[i], out[starts[i]:starts[i + 1]]), range(len(paths))))
    return out, headers
