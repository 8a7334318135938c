"""Varian XIM reader (host side): the header / property walk of ``pylinac.core.image.XIM`` (core/image.py:1119-1183, with
``decode_binary``, core/utilities.py:232-285), and batched ingest whose pixel decode runs on the GPU (``epid_xim_decode``,
csrc/xim.cu).  Nothing here touches pixel values: the compressed bytes go to the device as they are in the file.

An XIM file is "VMS.XI" padded to 8 bytes, six int32 (format_version, width, height, bits_per_pixel, bytes_per_pixel,
compression), then for compressed files the 2-bit lookup table and the compressed pixel buffer (each preceded by its int32 size)
and an int32, then the histogram and the typed property list.
"""
from __future__ import annotations

import os
import struct

import numpy as np

from . import _native as nat

PROP_INT, PROP_DOUBLE, PROP_STRING, PROP_DOUBLE_ARRAY, PROP_INT_ARRAY = 0, 1, 2, 4, 5   # core/image.py:71-75
_NATURAL = {1: np.int16, 2: np.int16, 4: np.int32, 8: np.int64}   # device dtype per bytes_per_pixel (bpp 1: int8 values in int16)
_REF_DTYPES = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}
_BPP_ERROR = "The XIM image has an unsupported bytes per pixel value. Raise a ticket on the pylinac Github with this file."


class XimHeader:
    """Everything XIM reads from a file except the pixels, plus where the compressed pixels are:
    ``lut_offset`` / ``lookup_table`` (the table as read), ``pix_offset`` / ``pix_bytes`` (the pixel bytes present in the file, at
    most the declared size).  ``trailer_error`` is the exception the walk met after the pixel buffer; the reference raises it only
    after a successful decode, so it is kept until then."""

    path: str
    lookup_table: np.ndarray
    trailer_error: Exception | None = None

    @property
    def shape(self) -> tuple[int, int]:
        return self.img_height_px, self.img_width_px


# ------------------------------------------------------------------------------------------------ decode_binary
def _read(f, n: int) -> bytes:
    b = f.read(max(n, 0)) if n >= 0 else f.read()
    if len(b) != max(n, 0):
        raise struct.error(f"unpack requires a buffer of {max(n, 0)} bytes")
    return b


def _int(f, count: int = 1):
    """decode_binary(f, int, count): a Python int for one value, else np.asarray of the values (float64 when empty)"""
    vals = np.asarray(struct.unpack("<%di" % max(count, 0), _read(f, 4 * count)))
    return int(np.squeeze(vals)) if len(vals) == 1 else vals


def _double(f, count: int = 1):
    """decode_binary(f, "d", count): a float for one value, else a tuple"""
    vals = struct.unpack("<%dd" % max(count, 0), _read(f, 8 * count))
    return vals[0] if len(vals) == 1 else vals


def _str(f, count: int) -> str:
    """decode_binary(f, str, count): the bytes without NULs, each decoded on its own (non-ASCII raises UnicodeDecodeError)"""
    return _read(f, count).replace(b"\x00", b"").decode("ascii")


def _properties(f, hd: XimHeader) -> None:
    hd.num_hist_bins = _int(f)
    hd.histogram = _int(f, hd.num_hist_bins)
    hd.num_properties = _int(f)
    hd.properties = {}
    for _ in range(hd.num_properties):
        name = _str(f, _int(f))
        tipe = _int(f)
        if tipe == PROP_INT:
            value = _int(f)
        elif tipe == PROP_DOUBLE:
            value = _double(f)
        elif tipe == PROP_STRING:
            value = _str(f, _int(f))
        elif tipe == PROP_DOUBLE_ARRAY:
            value = _double(f, int(_int(f) // 8))
        elif tipe == PROP_INT_ARRAY:
            value = _int(f, int(_int(f) // 4))
        # an unknown type reads no value: the reference stores the previous property's value again (UnboundLocalError if none)
        hd.properties[name] = value  # noqa: F821


def walk(path, read_pixels: bool = True) -> XimHeader:
    """The reference constructor's walk of the file (core/image.py:1131-1183) without decoding pixels.

    read_pixels=True: bytes_per_pixel is checked and the pixel buffer located as ``_parse_compressed_bytes`` would read it; an
    error after it is kept in ``trailer_error``.  read_pixels=False: the pixel buffer is skipped like the reference skips it."""
    hd = XimHeader()
    hd.path = str(path)
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        hd.format_id = _str(f, 8)
        hd.format_version = _int(f)
        hd.img_width_px = _int(f)
        hd.img_height_px = _int(f)
        hd.bits_per_pixel = _int(f)
        hd.bytes_per_pixel = _int(f)
        hd.compression = _int(f)
        if not hd.compression:
            hd.pixel_buffer = _str(f, _int(f))
            _properties(f, hd)
            return hd
        lut_size = _int(f)
        hd.lut_offset = f.tell()
        hd.lookup_table = np.frombuffer(f.read(max(lut_size, 0)) if lut_size >= 0 else f.read(), np.uint8).copy()
        if not read_pixels:
            _read(f, _int(f))
            _int(f)
            _properties(f, hd)
            return hd
        if hd.bytes_per_pixel not in _REF_DTYPES:
            raise ValueError(_BPP_ERROR)
        comp = _int(f)
        hd.pix_offset = f.tell()
        rest = size - hd.pix_offset
        hd.pix_bytes = rest if comp < 0 else min(comp, rest)
        f.seek(hd.pix_offset + hd.pix_bytes)
        try:
            _int(f)
            _properties(f, hd)
        except Exception as e:  # raised by the reference after the decode
            hd.trailer_error = e
    return hd


def read_header(path) -> XimHeader:
    """Header, histogram and properties of a compressed XIM file, and where its lookup table and pixel buffer are.  Raises what
    the reference's constructor raises for the parts it reads (bad bytes_per_pixel, truncation)."""
    hd = walk(path, read_pixels=True)
    if not hd.compression:
        raise ValueError(f"{path}: uncompressed XIM files carry no pixel array")
    if hd.trailer_error is not None:
        raise hd.trailer_error
    return hd


# ------------------------------------------------------------------------------------------------ device decode
def _slot(n: int) -> int:
    return (n + 15) & ~15


def raise_status(status: int, what: str) -> None:
    """the reference's exception for a per-frame status of epid_xim_decode"""
    if status == nat.XIM_LOOKUP_CODE3:
        raise KeyError(3)          # LOOKUP_CONVERSION[3] (core/image.py:1297-1300)
    if status == nat.XIM_SHORT_BUFFER:
        raise ValueError(f"{what}: the compressed pixel buffer is shorter than its lookup table requires")
    if status == nat.XIM_U16_RANGE:
        raise ValueError(f"{what}: pixel values outside [0, 65535] do not fit a uint16 frame")
    if status != nat.XIM_OK:
        raise RuntimeError(f"{what}: unknown XIM decode status {status}")


def check_header(hd: XimHeader) -> None:
    """the reference's failures that need no pixel decode, raised as it raises them (core/image.py:1286-1294 and the row loop's
    sliding window): one row, a pixel buffer shorter than the raw int32 head, an empty lookup table"""
    h, w = hd.img_height_px, hd.img_width_px
    if h < 2:   # the head fills a one-row array only when exactly W values are present; then the (empty) table is indexed
        if len(hd.lookup_table) == 0 and min(hd.pix_bytes, 4 * (w + 1)) == 4 * w:
            raise IndexError("index 0 is out of bounds for axis 0 with size 0")
        raise ValueError(f"{hd.path}: an XIM image needs at least two rows")
    if hd.pix_bytes < 4 * (w + 1):
        raise ValueError(f"{hd.path}: the pixel buffer is shorter than the raw head of {w + 1} int32 values")
    if len(hd.lookup_table) == 0:
        raise IndexError("index 0 is out of bounds for axis 0 with size 0")


def arena_layout(headers):
    """-> (arena bytes, desc int64 [n, 4]): every file's lookup table and pixel buffer in 16-byte-aligned slots"""
    desc = np.zeros((len(headers), 4), np.int64)
    pos = 0
    for i, hd in enumerate(headers):
        desc[i, 0], desc[i, 1] = pos, len(hd.lookup_table)
        pos += _slot(len(hd.lookup_table))
        desc[i, 2], desc[i, 3] = pos, hd.pix_bytes
        pos += _slot(hd.pix_bytes)
    return max(pos, 16), desc


def decode_arena(arena: np.ndarray, desc: np.ndarray, h: int, w: int, bpp: int, dtype=None, device: int | None = None):
    """One device decode of every frame in `arena` (uint8, 16-byte aligned; page-locked for a DMA copy) -> (Batch, status [n])."""
    if bpp not in _REF_DTYPES:
        raise ValueError(_BPP_ERROR)
    ctx = nat.Context.default(device)
    dt = np.dtype(_NATURAL[bpp] if dtype is None else dtype)
    return nat.xim_decode(ctx, arena, desc, h, w, bpp, dt)


def _fill(arena: np.ndarray, hd: XimHeader, lut_off: int, pix_off: int) -> None:
    k = len(hd.lookup_table)
    arena[lut_off : lut_off + k] = hd.lookup_table
    with open(hd.path, "rb", buffering=0) as f:
        f.seek(hd.pix_offset)
        mv = memoryview(arena[pix_off : pix_off + hd.pix_bytes])
        got = 0
        while got < len(mv):
            r = f.readinto(mv[got:])
            if not r:
                raise ValueError(f"{hd.path}: the file changed while it was read")
            got += r


def read_frames(paths, *, device: int | None = None, dtype=None, threads: int = 8):
    """Batched XIM ingest: headers on a thread pool, every file's lookup table and compressed pixel buffer ``readinto`` its
    16-byte-aligned slot of ONE page-locked arena, then one device decode (one H2D copy of the compressed bytes).  All files must
    share height, width and bytes_per_pixel.  dtype None: the reference's dtype (int16 for bytes_per_pixel 1 and 2 -- the int8
    values of bpp 1 sign-extended --, int32, int64); np.uint16: the values checked against [0, 65535] (ValueError otherwise), a
    batch every ``analyze_batch`` that takes a device batch accepts.  Returns (device-resident nat.Batch, headers)."""
    from concurrent.futures import ThreadPoolExecutor

    paths = [str(p) for p in paths]
    if not paths:
        raise ValueError("no files")
    if dtype is not None and np.dtype(dtype) != np.uint16:
        raise TypeError("dtype must be None (the reference's dtype) or np.uint16")
    with ThreadPoolExecutor(max(1, min(threads, len(paths)))) as pool:
        headers = list(pool.map(read_header, paths))
        h0 = headers[0]
        key = (h0.img_height_px, h0.img_width_px, h0.bytes_per_pixel)
        for hd in headers:
            if (hd.img_height_px, hd.img_width_px, hd.bytes_per_pixel) != key:
                raise ValueError(f"{hd.path}: {hd.img_height_px} x {hd.img_width_px} at {hd.bytes_per_pixel} bytes per pixel differs "
                                 f"from the first file's {key[0]} x {key[1]} at {key[2]}")
        for hd in headers:
            check_header(hd)
        total, desc = arena_layout(headers)
        arena = nat.pinned_empty((total,), np.uint8)
        list(pool.map(lambda i: _fill(arena, headers[i], int(desc[i, 0]), int(desc[i, 2])), range(len(paths))))
    batch, status = decode_arena(arena, desc, key[0], key[1], key[2], dtype, device)
    bad = np.flatnonzero(status)
    if bad.size:
        batch.free()
        raise_status(int(status[bad[0]]), headers[bad[0]].path)
    return batch, headers


def decode_file(hd: XimHeader, device: int | None = None) -> np.ndarray:
    """The pixel array of one walked file (n = 1 through the same entry point), in the reference's dtype."""
    h, w, bpp = hd.img_height_px, hd.img_width_px, hd.bytes_per_pixel
    check_header(hd)
    total, desc = arena_layout([hd])
    arena = nat.pinned_empty((total,), np.uint8)
    _fill(arena, hd, int(desc[0, 0]), int(desc[0, 2]))
    batch, status = decode_arena(arena, desc, h, w, bpp, None, device)
    with batch:
        raise_status(int(status[0]), hd.path)
        a = batch.download()[0]
    return a.astype(np.int8) if bpp == 1 else a
