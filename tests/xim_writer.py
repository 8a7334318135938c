"""Test helper: write Varian XIM files (the layout XIM reads, core/image.py:1105-1318) from an integer array, without the vendor
encoder.  The pixel stream is the reference's: the first W + 1 values raw int32, then for raster index i = W+1 .. H*W-1 the diff
d = v[i] - v[i-1] - v[i-W] + v[i-W-1] (modulo 2^(8 bpp)) in 1, 2 or 4 bytes, the width of each diff given by a 2-bit lookup code
(four per byte, LSB first).  Options force the code layouts the decoder must handle."""
from __future__ import annotations

import struct

import numpy as np

PROP_INT, PROP_DOUBLE, PROP_STRING, PROP_DOUBLE_ARRAY, PROP_INT_ARRAY = 0, 1, 2, 4, 5
_DTYPES = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}


def diffs(v: np.ndarray, bpp: int) -> np.ndarray:
    """the reference's diffs of `v` (H x W), as signed values of the bpp-byte dtype (int64 array of length H*W - W - 1)"""
    h, w = v.shape
    f = v.astype(np.int64).ravel()
    i = np.arange(w + 1, h * w)
    d = f[i] - f[i - 1] - f[i - w] + f[i - w - 1]
    return d.astype(_DTYPES[bpp]).astype(np.int64)


def min_widths(d: np.ndarray) -> np.ndarray:
    """smallest code (0: 1 byte, 1: 2 bytes, 2: 4 bytes) that holds each diff"""
    c = np.full(d.shape, 2, np.uint8)
    c[(d >= -32768) & (d <= 32767)] = 1
    c[(d >= -128) & (d <= 127)] = 0
    return c


def pack_codes(codes: np.ndarray) -> bytes:
    c = np.asarray(codes, np.uint8)
    c = np.concatenate([c, np.zeros((-len(c)) % 4, np.uint8)]).reshape(-1, 4)
    return (c[:, 0] | (c[:, 1] << 2) | (c[:, 2] << 4) | (c[:, 3] << 6)).astype(np.uint8).tobytes()


def encode_pixels(v: np.ndarray, bpp: int, layout: str = "min", rng=None, n_codes: int | None = None, pad_codes=None):
    """-> (lookup table bytes, compressed pixel bytes).

    layout: 'min' smallest width per diff; 'all4' every diff 4 bytes; 'switch' widths switch at single elements (every diff at
    least its minimum, widened at random to 2 / 4 bytes: the 1-element runs of the RAM-2414 regression).
    n_codes: write only the first n_codes codes (and their diffs): the decoder treats the rest as 0.
    pad_codes: extra 2-bit codes appended after the last one (e.g. [3] for code-3 padding)."""
    h, w = v.shape
    d = diffs(v, bpp)
    codes = min_widths(d)
    if layout == "all4":
        codes[:] = 2
    elif layout == "switch":
        rng = rng or np.random.default_rng(0)
        up = rng.integers(0, 3, d.size).astype(np.uint8)
        codes = np.maximum(codes, up)
    elif layout != "min":
        raise ValueError(layout)
    if n_codes is not None:
        codes, d = codes[:n_codes], d[:n_codes]
    head = v.ravel()[: w + 1].astype(np.int64).astype(np.int32).astype("<i4").tobytes()
    width = (1 << codes.astype(np.int64))
    off = np.concatenate([[0], np.cumsum(width)[:-1]]).astype(np.int64)
    u = d.astype(np.uint64)                            # two's complement: the low bytes are the value modulo the code's width
    buf = np.zeros(int(width.sum()), np.uint8)
    for k in range(4):
        sel = width > k
        buf[off[sel] + k] = ((u[sel] >> np.uint64(8 * k)) & np.uint64(0xFF)).astype(np.uint8)
    pix = head + buf.tobytes()
    all_codes = codes if pad_codes is None else np.concatenate([codes, np.asarray(pad_codes, np.uint8)])
    return pack_codes(all_codes), pix


def _prop(name: str, kind: int, value) -> bytes:
    nb = name.encode("ascii")
    out = struct.pack("<i", len(nb)) + nb + struct.pack("<i", kind)
    if kind == PROP_INT:
        return out + struct.pack("<i", int(value))
    if kind == PROP_DOUBLE:
        return out + struct.pack("<d", float(value))
    if kind == PROP_STRING:
        b = value.encode("ascii") if isinstance(value, str) else bytes(value)
        return out + struct.pack("<i", len(b)) + b
    if kind == PROP_DOUBLE_ARRAY:
        return out + struct.pack("<i", 8 * len(value)) + struct.pack("<%dd" % len(value), *value)
    if kind == PROP_INT_ARRAY:
        return out + struct.pack("<i", 4 * len(value)) + struct.pack("<%di" % len(value), *value)
    return out                                          # unknown type: no value bytes (the reader keeps the previous value)


DEFAULT_PROPS = [("PixelWidth", PROP_DOUBLE, 0.0392), ("PixelHeight", PROP_DOUBLE, 0.0392), ("GantryRtn", PROP_DOUBLE, 180.0),
                 ("MVCollimatorRtn", PROP_DOUBLE, 90.0), ("CouchRtn", PROP_DOUBLE, 0.0), ("KVSourceRtn", PROP_DOUBLE, 90.0),
                 ("AcqType", PROP_STRING, "Image"), ("MVBeamEnergy", PROP_INT, 6), ("PixelOffsets", PROP_INT_ARRAY, [1, -2, 3]),
                 ("KVFilterPos", PROP_DOUBLE_ARRAY, [0.5, 1.25]), ("OneDouble", PROP_DOUBLE_ARRAY, [2.5]),
                 ("OneInt", PROP_INT_ARRAY, [7]), ("NoInts", PROP_INT_ARRAY, [])]


def xim_bytes(v: np.ndarray, bpp: int = 4, *, layout: str = "min", rng=None, n_codes=None, pad_codes=None, properties=None,
              histogram=None, compression: int = 1, bits_per_pixel: int | None = None, format_version: int = 3,
              comp_size_delta: int = 0, raw_text: bytes = b"") -> bytes:
    """the bytes of a whole XIM file.  comp_size_delta: declared pixel-buffer size minus the bytes written (negative: a buffer
    shorter than the codes need).  compression=0 writes `raw_text` as the (text) pixel buffer."""
    v = np.asarray(v)
    h, w = v.shape
    props = DEFAULT_PROPS if properties is None else properties
    hist = np.arange(7, dtype=np.int32) * 3 if histogram is None else np.asarray(histogram, np.int32)
    out = b"VMS.XI\x00\x00" + struct.pack("<6i", format_version, w, h, bits_per_pixel or 8 * bpp, bpp, compression)
    if compression:
        lut, pix = encode_pixels(v, bpp, layout, rng, n_codes, pad_codes)
        if comp_size_delta < 0:
            pix = pix[: len(pix) + comp_size_delta]
        elif comp_size_delta > 0:
            pix = pix + b"\x5a" * comp_size_delta      # bytes past the last diff are ignored
        out += struct.pack("<i", len(lut)) + lut + struct.pack("<i", len(pix)) + pix + struct.pack("<i", h * w * bpp)
    else:
        out += struct.pack("<i", len(raw_text)) + raw_text
    out += struct.pack("<i", len(hist)) + hist.astype("<i4").tobytes()
    out += struct.pack("<i", len(props)) + b"".join(_prop(*p) for p in props)
    return out


def write_xim(path, v, bpp: int = 4, *, truncate: int | None = None, **kw) -> str:
    """write xim_bytes(v, bpp, **kw) to `path`, optionally cut to its first `truncate` bytes"""
    b = xim_bytes(v, bpp, **kw)
    if truncate is not None:
        b = b[:truncate]
    with open(path, "wb") as f:
        f.write(b)
    return str(path)


def section_offsets(v, bpp: int = 4, **kw) -> dict:
    """byte offsets of the sections of xim_bytes(v, bpp, **kw): 'lut' (lookup bytes), 'pix' (pixel bytes), 'trailer'"""
    h, w = np.asarray(v).shape
    lut, pix = encode_pixels(np.asarray(v), bpp, kw.get("layout", "min"), kw.get("rng"), kw.get("n_codes"), kw.get("pad_codes"))
    lut0 = 8 + 24 + 4
    pix0 = lut0 + len(lut) + 4
    return {"lut": lut0, "pix": pix0, "trailer": pix0 + len(pix)}
