"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference's XIM pixel decode (core/image.py:1186-1309) in closed form.

The reference's row loop is v[i] = d[i] + v[i-1] + v[i-W] - v[i-W-1] modulo 2^(8 bpp) for i >= W+1, v[0..W] the raw int32 head.
With e[i] = v[i] - v[i-W]: e is the inclusive scan of the diffs starting from e[W] = v[W] - v[0], and v is the per-column
inclusive scan of e below row 0.  Everything is computed in int64 (wrapping) and truncated to the reference's dtype at the end.

The reference's exceptions, in the order it raises them:
  ValueError  bytes_per_pixel not in {1, 2, 4, 8}; fewer pixel bytes than the raw head and the coded diffs need (checked run by run,
              so only the runs before the first code 3 count); one row
  IndexError  an empty lookup table (the first run is indexed), once the raw head is present
  KeyError    a 2-bit code 3 anywhere in the lookup table (LOOKUP_CONVERSION[3]), including the padding after the last diff
"""
from __future__ import annotations

import numpy as np

DTYPES = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}


def lookup_codes(lut: bytes | np.ndarray) -> np.ndarray:
    b = np.frombuffer(bytes(lut), np.uint8) if not isinstance(lut, np.ndarray) else lut.astype(np.uint8)
    return ((b[:, None] >> np.array([0, 2, 4, 6], np.uint8)) & 3).ravel()


def decode(lut, pix, h: int, w: int, bpp: int) -> np.ndarray:
    """lookup table bytes + compressed pixel bytes (as read from the file) -> the reference's array, or its exception"""
    if bpp not in DTYPES:
        raise ValueError("The XIM image has an unsupported bytes per pixel value.")
    buf = np.frombuffer(bytes(pix), np.uint8)
    codes = lookup_codes(lut)
    n_diffs = h * w - w - 1
    head = 4 * (w + 1)
    if h < 2:   # the head fills the whole (single-row) array only when exactly W values are present, then the table is indexed
        if codes.size == 0 and min(buf.size, head) == 4 * w:
            raise IndexError("empty XIM lookup table")
        raise ValueError("an XIM image needs at least two rows")
    if buf.size < head:
        raise ValueError("the XIM pixel buffer is shorter than the raw head")
    if codes.size == 0:
        raise IndexError("empty XIM lookup table")
    threes = np.flatnonzero(codes == 3)
    first3 = int(threes[0]) if threes.size else None
    c = codes[: min(n_diffs, codes.size)].astype(np.int64)
    width = np.where(c == 3, 0, 1 << np.minimum(c, 2))
    stop = n_diffs if first3 is None else min(first3, n_diffs)
    need = int(width[:stop].sum())
    if buf.size - head < need:
        raise ValueError("the XIM pixel buffer is shorter than its lookup table requires")
    if first3 is not None:
        raise KeyError(3)
    raw = buf[:head].view("<i4").astype(np.int64)
    off = head + np.concatenate([[0], np.cumsum(width)[:-1]]).astype(np.int64)
    pad = np.concatenate([buf, np.zeros(4, np.uint8)])
    b = [pad[off + k].astype(np.int64) for k in range(4)]
    u32 = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24)
    d = np.where(width == 1, u32 & 0xFF, np.where(width == 2, u32 & 0xFFFF, u32 & 0xFFFFFFFF))
    sign = np.where(width == 1, 1 << 7, np.where(width == 2, 1 << 15, 1 << 31))
    d = (d ^ sign) - sign                              # sign-extend from the code's width
    diffs = np.zeros(n_diffs, np.int64)
    diffs[: d.size] = d                                # diffs past the end of the table are 0
    flat = np.empty(h * w - w, np.int64)
    flat[0] = raw[w] - raw[0]
    flat[1:] = diffs
    e = np.cumsum(flat)                                # wraps modulo 2^64, exact modulo 2^(8 bpp)
    v = np.empty((h, w), np.int64)
    v[0] = raw[:w]
    v[1:] = raw[:w][None, :] + np.cumsum(e.reshape(h - 1, w), axis=0)
    return v.astype(DTYPES[bpp])


def as_u16(a: np.ndarray) -> np.ndarray:
    """the checked uint16 view of a decoded frame (image.frame_u16's rule for integer arrays)"""
    if a.min() < 0 or a.max() > 65535:
        raise ValueError("XIM pixel values outside [0, 65535]")
    return a.astype(np.uint16)
