"""Seeded XIM files for tests/golden/xim_golden.npz (make_xim_golden.py runs the unmodified reference's XIM on them).

case(name) -> (file bytes, expected shape, bytes_per_pixel).  Every file is rebuilt from its seed by tests/xim_writer.py; the
golden stores each file's sha1 so a change in the writer shows up as a golden mismatch rather than a silent new input."""
from __future__ import annotations

import numpy as np

from tests import xim_writer as xw

LARGE = ("epid_1024x768_bpp4", "noisy_1280x1280_bpp2")     # arrays stored as sha1 + subsample
SUB_ROWS, SUB_COLS = slice(None, None, 37), slice(None, None, 41)


def smooth_field(h: int, w: int, seed: int, peak: float = 30000.0, noise: float = 3.0) -> np.ndarray:
    """an EPID-like open field: a flat top with sloped edges plus a little noise, int64 values in [0, 65535]"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    r = np.maximum(np.abs(x - w / 2) / (0.35 * w), np.abs(y - h / 2) / (0.35 * h))
    f = peak / (1 + np.exp((r - 1) * 12)) + 800 + 0.02 * x
    return np.clip(np.rint(f + rng.normal(0, noise, (h, w))), 0, 65535).astype(np.int64)


def _arr(h, w, seed, lo, hi):
    return np.random.default_rng(seed).integers(lo, hi, (h, w), dtype=np.int64)


def _patch(b: bytes, at: int, new: bytes) -> bytes:
    return b[:at] + new + b[at + len(new):]


def case(name: str):
    if name == "bpp2_wrap_2x7":
        v = _arr(2, 7, 1, -40000, 40000)
        return xw.xim_bytes(v, 2), (2, 7), 2
    if name == "bpp1_wrap_5x9":
        v = _arr(5, 9, 2, -300, 300)
        return xw.xim_bytes(v, 1), (5, 9), 1
    if name == "bpp1_switch_9x33":
        v = _arr(9, 33, 3, -128, 128)
        return xw.xim_bytes(v, 1, layout="switch", rng=np.random.default_rng(30)), (9, 33), 1
    if name == "bpp2_switch_31x17":
        v = _arr(31, 17, 4, -40000, 40000)
        return xw.xim_bytes(v, 2, layout="switch", rng=np.random.default_rng(40)), (31, 17), 2
    if name == "bpp4_switch_33x17":
        v = _arr(33, 17, 5, -(1 << 31), (1 << 31) - 1)
        return xw.xim_bytes(v, 4, layout="switch", rng=np.random.default_rng(50)), (33, 17), 4
    if name == "bpp4_all4_20x31":
        v = smooth_field(20, 31, 6)
        return xw.xim_bytes(v, 4, layout="all4"), (20, 31), 4
    if name == "bpp8_6x11":
        v = _arr(6, 11, 7, -(1 << 29), 1 << 29)
        return xw.xim_bytes(v, 8, layout="switch", rng=np.random.default_rng(70)), (6, 11), 8
    if name == "bpp8_wide_head_7x5":
        # head values beyond int32 are truncated then sign-extended; diffs stay within int32
        v = _arr(7, 5, 8, -1000, 1000) + (np.int64(5) << 33)
        return xw.xim_bytes(v, 8), (7, 5), 8
    if name == "short_lut_16x16":
        v = smooth_field(16, 16, 9)
        return xw.xim_bytes(v, 4, n_codes=100), (16, 16), 4
    if name == "extra_pixel_bytes_12x10":
        v = smooth_field(12, 10, 10)
        return xw.xim_bytes(v, 2, comp_size_delta=13), (12, 10), 2
    if name == "code3_padding":
        v = smooth_field(8, 9, 11)
        return xw.xim_bytes(v, 2, pad_codes=[0, 0, 3]), (8, 9), 2
    if name == "code3_middle":
        v = smooth_field(12, 12, 12)
        b = xw.xim_bytes(v, 4, layout="switch", rng=np.random.default_rng(120))
        return _patch(b, xw.section_offsets(v, 4, layout="switch", rng=np.random.default_rng(120))["lut"] + 7, b"\xc0"), (12, 12), 4
    if name == "short_buffer":
        v = smooth_field(10, 11, 13)
        return xw.xim_bytes(v, 4, layout="all4", comp_size_delta=-10), (10, 11), 4
    if name == "short_before_code3":
        # the buffer runs out before the first code 3 is reached: ValueError wins
        v = smooth_field(10, 11, 14)
        return xw.xim_bytes(v, 4, layout="all4", comp_size_delta=-10, pad_codes=[3]), (10, 11), 4
    if name == "code3_before_short":
        # a code 3 early in the table, the buffer short only at the end: KeyError wins
        v = smooth_field(10, 11, 15)
        b = xw.xim_bytes(v, 4, layout="all4", comp_size_delta=-10)
        return _patch(b, xw.section_offsets(v, 4, layout="all4")["lut"] + 2, b"\x30"), (10, 11), 4
    if name == "empty_lookup":
        # an empty table: the reference indexes its first run and raises IndexError
        v = smooth_field(6, 40, 16)
        return xw.xim_bytes(v, 2, n_codes=0), (6, 40), 2
    if name == "short_head":
        # fewer pixel bytes than the raw int32 head of W + 1 values
        v = smooth_field(6, 40, 16)
        return xw.xim_bytes(v, 2, layout="all4", comp_size_delta=-860), (6, 40), 2
    if name == "bad_bpp":
        v = smooth_field(6, 7, 17)
        return _patch(xw.xim_bytes(v, 4), 8 + 16, np.array([3], "<i4").tobytes()), (6, 7), 3
    if name == "one_row":
        v = smooth_field(1, 9, 18)
        return xw.xim_bytes(v, 2), (1, 9), 2
    if name == "one_row_with_codes":
        v = smooth_field(1, 9, 18)
        return xw.xim_bytes(v, 2, pad_codes=[0]), (1, 9), 2
    if name == "trunc_header":
        return xw.xim_bytes(smooth_field(6, 7, 19), 2)[:22], (6, 7), 2
    if name == "trunc_lookup":
        v = smooth_field(30, 30, 20)
        return xw.xim_bytes(v, 2)[: xw.section_offsets(v, 2)["lut"] + 50], (30, 30), 2
    if name == "trunc_pixels":
        v = smooth_field(30, 30, 21)
        return xw.xim_bytes(v, 2, layout="all4")[: xw.section_offsets(v, 2, layout="all4")["pix"] + 700], (30, 30), 2
    if name == "trunc_trailer":
        v = smooth_field(30, 30, 22)
        return xw.xim_bytes(v, 2)[: xw.section_offsets(v, 2)["trailer"] + 6], (30, 30), 2
    if name == "uncompressed":
        v = smooth_field(4, 4, 23)
        return xw.xim_bytes(v, 2, compression=0, raw_text=b"pixel\x00text"), (4, 4), 2
    if name == "unknown_property_type":
        v = smooth_field(5, 6, 24)
        props = [("PixelWidth", xw.PROP_DOUBLE, 0.05), ("PixelHeight", xw.PROP_DOUBLE, 0.05), ("Odd", 3, None),
                 ("Empty", xw.PROP_DOUBLE_ARRAY, []), ("Name", xw.PROP_STRING, "a\x00b")]
        return xw.xim_bytes(v, 2, properties=props, histogram=[5]), (5, 6), 2
    if name == "unequal_pixel_size":
        v = smooth_field(5, 6, 25)
        props = [("PixelWidth", xw.PROP_DOUBLE, 0.0392), ("PixelHeight", xw.PROP_DOUBLE, 0.0391)]
        return xw.xim_bytes(v, 4, properties=props, histogram=[]), (5, 6), 4
    if name == "epid_1024x768_bpp4":
        v = smooth_field(768, 1024, 26)
        return xw.xim_bytes(v, 4), (768, 1024), 4
    if name == "noisy_1280x1280_bpp2":
        v = _arr(1280, 1280, 27, 0, 30000)
        return xw.xim_bytes(v, 2), (1280, 1280), 2
    raise KeyError(name)


CASES = ("bpp2_wrap_2x7", "bpp1_wrap_5x9", "bpp1_switch_9x33", "bpp2_switch_31x17", "bpp4_switch_33x17", "bpp4_all4_20x31",
         "bpp8_6x11", "bpp8_wide_head_7x5", "short_lut_16x16", "extra_pixel_bytes_12x10", "code3_padding", "code3_middle",
         "short_buffer", "short_before_code3", "code3_before_short", "empty_lookup", "short_head", "bad_bpp", "one_row",
         "one_row_with_codes", "trunc_header",
         "trunc_lookup", "trunc_pixels", "trunc_trailer", "uncompressed", "unknown_property_type", "unequal_pixel_size") + LARGE
