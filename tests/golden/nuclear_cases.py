"""Seeded gamma-camera flood frames for the pylinac.nuclear goldens (make_nuclear_golden.py) and the tests that check them.

CASES: name -> (frames builder, pixel size mm, PlanarUniformity.analyze kwargs, modality).  COUNT_CASES: name -> (frames builder,
frame_duration) for MaxCountRate.  Every builder is deterministic in its seed."""
from __future__ import annotations

import hashlib

import numpy as np


def digest(a) -> str:
    """sha256 of an array's dtype, shape and bytes"""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def flood(seed, shape, *, field="circle", frac=0.8, counts=200.0, background=0.3, spots=(), gradient=0.0, hot_pixels=0, blobs=(),
          dtype=np.uint16):
    """A Poisson flood: a circular or rectangular detector field of `counts` mean counts per pixel over a `background` level.
    spots: (row frac, col frac, radius frac, gain) PMT hot (gain > 1) / cold (gain < 1) spots; gradient: linear gain across the
    columns; hot_pixels: isolated bright pixels outside the field; blobs: (row, col, half size, counts) detached squares."""
    rng = np.random.default_rng(seed)
    h, w = shape
    rr, cc = np.mgrid[0:h, 0:w].astype(float)
    cy, cx = (h - 1) / 2, (w - 1) / 2
    if field == "circle":
        inside = (rr - cy) ** 2 + (cc - cx) ** 2 <= (frac * min(h, w) / 2) ** 2
    else:
        inside = (np.abs(rr - cy) <= frac * h / 2) & (np.abs(cc - cx) <= frac * w / 2)
    lam = np.where(inside, counts, background) * (1 + gradient * (cc - cx) / w)
    for fr, fc, fs, gain in spots:
        lam = np.where((rr - fr * h) ** 2 + (cc - fc * w) ** 2 <= (fs * min(h, w)) ** 2, lam * gain, lam)
    for r0, c0, hs, cnt in blobs:
        lam[max(r0 - hs, 0):r0 + hs + 1, max(c0 - hs, 0):c0 + hs + 1] = cnt
    img = rng.poisson(np.clip(lam, 0, None))
    if hot_pixels:
        out_r, out_c = np.nonzero(~inside)
        pick = rng.choice(len(out_r), size=min(hot_pixels, len(out_r)), replace=False)
        img[out_r[pick], out_c[pick]] = counts * 50
    return np.clip(img, 0, np.iinfo(dtype).max).astype(dtype)


def _line_frame():
    """a thin bright line and nothing else: the CFOV erosion of its longest side empties the CFOV"""
    f = np.zeros((40, 60), np.uint16)
    f[20, 5:55] = 1000
    return f[None]


def _two_equal():
    """two components of equal area after the filter (each loses its four corners) but different longest sides: the one with the
    lower label (the first in raster order) is the largest"""
    f = np.zeros((96, 96), np.uint16)
    f[20:60, 8:48] = 400
    f[40, 20] = 430
    f[12:92, 60:80] = 400
    return f[None]


def _window_frame():
    f = np.zeros((8, 8), np.uint16)
    f[2:6, 2:6] = 900
    return f[None]


CASES = {
    "circ_128_bin1": (lambda: flood(1, (128, 128))[None], 5.0, {}, "NM"),
    "rect_256_bin2_hot": (lambda: flood(2, (256, 256), field="rect", frac=0.85, counts=150, spots=[(0.3, 0.6, 0.06, 1.4)])[None],
                          2.4, {}, "NM"),
    "circ_512_bin4_cold_grad": (lambda: flood(3, (512, 512), counts=40, spots=[(0.55, 0.4, 0.05, 0.6)], gradient=0.2)[None],
                                1.2, {}, "NM"),
    "rect_1024_bin8_two_heads": (lambda: np.stack([flood(4, (1024, 1024), field="rect", counts=12),
                                                   flood(5, (1024, 1024), field="circle", counts=10, gradient=-0.15)]), 0.6, {}, "NM"),
    "circ_1024_bin16": (lambda: flood(6, (1024, 1024), counts=4)[None], 0.3, {}, "NM"),
    "odd_301x257_bin4": (lambda: flood(7, (301, 257), counts=30, frac=0.9)[None], 1.5, {}, "NM"),
    "odd_97x131_bin2": (lambda: flood(8, (97, 131), field="rect", counts=120)[None], 2.3, {}, "NM"),
    "hot_pixels": (lambda: flood(9, (128, 128), counts=300, frac=0.7, hot_pixels=12)[None], 4.6, {}, "NM"),
    "detached_blob": (lambda: flood(10, (128, 128), counts=300, frac=0.6, blobs=[(10, 112, 6, 300)])[None], 5.0, {}, "NM"),
    "two_equal_components": (_two_equal, 5.0, {}, "NM"),
    "tiny_field": (lambda: flood(12, (48, 48), counts=500, frac=0.18, background=0.0)[None], 5.0, {}, "NM"),
    "blank": (lambda: np.zeros((1, 64, 64), np.uint16), 5.0, {}, "NM"),
    "blank_second_frame": (lambda: np.stack([flood(13, (64, 64), counts=200), np.zeros((64, 64), np.uint16)]), 5.0, {}, "NM"),
    "window3_ratios": (lambda: flood(14, (128, 128), counts=250, spots=[(0.5, 0.5, 0.1, 1.2)])[None], 5.0,
                       {"window_size": 3, "ufov_ratio": 0.9, "cfov_ratio": 0.6, "threshold": 0.6}, "NM"),
    "window7_threshold": (lambda: flood(15, (200, 180), field="rect", counts=60, gradient=0.3)[None], 2.5,
                          {"window_size": 7, "threshold": 0.85}, "NM"),
    "u8_flood": (lambda: flood(16, (128, 128), counts=60, dtype=np.uint8)[None], 5.0, {}, "NM"),
    "thin_line": (_line_frame, 5.0, {}, "NM"),
    "window_larger_than_frame": (_window_frame, 5.0, {"window_size": 9}, "NM"),
    "not_nm": (lambda: flood(17, (32, 32))[None], 5.0, {}, "CT"),
}


def _dynamic(seed, n, tie):
    rng = np.random.default_rng(seed)
    rate = 50 + 400 * np.exp(-((np.arange(n) - n * 0.4) / (n * 0.2)) ** 2)
    frames = np.stack([rng.poisson(r, size=(32, 32)) for r in rate]).astype(np.uint16)
    if tie:                   # a later frame with the same sum as the maximum: the first one wins
        k = int(np.argmax(frames.reshape(n, -1).sum(1)))
        frames[k + 3] = frames[k][::-1]
    return frames


COUNT_CASES = {
    "dynamic_40": (lambda: _dynamic(21, 40, False), 1.0),
    "dynamic_tie": (lambda: _dynamic(22, 30, True), 0.5),
    "single_frame": (lambda: _dynamic(23, 1, False), 2.0),
}
