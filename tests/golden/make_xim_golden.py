"""Generate tests/golden/xim_golden.npz by running the UNMODIFIED reference's XIM (core/image.py:1105-1318, stub-imported) on the
seeded files of xim_cases.py: decoded arrays (sha1 + a subsample for the large ones), dtypes, properties, histogram, dpmm and the
exception type of every bad file, for read_pixels=True and False, plus each file's sha1.

Run from the repository root, where oracle/refstub.py can import the unmodified reference:  python -m tests.golden.make_xim_golden
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import tempfile
import time
import warnings

import numpy as np

from oracle.refstub import import_reference
from tests.golden.xim_cases import CASES, LARGE, SUB_COLS, SUB_ROWS, case


def sha1(b: bytes) -> np.ndarray:
    return np.frombuffer(hashlib.sha1(b).digest(), dtype=np.uint8)


def encode_value(v):
    """a property value with its Python type, as JSON"""
    if isinstance(v, np.ndarray):
        return {"t": "ndarray", "dtype": str(v.dtype), "v": v.tolist()}
    if isinstance(v, tuple):
        return {"t": "tuple", "v": list(v)}
    return {"t": type(v).__name__, "v": v}


def exc_name(e: BaseException) -> str:
    return f"{type(e).__module__}.{type(e).__qualname__}"


def main():
    warnings.simplefilter("ignore")
    import_reference()
    from pylinac.core.image import XIM

    store = {}
    tmp = tempfile.mkdtemp()
    for name in CASES:
        data, shape, bpp = case(name)
        store[f"{name}/file_sha1"] = sha1(data)
        path = os.path.join(tmp, name + ".xim")
        with open(path, "wb") as f:
            f.write(data)
        for rp in (True, False):
            key = f"{name}/{'pixels' if rp else 'header'}"
            t = time.time()
            try:
                img = XIM(path, read_pixels=rp)
            except Exception as e:  # noqa: BLE001 -- the exception type is the golden
                store[f"{key}/raised"] = np.array(exc_name(e))
                print(key, "raised", exc_name(e), e)
                continue
            store[f"{key}/raised"] = np.array("")
            meta = {k: encode_value(getattr(img, k)) for k in ("format_id", "format_version", "img_width_px", "img_height_px",
                                                                "bits_per_pixel", "bytes_per_pixel", "compression", "num_hist_bins",
                                                                "num_properties")}
            meta["properties"] = {k: encode_value(v) for k, v in img.properties.items()}
            meta["histogram"] = encode_value(img.histogram)
            meta["has_array"] = hasattr(img, "array")
            meta["pixel_buffer"] = getattr(img, "pixel_buffer", None)
            try:
                meta["dpmm"] = {"v": img.dpmm}
            except Exception as e:  # noqa: BLE001
                meta["dpmm"] = {"raised": exc_name(e)}
            store[f"{key}/meta"] = np.array(json.dumps(meta))
            if hasattr(img, "lookup_table"):
                store[f"{key}/lookup_table"] = np.asarray(img.lookup_table)
            if rp and hasattr(img, "array"):
                a = img.array
                store[f"{key}/dtype"] = np.array(str(a.dtype))
                store[f"{key}/array_sha1"] = sha1(np.ascontiguousarray(a).tobytes())
                store[f"{key}/array"] = a[SUB_ROWS, SUB_COLS] if name in LARGE else a
            print(key, "ok", round(time.time() - t, 2), "s")
    np.savez_compressed("tests/golden/xim_golden.npz", **store)


if __name__ == "__main__":
    sys.exit(main())
