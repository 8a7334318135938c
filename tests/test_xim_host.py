"""CPU: the XIM header / property walk against the unmodified reference (tests/golden/xim_golden.npz), the errors the reference
raises before any pixel is decoded, and the numpy closed form of the decode (oracle/xim_oracle.py) pinned to the goldens."""
import hashlib
import json

import numpy as np
import pytest

from oracle import xim_oracle
from tests.golden.xim_cases import CASES, LARGE, SUB_ROWS, SUB_COLS, case

def _golden():
    import os

    return np.load(os.path.join(os.path.dirname(__file__), "golden", "xim_golden.npz"))


G = _golden()

# the reference's exceptions by the name stored in the golden
EXC = {"builtins.ValueError": ValueError, "builtins.KeyError": KeyError, "builtins.IndexError": IndexError,
       "struct.error": __import__("struct").error, "builtins.UnboundLocalError": UnboundLocalError}
# cases whose reference failure comes before any pixel is decoded: the host raises it without a device
NO_DEVICE_FAILURES = ("bad_bpp", "one_row", "one_row_with_codes", "empty_lookup", "short_head", "trunc_header", "trunc_lookup")


def write_case(tmp_path, name):
    data, _, _ = case(name)
    p = tmp_path / f"{name}.xim"
    p.write_bytes(data)
    return str(p)


def decode_value(d):
    t, v = d["t"], d["v"]
    if t == "ndarray":
        return np.asarray(v, dtype=d["dtype"])
    if t == "tuple":
        return tuple(v)
    return v


def assert_same_value(got, d):
    want = decode_value(d)
    assert type(got) is type(want), (got, want)
    if isinstance(want, np.ndarray):
        assert got.dtype == want.dtype and np.array_equal(got, want)
    else:
        assert got == want


def assert_meta(img, meta):
    for k in ("format_id", "format_version", "img_width_px", "img_height_px", "bits_per_pixel", "bytes_per_pixel", "compression",
              "num_hist_bins", "num_properties"):
        assert_same_value(getattr(img, k), meta[k])
    assert_same_value(img.histogram, meta["histogram"])
    assert list(img.properties) == list(meta["properties"])
    for k, d in meta["properties"].items():
        assert_same_value(img.properties[k], d)
    assert getattr(img, "pixel_buffer", None) == meta["pixel_buffer"]
    if "raised" in meta["dpmm"]:
        with pytest.raises(EXC[meta["dpmm"]["raised"]]):
            img.dpmm
    else:
        assert img.dpmm == meta["dpmm"]["v"]


@pytest.mark.parametrize("name", CASES)
def test_writer_reproduces_the_golden_files(name):
    data, _, _ = case(name)
    assert hashlib.sha1(data).digest() == G[f"{name}/file_sha1"].tobytes()


@pytest.mark.parametrize("name", CASES)
def test_header_walk_matches_reference(tmp_path, name):
    from pylinac_b200.core.image import XIM

    path = write_case(tmp_path, name)
    raised = str(G[f"{name}/header/raised"])
    if raised:
        with pytest.raises(EXC[raised]):
            XIM(path, read_pixels=False)
        return
    img = XIM(path, read_pixels=False)
    assert_meta(img, json.loads(str(G[f"{name}/header/meta"])))
    if f"{name}/header/lookup_table" in G:
        assert np.array_equal(img.lookup_table, G[f"{name}/header/lookup_table"])
    with pytest.raises(AttributeError):
        img.array


@pytest.mark.parametrize("name", NO_DEVICE_FAILURES)
def test_failures_before_the_decode_match_reference(tmp_path, name):
    from pylinac_b200.core.image import XIM

    raised = str(G[f"{name}/pixels/raised"])
    assert raised
    with pytest.raises(EXC[raised]):
        XIM(write_case(tmp_path, name))


def test_uncompressed_file_has_no_array(tmp_path):
    from pylinac_b200.core.image import XIM

    img = XIM(write_case(tmp_path, "uncompressed"))
    assert img.pixel_buffer == "pixeltext" and not hasattr(img, "array")
    assert_meta(img, json.loads(str(G["uncompressed/pixels/meta"])))


def oracle_decode_file(path):
    """the oracle on the bytes the reference reads, with its walk's ordering of errors"""
    from pylinac_b200 import xim

    hd = xim.walk(path, read_pixels=True)
    with open(path, "rb") as f:
        f.seek(hd.pix_offset)
        pix = f.read(hd.pix_bytes)
    a = xim_oracle.decode(hd.lookup_table, pix, hd.img_height_px, hd.img_width_px, hd.bytes_per_pixel)
    if hd.trailer_error is not None:
        raise hd.trailer_error
    return a, hd


@pytest.mark.parametrize("name", [c for c in CASES if c != "uncompressed"])
def test_oracle_matches_reference_goldens(tmp_path, name):
    path = write_case(tmp_path, name)
    raised = str(G[f"{name}/pixels/raised"])
    if raised:
        with pytest.raises(EXC[raised]):
            oracle_decode_file(path)
        return
    a, _ = oracle_decode_file(path)
    assert str(a.dtype) == str(G[f"{name}/pixels/dtype"])
    assert hashlib.sha1(np.ascontiguousarray(a).tobytes()).digest() == G[f"{name}/pixels/array_sha1"].tobytes()
    want = G[f"{name}/pixels/array"]
    assert np.array_equal(a[SUB_ROWS, SUB_COLS] if name in LARGE else a, want)


def test_oracle_u16_rule():
    assert xim_oracle.as_u16(np.array([[0, 65535]], np.int32)).dtype == np.uint16
    for bad in (-1, 65536):
        with pytest.raises(ValueError):
            xim_oracle.as_u16(np.array([[0, bad]], np.int32))
