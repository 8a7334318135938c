"""GPU: the XIM pixel decode (csrc/xim.cu) against the unmodified reference's goldens and the numpy closed form (oracle/xim_oracle.py,
pinned to the goldens by tests/test_xim_host.py), batched ingest with mixed compressed sizes, every per-frame status, the uint16
range check, and XIM frames through the image metrics and PicketFence."""
import hashlib
import json

import numpy as np
import pytest

from oracle import xim_oracle
from tests import xim_writer as xw
from tests.golden.xim_cases import CASES, LARGE, SUB_COLS, SUB_ROWS, case, smooth_field
from tests.test_xim_host import EXC, G, assert_meta, write_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", [c for c in CASES if c != "uncompressed"])
def test_decode_matches_reference_goldens(tmp_path, name):
    from pylinac_b200.core.image import XIM

    path = write_case(tmp_path, name)
    raised = str(G[f"{name}/pixels/raised"])
    if raised:
        with pytest.raises(EXC[raised]):
            XIM(path)
        return
    img = XIM(path)
    a = img.array
    assert str(a.dtype) == str(G[f"{name}/pixels/dtype"])
    assert hashlib.sha1(np.ascontiguousarray(a).tobytes()).digest() == G[f"{name}/pixels/array_sha1"].tobytes()
    assert np.array_equal(a[SUB_ROWS, SUB_COLS] if name in LARGE else a, G[f"{name}/pixels/array"])
    assert_meta(img, json.loads(str(G[f"{name}/pixels/meta"])))


def _oracle(path):
    from pylinac_b200 import xim

    hd = xim.walk(path)
    with open(path, "rb") as f:
        f.seek(hd.pix_offset)
        return xim_oracle.decode(hd.lookup_table, f.read(hd.pix_bytes), hd.img_height_px, hd.img_width_px, hd.bytes_per_pixel)


SPANS = {1: 300, 2: 40000, 4: 3_000_000_000, 8: 1 << 40}


@pytest.mark.parametrize("bpp", [1, 2, 4, 8])
@pytest.mark.parametrize("shape", [(2, 5), (2, 4099), (7, 333), (768, 1024), (1280, 1280)])
@pytest.mark.parametrize("layout", ["min", "switch"])
def test_decode_matches_oracle_with_wraparound(tmp_path, bpp, shape, layout):
    from pylinac_b200.core.image import XIM

    rng = np.random.default_rng(1000 * bpp + 7 * shape[0] + shape[1] + (layout == "switch"))
    if bpp == 8:      # diffs must fit the widest (4-byte) code
        v = np.cumsum(rng.integers(-(1 << 28), 1 << 28, shape), axis=1) // 4
    else:
        v = rng.integers(-SPANS[bpp], SPANS[bpp], shape)
    path = xw.write_xim(tmp_path / "f.xim", v, bpp, layout=layout, rng=rng)
    a = XIM(path).array
    want = _oracle(path)
    assert a.dtype == want.dtype and np.array_equal(a, want)
    if bpp < 8:
        assert np.array_equal(a, v.astype(want.dtype))     # modular round trip of the writer's array


def test_batch_of_mixed_compressed_sizes(tmp_path):
    """40 frames of 300 x 257 (19 tiles each) with every code layout: one arena, one launch sequence"""
    from pylinac_b200 import xim

    rng = np.random.default_rng(5)
    paths = []
    for i in range(40):
        v = smooth_field(300, 257, 100 + i, noise=[1.0, 30.0, 3000.0][i % 3])
        layout = ["min", "switch", "all4"][(i // 3) % 3]
        paths.append(xw.write_xim(tmp_path / f"{i}.xim", v, 4, layout=layout, rng=rng, comp_size_delta=(i % 5) * 3))
    sizes = {xim.read_header(p).pix_bytes for p in paths}
    assert len(sizes) > 10
    batch, headers = xim.read_frames(paths)
    try:
        got = batch.download()
    finally:
        batch.free()
    assert got.shape == (40, 300, 257) and got.dtype == np.int32
    for i, p in enumerate(paths):
        assert np.array_equal(got[i], _oracle(p)), i
    batch, _ = xim.read_frames(paths, dtype=np.uint16)
    try:
        got16 = batch.download()
    finally:
        batch.free()
    assert np.array_equal(got16, got.astype(np.uint16))


def test_every_status_in_one_launch(tmp_path):
    from pylinac_b200 import _native as nat
    from pylinac_b200 import xim

    v = smooth_field(40, 50, 1)
    neg = v.copy()
    neg[3, 4] = -1
    files = [xw.write_xim(tmp_path / "ok.xim", v, 4),
             xw.write_xim(tmp_path / "c3.xim", v, 4, pad_codes=[3]),
             xw.write_xim(tmp_path / "short.xim", v, 4, layout="all4", comp_size_delta=-40),
             xw.write_xim(tmp_path / "neg.xim", neg, 4)]
    headers = [xim.walk(p) for p in files]
    total, desc = xim.arena_layout(headers)
    arena = nat.pinned_empty((total,), np.uint8)
    for hd, d in zip(headers, desc):
        xim._fill(arena, hd, int(d[0]), int(d[2]))
    batch, status = xim.decode_arena(arena, desc, 40, 50, 4, np.uint16)
    batch.free()
    assert status.tolist() == [nat.XIM_OK, nat.XIM_LOOKUP_CODE3, nat.XIM_SHORT_BUFFER, nat.XIM_U16_RANGE]
    batch, status = xim.decode_arena(arena, desc, 40, 50, 4)
    got = batch.download()
    batch.free()
    assert status.tolist() == [nat.XIM_OK, nat.XIM_LOOKUP_CODE3, nat.XIM_SHORT_BUFFER, nat.XIM_OK]
    assert np.array_equal(got[3], neg) and np.array_equal(got[0], v)
    for p, exc in zip(files[1:3], (KeyError, ValueError)):
        with pytest.raises(exc):
            xim.read_frames([files[0], p])
    with pytest.raises(ValueError):
        xim.read_frames(files[3:], dtype=np.uint16)


@pytest.mark.parametrize("value, ok", [(0, True), (65535, True), (-1, False), (65536, False)])
def test_u16_range_check(tmp_path, value, ok):
    from pylinac_b200 import xim

    v = smooth_field(64, 70, 2)
    v[10, 11] = value
    p = xw.write_xim(tmp_path / "u.xim", v, 4)
    if not ok:
        with pytest.raises(ValueError):
            xim.read_frames([p], dtype=np.uint16)
        return
    batch, _ = xim.read_frames([p], dtype=np.uint16)
    got = batch.download()[0]
    batch.free()
    assert got.dtype == np.uint16 and np.array_equal(got, v.astype(np.uint16)) and got[10, 11] == value


def test_disk_locator_on_xim_equals_array_image(tmp_path):
    from pylinac_b200.core.image import XIM, ArrayImage
    from pylinac_b200.metrics.image import SizedDiskLocator
    from tests.test_gpu_metrics import create_bb_image

    fr = create_bb_image(bb_size=5)
    props = [("PixelWidth", xw.PROP_DOUBLE, fr.pixel_size / 10), ("PixelHeight", xw.PROP_DOUBLE, fr.pixel_size / 10)]
    img = XIM(xw.write_xim(tmp_path / "bb.xim", fr.image.astype(np.int64), 4, properties=props))
    assert np.array_equal(img.array, fr.image)

    class Same(ArrayImage):
        dpmm = img.dpmm

    ref = Same(img.array.copy())
    kw = dict(expected_position=(511.5, 383.5), search_window=(50, 50), radius=6, radius_tolerance=1, max_number=1)
    a = img.compute(metrics=[SizedDiskLocator(**kw)])
    b = ref.compute(metrics=[SizedDiskLocator(**kw)])
    assert len(a) == len(b) == 1 and (a[0].x, a[0].y) == (b[0].x, b[0].y)


def test_picketfence_from_xim_batch_equals_uint16_frames(tmp_path):
    from oracle import synth
    from pylinac_b200 import picketfence as pf
    from pylinac_b200 import xim

    frames = np.stack([synth.bench_pf_frame(i) for i in range(6)])
    paths = [xw.write_xim(tmp_path / f"pf{i}.xim", f.astype(np.int64), 4) for i, f in enumerate(frames)]
    batch, _ = xim.read_frames(paths, dtype=np.uint16)
    try:
        assert np.array_equal(batch.download(), frames)
        r_x = pf.analyze_batch(batch, 2.56)
    finally:
        batch.free()
    r_u = pf.analyze_batch(frames, 2.56)
    assert r_x.summary.tobytes() == r_u.summary.tobytes()
    assert r_x.meas.tobytes() == r_u.meas.tobytes()
