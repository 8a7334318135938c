"""Frame statistics against numpy at their edges.

Integer results (min, max, sums, histograms) must be bit-exact and percentiles must equal ``np.percentile(..., method="linear")``
bit for bit, on every kernel path of ``epid_frame_stats`` / ``epid_frame_histogram`` (stats.cu).  The certified decisions
(FieldAnalysis / Starshot inversion, PicketFence's noise and orientation front end) must equal what numpy decides, whether the
frame is certified from counts or falls back to exact order statistics.  Every adversarial case asserts the counter deltas or
launch counts that prove it reached the path it targets.
"""
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SWEEP_SHAPES = [(1024, 1024), (1008, 1008), (1280, 1280), (1190, 1190), (768, 1024), (384, 512), (300, 400), (1001, 1019)]
EXTRA_Q = [0.5, 4, 5, 50, 85, 90, 95, 96, 99, 99.5, 99.9]
SWEEP_Q = np.concatenate([np.arange(10001) / 100.0, EXTRA_Q])


@pytest.fixture(scope="module")
def ctx():
    from pylinac_b200 import _native as nat

    c = nat.Context.default()
    yield c
    for opt in (nat.OPT_PF_EXACT_ONLY, nat.OPT_STATS_EXACT):
        c.set_option(opt, 0)


def _plan(n, q):
    """np.percentile's "linear" plan (the virtual index (n - 1) * q / 100), used only to build frames near a rank."""
    vi = (n - 1) * (q / 100.0)
    if vi >= n - 1:
        return n - 1, n - 1
    p = int(np.floor(vi))
    return p, p + 1


def _stats(ctx, frames, view=None, qs=()):
    from pylinac_b200 import _native as nat

    b = nat.Batch.upload(ctx, frames)
    try:
        return nat.frame_stats(ctx, b, view=view, percentiles=qs), nat.frame_histogram(ctx, b, view=view)
    finally:
        b.free()


def _check(ctx, frames, label, view=None, qs=(0, 0.5, 5, 50, 95, 99.5, 100)):
    """frame_stats + frame_histogram of every frame's view equal numpy's."""
    frames = np.asarray(frames)
    if frames.ndim == 2:
        frames = frames[None]
    n, h, w = frames.shape
    r0, c0, vh, vw = view if view is not None else (0, 0, h, w)
    st, hist = _stats(ctx, frames, view, qs)
    for i in range(n):
        sub = frames[i, r0:r0 + vh, c0:c0 + vw]
        msg = f"{label}, frame {i}, view {(r0, c0, vh, vw)} of {frames.shape} {frames.dtype}"
        assert st["min"][i] == sub.min() and st["max"][i] == sub.max(), msg
        assert st["sum"][i] == sub.sum(dtype=np.int64), msg
        np.testing.assert_array_equal(st["rowsum"][i], sub.sum(axis=1, dtype=np.int64), err_msg=msg)
        np.testing.assert_array_equal(st["colsum"][i], sub.sum(axis=0, dtype=np.int64), err_msg=msg)
        if len(qs):
            np.testing.assert_array_equal(st["percentiles"][i], np.percentile(sub, qs), err_msg=f"{msg}, q = {list(qs)}")
        np.testing.assert_array_equal(hist[i], np.bincount(sub.ravel(), minlength=65536), err_msg=msg)


# ------------------------------------------------------------------------------------------------ a. percentile sweep
@pytest.mark.parametrize("shape", SWEEP_SHAPES, ids=[f"{h}x{w}" for h, w in SWEEP_SHAPES])
def test_percentile_sweep_equals_numpy(ctx, shape):
    """q = 0 .. 100 in steps of 0.01 plus the module percentiles, on a random frame and on a permutation of arange(n) % 65536
    (adjacent order statistics differ often, so any error in the interpolation weight shows)."""
    from pylinac_b200 import _native as nat

    h, w = shape
    n = h * w
    rng = np.random.default_rng(n)
    frames = np.stack([rng.integers(0, 65536, shape, dtype=np.uint16),
                       rng.permutation(np.arange(n) % 65536).astype(np.uint16).reshape(shape)])
    ref = np.stack([np.percentile(f, SWEEP_Q) for f in frames])
    got = np.empty_like(ref)
    b = nat.Batch.upload(ctx, frames)
    try:
        for k in range(0, len(SWEEP_Q), 8):
            got[:, k:k + 8] = nat.frame_stats(ctx, b, percentiles=SWEEP_Q[k:k + 8])["percentiles"]
    finally:
        b.free()
    bad = [(("random", "permutation")[i], float(SWEEP_Q[j]), float(got[i, j]), float(ref[i, j])) for i, j in zip(*np.nonzero(got != ref))]
    assert not bad, f"{shape}: {len(bad)} percentiles differ from np.percentile (frame, q, device, numpy), first: {bad[:6]}"


# ------------------------------------------------------------------------------------------------ b. paths and shapes
def test_histogram_kernel_widths_and_column_strips(ctx):
    """k_hist_view with 4 and 8 vectors per lane (W <= 1010, 1011 .. 2040), and views wider than 2040 columns cut into strips of 2040
    columns, up to 4096."""
    rng = np.random.default_rng(1)
    for h, w in [(37, 1000), (33, 1010), (41, 1011), (29, 1024), (23, 1500), (17, 2040), (17, 2041), (64, 4096), (4096, 16), (300, 2100)]:
        frames = rng.integers(0, 65536, (2, h, w), dtype=np.uint16)
        frames[1] = rng.integers(30000, 30100, (h, w))
        _check(ctx, frames, f"{h}x{w}")


def test_column_offsets_and_unaligned_pitch(ctx):
    """Views at every 16-byte misalignment (column offsets 0..7) for each kernel, and batches whose width is not a multiple of
    8 pixels (the scalar-load path)."""
    rng = np.random.default_rng(2)
    for w, vw in [(1040, 1000), (1520, 1500), (2056, 2041)]:
        frames = rng.integers(0, 65536, (2, 40, w), dtype=np.uint16)
        for c0 in range(8):
            _check(ctx, frames, f"offset {c0}", view=(3, c0, 33, vw))
    for w in (1037, 2045, 13):
        frames = rng.integers(0, 65536, (2, 21, w), dtype=np.uint16)
        _check(ctx, frames, f"pitch {w}")
        _check(ctx, frames, f"pitch {w}, offset 3", view=(1, 3, 19, w - 5))


def test_histogram_of_a_view_wider_than_4096_columns(ctx):
    """frame_histogram takes views wider than frame_stats' 4096 columns (three 2040-column strips, the last one partial)."""
    from pylinac_b200 import _native as nat

    rng = np.random.default_rng(10)
    frames = rng.integers(0, 65536, (2, 8, 5008), dtype=np.uint16)
    frames[1] = rng.integers(30000, 30100, (8, 5008))
    b = nat.Batch.upload(ctx, frames)
    try:
        hist = nat.frame_histogram(ctx, b, view=(0, 3, 8, 5000))
    finally:
        b.free()
    for i in range(2):
        np.testing.assert_array_equal(hist[i], np.bincount(frames[i, :, 3:5003].ravel(), minlength=65536), err_msg=str(i))


def test_degenerate_views(ctx):
    rng = np.random.default_rng(3)
    frames = rng.integers(0, 65536, (3, 50, 3000), dtype=np.uint16)
    for view in [(7, 9, 1, 1), (0, 0, 1, 3000), (0, 0, 1, 2040), (4, 5, 1, 37), (0, 0, 50, 1), (3, 2999, 47, 1), (0, 0, 2, 2041)]:
        _check(ctx, frames, "degenerate", view=view, qs=(0, 1, 33.3, 50, 100))


def test_uint8_batches(ctx):
    rng = np.random.default_rng(4)
    for h, w in [(64, 1000), (32, 2100), (19, 37)]:
        frames = rng.integers(0, 256, (2, h, w), dtype=np.uint8)
        _check(ctx, frames, "uint8")
        _check(ctx, frames, "uint8 view", view=(1, 3, h - 2, w - 5))


def test_constant_two_value_and_extreme_frames(ctx):
    for h, w in [(48, 1000), (64, 2040), (64, 4096)]:
        frames = np.stack([np.full((h, w), 7, np.uint16), np.zeros((h, w), np.uint16), np.full((h, w), 65535, np.uint16),
                           np.where(np.indices((h, w)).sum(0) % 2 == 0, 0, 65535).astype(np.uint16),
                           np.where(np.arange(w) < w // 3, 12, 13).astype(np.uint16)[None].repeat(h, 0)])
        _check(ctx, frames, f"extreme {h}x{w}", qs=(0, 0.01, 33.33, 50, 66.67, 99.99, 100))


@pytest.mark.parametrize("value", [1000, 1001, "both"])
@pytest.mark.parametrize("w", [4096, 2040])
def test_more_than_65535_equal_pixels(ctx, value, w):
    """More than 65535 pixels of one even or odd value would overflow a 16-bit bin counter; k_hist_view counts in 32 bits, in
    one column strip (W = 2040) and in three (W = 4096).  Ranks at both ends of the repeated value and of its odd / even
    neighbour are read."""
    h = 64
    n = h * w
    rng = np.random.default_rng(w + (value if isinstance(value, int) else 7))
    a = rng.integers(0, 3000, n).astype(np.uint16)
    idx = rng.permutation(n)
    vals = (1000, 1001) if value == "both" else (value,)
    for k, v in enumerate(vals):
        a[idx[k * 70000:(k + 1) * 70000]] = v
    a = a.reshape(h, w)
    counts = np.bincount(a.ravel(), minlength=65536)
    assert counts.max() > 65535, "the frame must overflow a 16-bit bin counter"
    s = np.sort(a.ravel())
    qs = []
    for v in vals:
        lo, hi = np.searchsorted(s, v), np.searchsorted(s, v, side="right") - 1
        qs += [100.0 * r / (n - 1) for r in (lo - 1, lo, hi, hi + 1) if 0 <= r < n]
    _check(ctx, a, f"value {value}, {h}x{w}", qs=qs[:8])
    _check(ctx, a, f"value {value}, {h}x{w}", qs=(0, 1, 25, 50, 75, 99, 100))


def test_batch_of_300_frames_crosses_the_256_frame_chunk(ctx):
    from pylinac_b200 import _native as nat

    rng = np.random.default_rng(5)
    frames = rng.integers(0, 65536, (300, 24, 40), dtype=np.uint16)
    frames[::7] //= 3
    b = nat.Batch.upload(ctx, frames)
    try:
        l0 = ctx.launches()
        st = nat.frame_stats(ctx, b, percentiles=(0, 5, 50, 95, 100))
        launches = ctx.launches() - l0
        hist = nat.frame_histogram(ctx, b)
    finally:
        b.free()
    # k_refs_from_batch + (k_hist_view, k_stats_from_hist) per chunk of 256 frames
    assert launches == 1 + 2 * 2, f"{launches} launches for 300 frames: expected two 256-frame chunks"
    for i in range(300):
        f = frames[i]
        assert (st["min"][i], st["max"][i], st["sum"][i]) == (f.min(), f.max(), f.sum(dtype=np.int64)), i
        np.testing.assert_array_equal(st["rowsum"][i], f.sum(axis=1), err_msg=str(i))
        np.testing.assert_array_equal(st["colsum"][i], f.sum(axis=0), err_msg=str(i))
        np.testing.assert_array_equal(st["percentiles"][i], np.percentile(f, (0, 5, 50, 95, 100)), err_msg=str(i))
        np.testing.assert_array_equal(hist[i], np.bincount(f.ravel(), minlength=65536), err_msg=str(i))


def test_error_codes(ctx):
    from pylinac_b200 import _native as nat

    a16 = np.zeros((2, 16, 32), np.uint16)
    a8 = np.zeros((2, 16, 32), np.uint8)
    for arr in (a16, a8):
        b = nat.Batch.upload(ctx, arr)
        try:
            with pytest.raises(nat.NativeError):
                nat.frame_stats(ctx, b, percentiles=list(range(9)))
            for q in (-0.001, 100.001, float("nan")):
                with pytest.raises(ValueError, match="range"):
                    nat.frame_stats(ctx, b, percentiles=[50, q])
            for view in [(0, 0, 17, 32), (0, 1, 16, 32), (-1, 0, 4, 4), (0, 0, 0, 4)]:
                with pytest.raises(ValueError):
                    nat.frame_stats(ctx, b, view=view, percentiles=[50])
                with pytest.raises(ValueError):
                    nat.frame_histogram(ctx, b, view=view)
            assert nat.frame_stats(ctx, b, percentiles=[0, 100])["percentiles"].tolist() == [[0, 0], [0, 0]]
        finally:
            b.free()
    bf = nat.Batch.upload(ctx, a16.astype(np.float32))
    try:
        with pytest.raises(nat.NativeError):
            nat.frame_stats(ctx, bf, percentiles=[50])
        with pytest.raises(nat.NativeError):
            nat.frame_histogram(ctx, bf)
    finally:
        bf.free()


def test_array_utils_percentile_equals_numpy(ctx):
    from pylinac_b200.core import array_utils as au

    rng = np.random.default_rng(6)
    a = rng.integers(0, 65536, (768, 1024), dtype=np.uint16)
    for q in (1, 2.5, 95, 99.5):
        assert au.percentile(a, q) == np.percentile(a, q), q
    b = rng.integers(0, 65536, (300, 400), dtype=np.uint16)
    for q in (2.5, 95):
        assert au.percentile(b, q) == np.percentile(b, q), q


# ------------------------------------------------------------------------------------------------ c. certified inversion
PILOT_ROWS, PILOT_COLS = 16, 256     # k_inv_pilot's sample grid (stats.cu)


def _pilot_grid(h, w):
    rows = np.minimum(h - 1, ((2 * np.arange(PILOT_ROWS) + 1) * h) // (2 * PILOT_ROWS))
    cols = np.minimum(w - 1, ((2 * np.arange(PILOT_COLS) + 1) * w) // (2 * PILOT_COLS))
    return np.ix_(rows, cols)


def _rank_ramp(f, qs, targets, steps=(0, 0, 0)):
    """A frame with the ranks of ``f`` (ties broken by position) whose sorted values rise linearly between knots: the
    order statistics around percentile qs[k] take the value targets[k] (and targets[k] + steps[k] at the upper rank), so the
    two distances of check_inversion_by_histogram are set exactly.  Monotone in the rank: the image keeps its structure.  The
    values rise gently past the last knot, so that the pilot's brackets stay narrow enough to certify far from a tie."""
    n = f.size
    order = np.argsort(f.ravel(), kind="stable")
    kx, ky = [0], [0.0]
    for q, t, s in zip(qs, targets, steps):
        p, nx = _plan(n, q)
        kx += [p, nx]
        ky += [t, t + s]
    kx.append(n - 1)
    ky.append(min(65535.0, ky[-1] + 2000))
    vals = np.rint(np.interp(np.arange(n), kx, ky)).astype(np.uint16)
    out = np.empty(n, np.uint16)
    out[order] = vals
    return out.reshape(f.shape)


def _np_inverted(a, qs):
    lo, mid, hi = np.percentile(a, qs)
    return int(abs(mid - lo) > abs(mid - hi))


def _field_frames(shape):
    import bench

    out = {}
    for i in range(2):
        f = bench._gen_module_frames(("field", i))
        if shape != f.shape:
            t, l = (f.shape[0] - shape[0]) // 2, (f.shape[1] - shape[1]) // 2
            f = np.ascontiguousarray(f[t:t + shape[0], l:l + shape[1]])
        out[f"field{i}"] = f
    f = out["field0"]
    out["saturated"] = (65535 - f.astype(np.int64)).astype(np.uint16)        # > 5 % of pixels at 65535 (and field0: > 5 % zeros)
    D = 20000
    # (step at the p5 pair, offset of p95): d1 - d2 = -step * gamma5 - delta, gamma5 ~ 0.95 for both shapes
    for step, delta in [(0, 0), (0, 1), (0, -1), (10, -9), (10, -10), (0, 8000), (0, -8000)]:
        out[f"ramp_s{step}_d{delta}"] = _rank_ramp(f, (5, 50, 95), (2000, 2000 + D, 2000 + 2 * D + delta), (step, 0, 0))
    rows, cols = _pilot_grid(*shape)
    for name in ("field0", "ramp_s0_d0", "ramp_s0_d-8000"):
        for lie in (0, 65535):
            g = out[name].copy()
            g[rows, cols] = lie
            out[f"{name}_pilot{lie}"] = g
    return out


@pytest.mark.parametrize("shape", [(1280, 1280), (1190, 1190)], ids=["1280", "1190"])
def test_field_inversion_decision_equals_numpy(ctx, shape):
    from pylinac_b200 import _native as nat
    from pylinac_b200 import field_analysis as fa

    cases = _field_frames(shape)
    names = list(cases)
    dpmm = 1 / 0.336
    rows, unc = {}, {}
    try:
        ctx.set_option(nat.OPT_STATS_EXACT, 1)
        exact = fa.analyze_batch(np.stack([cases[k] for k in names]), dpmm).rows.copy()
        ctx.set_option(nat.OPT_STATS_EXACT, 0)
        for k in names:       # one frame per call: the uncertified-frame counter delta belongs to that frame
            u0 = ctx.counter(nat.CTR_STATS_UNCERTIFIED)
            rows[k] = fa.analyze_batch(cases[k][None], dpmm).rows.copy()[0]
            unc[k] = ctx.counter(nat.CTR_STATS_UNCERTIFIED) - u0
    finally:
        ctx.set_option(nat.OPT_STATS_EXACT, 0)
    report = {k: (int(rows[k]["hist_inverted"]), unc[k]) for k in names}
    for i, k in enumerate(names):
        assert int(rows[k]["hist_inverted"]) == _np_inverted(cases[k], (5, 50, 95)), f"{k}: (inverted, uncertified) = {report}"
        for f in exact.dtype.names:
            np.testing.assert_array_equal(rows[k][f], exact[f][i], err_msg=f"{k}/{f}; (inverted, uncertified) = {report}")
    assert all(unc[k] == 1 for k in names if "_d0" in k or "_d1" in k or "_d-1" in k or "_s10" in k), f"near ties must fall back: {report}"
    assert unc["field0"] == 0 and unc["ramp_s0_d-8000"] == 0, f"frames far from the boundary must certify: {report}"
    assert {report[k][0] for k in names} == {0, 1}, report


def test_field_inversion_geometry_gates(ctx):
    """launch_frame_stats_inversion certifies only views of >= 16 rows, 8 .. 2040 columns; others take the exact path.  On
    frames whose two distances are exactly equal an in-gate view is counted as uncertified and an out-of-gate view is not."""
    from pylinac_b200 import _native as nat
    from pylinac_b200 import field_analysis as fa

    rng = np.random.default_rng(8)
    dpmm = 1 / 0.336
    report = {}
    for (h, w), gated in [((15, 64), False), ((16, 64), True), ((64, 7), False), ((64, 8), True), ((24, 2040), True), ((24, 2041), False)]:
        frames = np.stack([_rank_ramp(rng.integers(0, 65536, (h, w)), (5, 50, 95), (1000, 1100 + 50 * i, 1200 + 100 * i)) for i in range(2)])
        try:
            ctx.set_option(nat.OPT_STATS_EXACT, 1)
            exact = fa.analyze_batch(frames, dpmm).rows.copy()
            ctx.set_option(nat.OPT_STATS_EXACT, 0)
            u0 = ctx.counter(nat.CTR_STATS_UNCERTIFIED)
            fast = fa.analyze_batch(frames, dpmm).rows.copy()
            report[(h, w)] = ctx.counter(nat.CTR_STATS_UNCERTIFIED) - u0
        finally:
            ctx.set_option(nat.OPT_STATS_EXACT, 0)
        for i in range(2):
            assert int(fast["hist_inverted"][i]) == _np_inverted(frames[i], (5, 50, 95)), (h, w, i)
        for f in exact.dtype.names:
            np.testing.assert_array_equal(fast[f], exact[f], err_msg=f"{(h, w)}/{f}")
        assert report[(h, w)] == (2 if gated else 0), f"uncertified frames per shape: {report}"


def test_starshot_inversion_and_local_max_equal_numpy(ctx):
    """hist_inverted = |p50 - p4| > |p96 - p50| and local_max = np.percentile(grounded central third, 90) bit for bit, at
    1023 x 1023: the central third has 341 x 341 pixels, where the 90 % virtual index is an integer that other ways of
    computing it miss by one ulp."""
    import bench
    from pylinac_b200 import _native as nat
    from pylinac_b200 import starshot as ss

    rng = np.random.default_rng(9)
    n90 = 341 * 341
    p, nx = _plan(n90, 90)
    # central third: a shuffled ramp with a step of one grey level between the order statistics of the 90 % pair, counted from
    # either end (the plan of an inverted frame reads the mirrored ranks)
    ramp = 20000 + np.arange(n90) * 20000 // n90
    ramp[nx:] += 1
    ramp[n90 - 1 - p:] += 1
    cases = {}
    for i in range(2):
        s = bench._gen_module_frames(("star", i))[:1023, :1023].copy()
        s[341:682, 341:682] = rng.permutation(ramp).reshape(341, 341)
        cases[f"star{i}"] = s
        cases[f"star{i}_inverted"] = (65535 - s.astype(np.int64)).astype(np.uint16)
    s = cases["star0"]
    for delta in (0, 1, -1, 6000, -6000):
        cases[f"ramp_d{delta}"] = _rank_ramp(s, (4, 50, 96), (3000, 23000, 43000 + delta))
    g = cases["ramp_d-6000"].copy()
    g[_pilot_grid(*g.shape)] = 65535
    cases["ramp_d-6000_pilot"] = g
    names = list(cases)
    frames = np.stack([cases[k] for k in names])
    params = ss.make_params(2.56)
    unc = {}
    try:
        ctx.set_option(nat.OPT_STATS_EXACT, 1)
        exact = nat.starshot_analyze(ctx, frames, params).copy()
        ctx.set_option(nat.OPT_STATS_EXACT, 0)
        rows = []
        for k in names:
            u0 = ctx.counter(nat.CTR_STATS_UNCERTIFIED)
            rows.append(nat.starshot_analyze(ctx, cases[k][None], params).copy()[0])
            unc[k] = ctx.counter(nat.CTR_STATS_UNCERTIFIED) - u0
    finally:
        ctx.set_option(nat.OPT_STATS_EXACT, 0)
    for i, k in enumerate(names):
        a = cases[k]
        inv = _np_inverted(a, (4, 50, 96))
        assert int(rows[i]["hist_inverted"]) == inv, f"{k}: uncertified = {unc}"
        g = (-a + a.max() + a.min()) if inv else a
        central = (g - g.min())[341:682, 341:682]
        if k.startswith("star"):
            srt = np.sort(central.ravel())
            assert srt[p] != srt[nx], f"{k}: the order statistics around the 90 % rank must differ"
        assert float(rows[i]["local_max"]) == np.percentile(central, 90), (k, float(rows[i]["local_max"]), np.percentile(central, 90))
        for f in exact.dtype.names:
            np.testing.assert_array_equal(rows[i][f], exact[f][i], err_msg=f"{k}/{f}")
    assert unc["ramp_d0"] == 1 and unc["star0"] == 0, f"uncertified frames: {unc}"


# ------------------------------------------------------------------------------------------------ d. PicketFence front end
PF_CTRS = ("CTR_PF_FALLBACKS", "CTR_PF_REDONE_FRAMES", "CTR_PF_EXACT_FRAMES")


def _pf_case(ctx, frame, **kw):
    """One frame through the fast pipeline (with its counter deltas) and through the exact-histogram pipeline; every summary
    field and measurement row must agree."""
    from pylinac_b200 import _native as nat
    from pylinac_b200 import picketfence as pf

    c0 = [ctx.counter(getattr(nat, c)) for c in PF_CTRS]
    fast = pf.analyze_batch(frame[None], 2.56, **kw)
    delta = {c[len("CTR_PF_"):].lower(): ctx.counter(getattr(nat, c)) - v for c, v in zip(PF_CTRS, c0)}
    try:
        ctx.set_option(nat.OPT_PF_EXACT_ONLY, 1)
        exact = pf.analyze_batch(frame[None], 2.56, **kw)
    finally:
        ctx.set_option(nat.OPT_PF_EXACT_ONLY, 0)
    for k in exact.summary.dtype.names:
        np.testing.assert_array_equal(exact.summary[k], fast.summary[k], err_msg=f"{k}, counters {delta}")
    if int(exact.summary["status"][0]) == 0:
        m = int(exact.summary["n_meas"][0])
        for k in exact.meas.dtype.names:
            np.testing.assert_array_equal(exact.meas[k][0, :m], fast.meas[k][0, :m], err_msg=f"{k}, counters {delta}")
    return fast.summary[0], delta


def _pf_oracle_check(frame, s, delta, crop_mm=3):
    from oracle import pf_oracle

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o = pf_oracle.pf_analyze(frame, 2.56, crop_mm=crop_mm)
    assert int(s["noise_median_passes"]) == o["noise_median_passes"], (int(s["noise_median_passes"]), o["noise_median_passes"], delta)
    assert int(s["orientation"]) == int(o["orientation"]), delta
    assert bool(s["corner_inverted"]) == o["corner_inverted"], delta
    assert int(s["status"]) == 0, delta
    assert np.array_equal(np.sort(s["picket_idx"][:int(s["n_pickets"])]), np.sort(o["picket_idx"])), delta
    assert int(s["n_meas"]) == o["n_meas"], delta


def _top_pixel(view, k):
    """(row, col) of a pixel strictly above the order statistic at rank k"""
    s = np.sort(view.ravel())
    r, c = np.nonzero(view > s[k])
    assert r.size, "no pixel above the rank"
    return r[0], c[0]


@pytest.mark.parametrize("crop_mm", [3, 0])
def test_pf_noise_boundary_max_side(ctx, crop_mm):
    """max > 1.25 * p99.5 decided at its boundary: one pixel already above the p99.5 order statistics is raised to m0 - 1 (no
    noise) and to m0 (noise), m0 the smallest integer above 1.25 * p99.5.  The order statistics do not move."""
    from oracle import pf_oracle, synth

    base = synth.bench_pf_frame(3) // 2
    c = int(round(crop_mm * 2.56))
    view = base[c:base.shape[0] - c, c:base.shape[1] - c]
    n = view.size
    p995 = np.percentile(view, 99.5)
    m0 = int(np.floor(1.25 * p995)) + 1
    r, cc = _top_pixel(view, _plan(n, 99.5)[1])
    report = {}
    for name, v in (("base", None), ("m0-1", m0 - 1), ("m0", m0)):
        f = base.copy()
        if v is not None:
            f[r + c, cc + c] = v
        fv = f[c:f.shape[0] - c, c:f.shape[1] - c]
        assert np.percentile(fv, 99.5) == p995
        assert pf_oracle.has_noise(fv) == (name == "m0"), name
        s, delta = _pf_case(ctx, f, crop_mm=crop_mm)
        report[name] = delta
        _pf_oracle_check(f, s, report, crop_mm)
    assert report["base"]["redone_frames"] == 0, f"the natural frame must certify: {report}"
    assert report["m0"]["redone_frames"] == 1 and report["m0"]["exact_frames"] == 0, f"m0: noise certified by one exact count: {report}"
    assert report["m0-1"]["exact_frames"] == 1, f"m0 - 1 is too close to certify: {report}"


def test_pf_noise_boundary_min_side(ctx):
    """min < 0.75 * p0.5 and |min - p0.5| > 0.1 (p99.5 - p0.5) at its boundary, on a frame with an offset floor."""
    from oracle import pf_oracle, synth

    base = synth.bench_pf_frame(4) // 2 + 20000
    c = 8
    view = base[c:-c, c:-c]
    n = view.size
    p005, p995 = np.percentile(view, [0.5, 99.5])
    m1 = int(np.ceil(0.75 * p005)) - 1                  # largest integer below 0.75 * p0.5
    assert abs(m1 - p005) > 0.1 * (p995 - p005)
    # the floor value fills more than the lowest 0.5 %: lowering one such pixel leaves the order statistics in place
    assert np.count_nonzero(view == view.min()) > _plan(n, 0.5)[1] + 1
    r, cc = np.argwhere(view == view.min())[0]
    report = {}
    for name, v in (("base", None), ("m1+1", m1 + 1), ("m1", m1)):
        f = base.copy()
        if v is not None:
            f[r + c, cc + c] = v
        fv = f[c:-c, c:-c]
        assert np.percentile(fv, 0.5) == p005
        assert pf_oracle.has_noise(fv) == (name == "m1"), name
        s, delta = _pf_case(ctx, f)
        report[name] = delta
        _pf_oracle_check(f, s, report)
    assert report["base"]["redone_frames"] == 0, f"the natural frame must certify: {report}"
    # only the max side of _has_noise can be certified by a count (k_pf_count_above): a frame noisy on its min side takes the
    # exact pipeline
    assert report["m1"]["exact_frames"] == 1, f"counter deltas per frame: {report}"


def test_pf_lying_pilot(ctx):
    """Frames whose pilot rows (16 + 32 k of the cropped view) or pilot grid misrepresent the frame, and alternating-pixel
    patterns that loosen the 4-pixel-group count bounds: results must equal the exact pipeline and the oracle."""
    from oracle import synth

    base = synth.bench_pf_frame(5)
    c = 8
    H, W = base.shape[0] - 2 * c, base.shape[1] - 2 * c
    cases = {"base": base}
    for lie in (0, int(base.max())):
        f = base.copy()
        f[c + 16::32, :] = lie
        cases[f"pilot_rows_{lie}"] = f
    f = base.copy()
    rows = c + ((2 * np.arange(8) + 1) * H) // 16
    cols = c + (np.arange(256) * W) // 256
    f[np.ix_(rows, cols)] = int(base.max())
    cases["t0_grid"] = f
    chk = (np.indices(base.shape).sum(0) % 2).astype(bool)
    f = base.copy()
    f[chk] = base.max()
    cases["alternating_max"] = f
    f = base.copy().astype(np.int64)
    f[chk] = f[chk] // 4
    cases["alternating_quarter"] = f.astype(np.uint16)
    report = {}
    for name, f in cases.items():
        s, delta = _pf_case(ctx, f)
        report[name] = delta
        if name in ("base", "pilot_rows_0", "t0_grid"):
            _pf_oracle_check(f, s, report)
    fell_back = [k for k, d in report.items() if d["redone_frames"] > 0]
    assert report["base"]["redone_frames"] == 0 and fell_back, f"counter deltas per frame: {report}"


def test_pf_orientation_near_square(ctx):
    """A frame equal to its transpose has equal row and column percentile ranges.  In exact arithmetic "row range < column
    range" is false (UP_DOWN); numpy's float sums of the two axes round differently, so the oracle is not asked at the tie.
    +-1 grey levels on the pixels above the median of one triangle break the tie by ~1e-3, far above that rounding."""
    from oracle import pf_oracle, synth

    b = synth.bench_pf_frame(6).astype(np.int64)
    sym = ((b + b.T) // 2).astype(np.uint16)
    assert np.array_equal(sym, sym.T)
    tri = np.triu(np.ones(sym.shape, bool), 1) & (sym > np.median(sym))
    cases = {"transpose": sym}
    for d in (1, -1):
        cases[f"triangle{d:+d}"] = (sym.astype(np.int64) + d * tri).astype(np.uint16)
    report = {}
    for name, f in cases.items():
        s, delta = _pf_case(ctx, f, crop_mm=0)
        report[name] = (int(s["orientation"]), delta)
        if name == "transpose":
            assert int(s["orientation"]) == pf_oracle.UP_DOWN, report
        else:
            _pf_oracle_check(f, s, report, crop_mm=0)
    assert {o for o, _ in report.values()} == {pf_oracle.UP_DOWN, pf_oracle.LEFT_RIGHT}, report
    assert report["transpose"][1]["exact_frames"] == 1, f"the exact tie must fall back: {report}"
