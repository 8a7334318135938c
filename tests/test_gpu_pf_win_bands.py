"""Window bands of k_pf_win_medians at the edges of its geometry: rows that wrap under sag_adjustment, frames re-run from the
filtered-frame pool, and four-picket bands wider than 256 pixels.  Each batch must reproduce the per-window kernel (OPT_PF_WIN2=0)
bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _compare(frames, dpmm, **kw):
    from pylinac_b200 import _native as nat
    from pylinac_b200 import picketfence as pf

    ctx = nat.Context.default()
    try:
        ctx.set_option(nat.OPT_PF_WIN2, 0)
        old = pf.analyze_batch(frames, dpmm, **kw)
        ctx.set_option(nat.OPT_PF_WIN2, 1)
        redone0 = ctx.counter(nat.CTR_PF_REDONE_FRAMES)
        new = pf.analyze_batch(frames, dpmm, **kw)
        redone = ctx.counter(nat.CTR_PF_REDONE_FRAMES) - redone0
    finally:
        ctx.set_option(nat.OPT_PF_WIN2, 1)
    for k in old.summary.dtype.names:
        np.testing.assert_array_equal(old.summary[k], new.summary[k], err_msg=k)
    n_ok = 0
    for i in range(len(frames)):
        if int(old.summary["status"][i]) == 0:
            n_ok += 1
            m = int(old.summary["n_meas"][i])
            assert m > 0
            for k in old.meas.dtype.names:
                np.testing.assert_array_equal(old.meas[k][i, :m], new.meas[k][i, :m], err_msg=k)
    assert n_ok == len(frames), old.summary["status"]
    return redone


@pytest.mark.parametrize("sag_mm", [9.0, -9.0])
def test_sag_wraps_the_outermost_bands(sag_mm):
    """The outermost in-view bench bands start 17 rows below the top of the cropped view and end 18 rows above its bottom, so a
    23-pixel sag makes one of them wrap around the view (np.roll) while the other bands stay contiguous."""
    from oracle import synth

    frames = np.stack([synth.bench_pf_frame(i) for i in range(200, 204)])
    _compare(frames, 2.56, sag_adjustment=sag_mm)


def test_hot_pixel_frames_rerun_from_the_filtered_pool():
    """Hot-pixel frames are median filtered into a pool and re-run by the fast pipeline: their bands are read from the pool
    (row pitch rounded up to 8 pixels), those of the other frames from the batch."""
    from oracle import synth

    frames = np.stack([synth.bench_pf_frame(i) for i in range(210, 226)])
    rng = np.random.default_rng(3)
    for i in (2, 7, 11):
        f = frames[i] // 2
        f.ravel()[rng.integers(0, f.size, 40)] = 65535
        frames[i] = f
    assert _compare(frames, 2.56) >= 3


def test_four_picket_bands_wider_than_256_pixels():
    """HD MLC leaves of 2.5 mm are 6-7 rows at 2.56 px/mm, so four 64-sample windows share a slot; with pickets 64 pixels apart
    their band is 32-33 vectors of 8 pixels."""
    from oracle import synth
    from pylinac_b200 import picketfence as pf

    frames = []
    for i in range(3):
        fr = synth.Frame((1024, 1024), 0.390625, 1000.0)
        err = np.random.default_rng(500 + i).uniform(-0.3, 0.3, size=8)
        frames.append(synth.picketfence_frame(fr, pickets=8, picket_spacing_mm=25, picket_width_mm=3, picket_height_mm=300,
                                              picket_offset_error=err, blur_mm=1.0, noise_sigma=0.002, seed=500 + i))
    _compare(np.stack(frames), 2.56, mlc=pf.MLC.HD_MILLENNIUM, picket_spacing=64.0)
