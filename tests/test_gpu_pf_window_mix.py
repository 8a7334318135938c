"""Batches that mix benchmark frames (two-kernel window path) with frames whose windows that path does not cover: a Left-Right
frame and ~100-sample windows (k_pf_windows_fast), ~280-sample windows (left by k_pf_windows_fast to the generic kernel).  The
window kernels run one resident wave deep and skip the frames another kernel owns, so every frame of the batch must come out
exactly as it does when it is analysed alone."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _assert_same(batch, single, i):
    for k in batch.summary.dtype.names:
        np.testing.assert_array_equal(batch.summary[k][i], single.summary[k][0], err_msg=f"frame {i}: {k}")
    m = int(single.summary["n_meas"][0])
    for k in batch.meas.dtype.names:
        np.testing.assert_array_equal(batch.meas[k][i, :m], single.meas[k][0, :m], err_msg=f"frame {i}: {k}")


def test_mixed_window_paths_equal_one_frame_per_call():
    from oracle import synth
    from pylinac_b200 import picketfence as pf

    fr = synth.epid1024()
    bench = [synth.bench_pf_frame(i) for i in range(300, 305)]
    left_right = np.ascontiguousarray(synth.bench_pf_frame(305).T)
    wide = synth.picketfence_frame(fr, pickets=5, picket_spacing_mm=40, picket_width_mm=3, seed=306)
    widest = synth.picketfence_frame(fr, pickets=3, picket_spacing_mm=110, picket_width_mm=3, seed=307)
    frames = np.stack([bench[0], left_right, bench[1], wide, bench[2], bench[3], widest, bench[4]])
    batch = pf.analyze_batch(frames, 2.56)
    assert [int(s) for s in batch.summary["status"]] == [0] * len(frames), batch.summary["status"]
    for i in range(len(frames)):
        _assert_same(batch, pf.analyze_batch(frames[i:i + 1], 2.56), i)
