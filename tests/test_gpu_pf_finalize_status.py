"""GPU: the last PicketFence stage on the benchmark frames -- the median of |errors| against numpy on the table it wrote (one and
two positions per measurement), and a table larger than the caller's capacity reported as EPID_PF_CAPACITY."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("separate", [False, True])
def test_abs_median_error_is_numpy_median_of_the_table(separate):
    from oracle import synth
    from pylinac_b200 import picketfence as pf

    frames = np.stack([synth.bench_pf_frame(i) for i in range(40, 48)])
    kw = {"separate_leaves": True, "nominal_gap_mm": 3} if separate else {}
    res = pf.analyze_batch(frames, 2.56, **kw)
    npos = 2 if separate else 1
    for i in range(len(frames)):
        assert int(res.summary["status"][i]) == 0
        m = int(res.summary["n_meas"][i])
        err = np.abs(res.meas["error"][i, :m, :npos])
        assert float(res.summary["abs_median_error_mm"][i]) == float(np.median(err))


def test_table_over_capacity_is_reported():
    from oracle import synth
    from pylinac_b200 import picketfence as pf

    a = synth.bench_pf_frame(1)[None]
    assert int(pf.analyze_batch(a, 2.56, meas_cap=100).summary["status"][0]) == 5      # EPID_PF_CAPACITY
    full = pf.analyze_batch(a, 2.56)
    assert int(full.summary["status"][0]) == 0 and int(full.summary["n_meas"][0]) > 100
