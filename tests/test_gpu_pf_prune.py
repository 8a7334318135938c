"""GPU: PicketFence in CUDA on frames whose leaf rows are pruned by the median kiss count (picketfence.py:810-828), on a .5 and a
9 median that leave a picket or every row without measurements, and on 1, 2 and 32 pickets -- against the golden vectors of the
unmodified reference (tests/golden/pf_prune_golden.npz), raised exception types included.

These frames reach the parts of k_pf_finalize that the benchmark-like frames never do: keep flags and row offsets of a table with
holes, fits and widths over a subset of rows, the removed-row count, kiss counts of 32 (the last histogram bin and picket bit 31),
and the automatic re-run with a larger table (1600 measurements)."""
import warnings

import numpy as np
import pytest

from tests.golden.pf_prune_cases import CASES, case_frame
from tests.test_gpu_pf import _compare_with_golden

pytestmark = pytest.mark.gpu

GOLD = np.load("tests/golden/pf_prune_golden.npz")
RAISING = [n for n in CASES if f"{n}/raises" in GOLD]
ANALYSED = [n for n in CASES if n not in RAISING]
# Up-Down frames with pruned rows (or a pruning that leaves a fit without points): the two-kernel window path covers them
PRUNED_UP_DOWN = ["rows_removed", "rows_removed_offset", "rows_removed_ht03", "rows_removed_separate", "rows_removed_hdmlc",
                  "median_half", "median_nine"]


def _args(name):
    from pylinac_b200 import picketfence as pf

    a, ps, sid, ck, ak = case_frame(name)
    ck = dict(ck)
    if ck.get("mlc") == "HD":
        ck["mlc"] = pf.MLC.HD_MILLENNIUM
    return a, (1 / ps) * sid / 1000.0, {**ck, **ak}


def _assert_rows_equal(sa, ma, sb, mb, what):
    assert sa.tobytes() == sb.tobytes(), (what, [k for k in sa.dtype.names if np.asarray(sa[k]).tobytes() != np.asarray(sb[k]).tobytes()])
    if int(sa["status"]) == 0:
        m = int(sa["n_meas"])
        assert ma[:m].tobytes() == mb[:m].tobytes(), what


@pytest.mark.parametrize("name", CASES)
def test_pf_prune_case_matches_reference_golden(name):
    from pylinac_b200 import picketfence as pf

    a, dpmm, kw = _args(name)
    r = pf.analyze_batch(a[None], dpmm, **kw)[0]
    _compare_with_golden(r, name, GOLD)


@pytest.mark.parametrize("name", ANALYSED)
def test_pf_leaf_rows_removed_equals_the_oracle(name):
    from oracle import pf_oracle
    from pylinac_b200 import picketfence as pf

    a, dpmm, kw = _args(name)
    r = pf.analyze_batch(a[None], dpmm, **kw)[0]
    okw = dict(kw)
    if "mlc" in okw:
        okw["mlc"] = "HD Millennium"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o = pf_oracle.pf_analyze(a, dpmm, **okw)
    assert r.status == 0
    assert int(r.s["n_leaves_removed"]) == o["n_leaves_removed"]


def _kw_groups():
    groups = {}
    for name in CASES:
        a, dpmm, kw = _args(name)
        groups.setdefault(repr(sorted(kw.items())), (dpmm, kw, []))[2].append((name, a))
    return list(groups.values())


@pytest.mark.parametrize("group", range(len(_kw_groups())))
def test_pf_prune_cases_in_a_batch_equal_their_one_frame_calls(group):
    """The cases between benchmark frames in one batch (one batch per set of analyze() arguments): every row of the summary and of
    the table is byte-identical to the one-frame call, so no shared-memory state of k_pf_finalize carries from frame to frame."""
    from oracle import synth
    from pylinac_b200 import picketfence as pf

    dpmm, kw, named = _kw_groups()[group]
    frames, names = [], []
    for k, (name, a) in enumerate(named):
        frames += [synth.bench_pf_frame(500 + k), a]
        names += [f"bench{500 + k}", name]
    frames.append(synth.bench_pf_frame(499))
    names.append("bench499")
    res = pf.analyze_batch(np.stack(frames), dpmm, **kw)
    for i, a in enumerate(frames):
        one = pf.analyze_batch(a[None], dpmm, **kw)
        _assert_rows_equal(res.summary[i], res.meas[i], one.summary[0], one.meas[0], names[i])


@pytest.mark.parametrize("name", PRUNED_UP_DOWN)
def test_pf_pruned_frames_equal_on_the_per_window_kernel(name):
    """The pruned Up-Down frames give byte-identical results with the two-kernel window path switched off."""
    from pylinac_b200 import _native as nat
    from pylinac_b200 import picketfence as pf

    a, dpmm, kw = _args(name)
    ctx = nat.Context.default()
    try:
        ctx.set_option(nat.OPT_PF_WIN2, 0)
        old = pf.analyze_batch(a[None], dpmm, **kw)
        ctx.set_option(nat.OPT_PF_WIN2, 1)
        new = pf.analyze_batch(a[None], dpmm, **kw)
    finally:
        ctx.set_option(nat.OPT_PF_WIN2, 1)
    _assert_rows_equal(old.summary[0], old.meas[0], new.summary[0], new.meas[0], name)
