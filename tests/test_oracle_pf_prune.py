"""CPU: the oracle restatement (oracle/pf_oracle.py) against the golden vectors that the UNMODIFIED reference produced on frames
whose leaf rows are pruned by the median kiss count, and on 1, 2 and 32 pickets (tests/golden/pf_prune_golden.npz, made by
tests/golden/make_pf_prune_golden.py).  Where the reference raises, the oracle raises the same exception type with the same
message."""
import builtins
import hashlib
import warnings

import numpy as np
import pytest

from oracle import pf_oracle
from tests.golden.pf_prune_cases import CASES, case_frame
from tests.test_oracle_pf import CLOSE, EXACT

GOLD = np.load("tests/golden/pf_prune_golden.npz")


def run_oracle(name):
    a, ps, sid, ck, ak = case_frame(name)
    ck = dict(ck)
    if ck.get("mlc") == "HD":
        ck["mlc"] = "HD Millennium"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return pf_oracle.pf_analyze(a, (1 / ps) * sid / 1000.0, **ck, **ak)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_prune_golden(name):
    a, _, _, _, _ = case_frame(name)
    sha = np.frombuffer(hashlib.sha1(a.tobytes()).digest(), dtype=np.uint8)
    assert np.array_equal(sha, GOLD[f"{name}/input_sha1"]), "synthetic input drifted from the one the golden was made with"
    if f"{name}/raises" in GOLD:
        exc = getattr(builtins, str(GOLD[f"{name}/raises_type"]))
        with pytest.raises(exc) as ei:
            run_oracle(name)
        assert type(ei.value) is exc
        assert str(ei.value) == str(GOLD[f"{name}/raises"])
        return
    o = run_oracle(name)
    for k in EXACT:
        assert np.array_equal(np.asarray(o[k]), GOLD[f"{name}/{k}"]), k
    for k in CLOSE:
        np.testing.assert_array_equal(np.asarray(o[k]), GOLD[f"{name}/{k}"], err_msg=k)
    assert str(o["max_error_leaf"]) == str(GOLD[f"{name}/max_error_leaf"])
    assert [str(x) for x in o["failed_leaves"]] == [str(x) for x in GOLD[f"{name}/failed_leaves"]]
    # the cases do what their names say: rows are dropped only where one picket is short
    assert (o["n_leaves_removed"] > 0) == name.startswith("rows_removed"), o["n_leaves_removed"]


def test_golden_raises_where_the_cases_say():
    raising = {n: str(GOLD[f"{n}/raises_type"]) for n in CASES if f"{n}/raises" in GOLD}
    assert raising == {"median_half": "TypeError", "median_nine": "TypeError", "picket1": "ValueError"}


def test_oracle_counts_the_removed_rows():
    """Picket 0 spans 150 of the 300 mm: the 20 in-view rows beyond it kiss 9 pickets, the 30 others 10, and the median is 10."""
    o = run_oracle("rows_removed")
    assert (o["n_meas"], o["n_leaves_removed"]) == (300, 20)
