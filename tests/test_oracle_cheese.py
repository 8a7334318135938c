"""CPU: oracle/ct_oracle.py reproduces every slice's localization row of tests/golden/cheese_golden.npz (rows the generator checked
against the unmodified reference's Slice.phantom_roi), every case reaches the path it was built for, and oracle/skimage_ct.py's Scharr
sums match ndimage.convolve's order."""
import json

import numpy as np
import pytest
from scipy import ndimage

from oracle import ct_oracle, skimage_ct
from tests.golden.cheese_cases import CASES, case_series
from tests.golden.make_cheese_golden import ROW_KEYS, check_expectations

GOLDEN = np.load("tests/golden/cheese_golden.npz")
SIZE = {"TomoCheese": 150.0, "CIRS062M": 155.0}
CLEAR = {"TomoCheese": True, "CIRS062M": False}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_rows_match_golden(name):
    raw, slopes, intercepts, px, _ = case_series(name)
    ph = CASES[name]["phantom"]
    size = np.pi * SIZE[ph] ** 2 / px**2
    rows = np.array([[ct_oracle.localize_slice(raw[z], slopes[z], intercepts[z], size, CLEAR[ph]).get(k, np.nan) for k in ROW_KEYS]
                     for z in range(len(raw))], dtype=np.float64)
    np.testing.assert_array_equal(rows, GOLDEN[f"{name}/rows"])
    # the case reaches what it was built for: statuses, messages, exceptions, roll, and (metal) a threshold clipping changes
    check_expectations(name, rows, json.loads(str(GOLDEN[f"{name}/reference"])), raw, slopes, intercepts)


def test_scharr_restatement_is_the_footprint_order():
    """the device's explicit sum order (csrc/ct.cu scharr3) restated in numpy equals skimage_ct.scharr (ndimage.convolve)"""
    rng = np.random.default_rng(3)
    a = rng.normal(0, 300, (37, 53)).round(1)
    p = np.pad(a, 1, mode="symmetric")
    v = [p[j:j + a.shape[0], i:i + a.shape[1]] for j in range(3) for i in range(3)]
    s, c = 0.1875, 0.625
    a0 = 0.0 + v[0] * -s
    for k, w in ((1, -c), (2, -s), (6, s), (7, c), (8, s)):
        a0 = a0 + v[k] * w
    a1 = 0.0 + v[0] * -s
    for k, w in ((2, s), (3, -c), (5, c), (6, -s), (8, s)):
        a1 = a1 + v[k] * w
    mine = np.sqrt(0.0 + a0 * a0 + a1 * a1) / 1.4142135623730951
    assert np.array_equal(mine, skimage_ct.scharr(a))
    assert np.array_equal(skimage_ct.gaussian(a), ndimage.gaussian_filter(a, 1, mode="nearest", truncate=4.0))
