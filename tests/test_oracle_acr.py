"""CPU: oracle/acr_oracle.py reproduces every golden localization row and region row of tests/golden/acr_golden.npz, and each case
reaches the path acr_cases.py states for it."""
import json

import numpy as np
import pytest

from oracle import acr_oracle
from tests.golden.acr_cases import CASES, EXPECT, case_series
from tests.golden.make_acr_golden import ROW_KEYS, check_expectations

GOLDEN = np.load("tests/golden/acr_golden.npz")


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_golden(name):
    raw, slopes, intercepts, px, thk = case_series(name)
    size = np.pi * 100.0**2 / px**2
    rows = np.array([[acr_oracle.localize_slice(raw[z], slopes[z], intercepts[z], size, False, 110 / px).get(k, np.nan)
                      for k in ROW_KEYS] for z in range(len(raw))], dtype=np.float64)
    np.testing.assert_array_equal(rows, GOLDEN[f"{name}/rows"])
    res = json.loads(str(GOLDEN[f"{name}/reference"]))
    check_expectations(name, rows, res, raw.shape[1], px)
    if f"{name}/regions" in GOLDEN.files:
        z = res[0]["origin_slice"]
        regions, thres, max_edge, _ = acr_oracle.slice_regions(raw[z], slopes[z], intercepts[z], 110 / px)
        assert json.loads(json.dumps(acr_oracle.region_rows(regions, raw.shape[2]))) == json.loads(str(GOLDEN[f"{name}/regions"]))
        assert [thres, max_edge] == GOLDEN[f"{name}/region_threshold"].tolist()
        assert [r.eccentricity for r in regions] == GOLDEN[f"{name}/eccentricity"].tolist()


def test_every_case_states_its_path():
    assert set(EXPECT) == set(CASES)


def test_disk_clips_to_the_shape():
    """the clipped disk is the unclipped one minus the pixels outside the image (a half-integer or integer centre)"""
    for h, w, rad in ((20, 31, 25.0), (64, 64, 40.5), (33, 12, 7.0)):
        rr, cc = acr_oracle.disk((h / 2 - 0.5, w / 2 - 0.5), rad, shape=(h, w))
        r0, c0 = acr_oracle.disk((h / 2 - 0.5, w / 2 - 0.5), rad)
        keep = (r0 >= 0) & (r0 < h) & (c0 >= 0) & (c0 < w)
        assert np.array_equal(rr, r0[keep]) and np.array_equal(cc, c0[keep])
