"""CPU: the gamma_2d oracle against the reference's goldens, the disk of offsets against skimage's membership test, and the
argument errors of core.gamma.gamma_2d (raised before anything reaches a device)."""
import os

import numpy as np
import pytest

from oracle import gamma2d_oracle, skimage_draw
from pylinac_b200.core import gamma as G
from tests.golden.gamma2d_cases import CASES, ERROR_CASES, case_pair

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "gamma2d_golden.npz"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference_bit_for_bit(name):
    ref, ev, kw = case_pair(name)
    np.testing.assert_array_equal(gamma2d_oracle.gamma_2d(ref, ev, **kw), GOLDEN[name])


def test_boundary_point_of_the_dta40_disk_decides_a_pixel():
    """(5, 3) + (40, 9) is the only evaluation pixel within dose; only the floating-point disk reaches it."""
    g = GOLDEN["dta40_boundary_f64"]
    assert g[5, 3] == np.sqrt((40 / 40) ** 2 + (9 / 40) ** 2)
    ref, ev, kw = case_pair("dta40_boundary_f64")
    assert 40 ** 2 + 9 ** 2 == 41 ** 2 and ev[45, 12] == ref[5, 3]


@pytest.mark.parametrize("dta", range(0, 65))
def test_offset_table_is_skimage_disk(dta):
    offsets, dist2 = G._disk_offsets(dta)
    rr, cc = skimage_draw.disk((0, 0), dta + 1)
    assert sorted(map(tuple, offsets.tolist())) == sorted(zip(rr.tolist(), cc.tolist()))
    # sorted by distance, raster order among equal distances
    with np.errstate(divide="ignore", invalid="ignore"):
        expect = (rr / dta) ** 2 + (cc / dta) ** 2
    order = np.argsort(expect, kind="stable")
    np.testing.assert_array_equal(offsets, np.stack([rr[order], cc[order]], axis=1))
    np.testing.assert_array_equal(dist2, expect[order])
    integer = {(r, c) for r in range(-dta - 1, dta + 2) for c in range(-dta - 1, dta + 2) if r * r + c * c < (dta + 1) ** 2}
    extra = set(map(tuple, offsets.tolist())) - integer
    assert integer <= set(map(tuple, offsets.tolist()))
    if dta == 40:
        assert extra == {(sr * a, sc * b) for a, b in ((40, 9), (9, 40)) for sr in (-1, 1) for sc in (-1, 1)}
    else:
        assert not extra


@pytest.mark.parametrize("name", sorted(ERROR_CASES))
def test_argument_errors_are_the_reference_s(name):
    rshape, eshape, kw = ERROR_CASES[name]
    kind, msg = GOLDEN["error:" + name]
    with pytest.raises(Exception) as info:
        G.gamma_2d(np.ones(rshape), np.ones(eshape), **kw)
    assert type(info.value).__name__ == kind and str(info.value) == msg


def test_smaller_evaluation_is_rejected_up_front():
    with pytest.raises(ValueError, match="smaller than the reference"):
        G.gamma_2d(np.ones((6, 6)), np.ones((6, 5)))


def test_empty_frames_follow_the_reference():
    with pytest.raises(ValueError, match="zero-size array"):
        G.gamma_2d(np.ones((0, 3)), np.ones((0, 3)))
    with pytest.raises(ValueError, match="can't extend empty axis"):
        G.gamma_2d(np.ones((0, 3)), np.ones((0, 3)), global_dose=False)
    assert G.gamma_2d(np.ones((0, 3)), np.ones((0, 3)), distance_to_agreement=0, global_dose=False).shape == (0, 3)
