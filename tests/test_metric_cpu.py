"""The scipy restatement of medpy's surface metrics (tests/_metric_oracle.py, the reference of the GPU metric tests) against
closed forms, and against val_2D.hd95 at unit spacing; the percentile's last step of wsl4mis_b200.metric against np.percentile."""
import numpy as np
import pytest

import _metric_oracle as M


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("k", [1, 3])
def test_shifted_boxes_give_the_shift_times_the_spacing(axis, k):
    sp = (10.0, 1.5, 1.5)
    a = np.zeros((12, 30, 30), bool)
    a[3:8, 8:20, 6:18] = True
    b = np.roll(a, k, axis=axis)
    assert M.hd95(a, b, sp) == k * sp[axis]
    assert M.hd95(a, b, 2.0) == k * 2.0


def test_single_voxel_against_a_box():
    a = np.zeros((9, 20, 20), bool)
    a[4, 10, 10] = True
    b = np.zeros_like(a)
    b[2:7, 5:16, 5:16] = True
    # nearest surface of the box: 2 slices away at 10 per slice, or 5 pixels at 1.5
    assert M.asd(a, b, (10.0, 1.5, 1.5)) == 7.5
    assert M.asd(a, b, (1.0, 3.0, 3.0)) == 2.0
    # box surface -> the single voxel: the farthest corners dominate the 95th percentile
    d = M.surface_distances(b, a, (1.0, 1.0, 1.0))
    assert d.max() == np.sqrt(2 * 2 + 5 * 5 + 5 * 5)
    assert M.dc(a, b) == 2.0 / (1 + 5 * 11 * 11) and M.jc(a, b) == 1.0 / (5 * 11 * 11)


def test_rank2_slice_and_single_slice_volume_have_different_surfaces():
    sq = np.zeros((6, 6), bool)
    sq[1:5, 1:5] = True
    assert np.count_nonzero(M.surface(sq)) == 12
    assert np.count_nonzero(M.surface(sq[None])) == 16


def test_empty_masks_and_spacing_length():
    a = np.zeros((4, 4), bool)
    b = np.ones((4, 4), bool)
    with pytest.raises(RuntimeError, match="first"):
        M.hd95(a, b)
    with pytest.raises(RuntimeError, match="second"):
        M.asd(b, a)
    with pytest.raises(RuntimeError, match="length"):
        M.hd95(b, b, (1.0, 2.0, 3.0))
    assert M.dc(a, a) == 0.0


def test_oracle_equals_val_2d_hd95_at_unit_spacing():
    from wsl4mis_b200 import val_2D
    rs = np.random.RandomState(0)
    for shape in [(5, 40, 30), (1, 33, 17), (28, 19)]:
        a = rs.rand(*shape) > 0.6
        b = rs.rand(*shape) > 0.5
        assert M.hd95(a, b) == val_2D.hd95(a, b)
        assert M.hd95(a, b, 1.0) == val_2D.hd95(a, b)


def test_percentile_from_order_statistics_matches_numpy():
    from wsl4mis_b200.metric import _percentile95
    rs = np.random.RandomState(1)
    for n in list(range(1, 70)) + [641, 1000, 20 * 997 + 1, 654321]:
        x = np.round(rs.rand(n) * 50, 1) if n % 2 else rs.rand(n) * 37.0
        s = np.sort(x)
        vi = (n - 1) * 0.95
        lo = min(int(np.floor(vi)), n - 1)
        hi = min(lo + 1, n - 1)
        assert _percentile95(float(s[lo]), float(s[hi]), n) == np.percentile(x, 95), n
