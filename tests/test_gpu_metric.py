"""GPU surface metrics (csrc/metrics.cu, wsl4mis_b200.metric) against medpy's algorithm restated on scipy (tests/_metric_oracle.py):
hd95 bit for bit and dc / jc identical at unit and integer spacings, hd95 / asd to 1e-12 otherwise; the per-volume form and the
validation pass that uses it."""
import zlib

import numpy as np
import pytest
import torch
from scipy.ndimage import binary_erosion

import _metric_oracle as M

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200 import metric, val_2D
    from wsl4mis_b200.dataloaders.dataset import fold_ids, synthetic_acdc
    from wsl4mis_b200.networks.unet import UNet

SHAPES = [(10, 256, 216), (1, 64, 48), (7, 33, 129), (21, 512, 428), (256, 216), (17, 40)]
SPACINGS = [None, 2.0, (10.0, 1.5625, 1.5625), (5.0, 1.37, 1.41)]


def _blobs(shape, rs, n=4):
    grids = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij")
    m = np.zeros(shape, bool)
    for _ in range(n):
        c = [rs.uniform(0, s) for s in shape]
        r = [max(1.0, rs.uniform(0.1, 0.35) * s) for s in shape]
        m |= sum(((g - ci) / ri) ** 2 for g, ci, ri in zip(grids, c, r)) < 1.0
    return m


def _mask(kind, shape, rs):
    if kind == "blobs":
        return _blobs(shape, rs)
    if kind == "faces":              # touches every face of the array
        m = ~_blobs(shape, rs, 2)
        for ax in range(len(shape)):
            sl = [slice(None)] * len(shape)
            for end in (0, -1):
                sl[ax] = end
                m[tuple(sl)] = True
        return m
    if kind == "voxel":
        m = np.zeros(shape, bool)
        m[tuple(rs.randint(0, s) for s in shape)] = True
        return m
    if kind == "full":
        return np.ones(shape, bool)
    if kind == "lines":              # one-voxel lines along every axis
        m = np.zeros(shape, bool)
        for ax in range(len(shape)):
            p = [rs.randint(0, s) for s in shape]
            p[ax] = slice(None)
            m[tuple(p)] = True
        return m
    if kind == "checker":            # every voxel is on the surface
        return (np.indices(shape).sum(0) % 2) == 0
    raise ValueError(kind)


PAIRS = [("blobs", "blobs"), ("faces", "blobs"), ("voxel", "blobs"), ("full", "blobs"), ("lines", "faces"), ("checker", "blobs")]


def _spacing(sp, ndim):
    return sp[-ndim:] if isinstance(sp, tuple) else sp


def _integer(sp):
    return sp is None or all(float(v).is_integer() for v in np.atleast_1d(sp))


@pytest.mark.parametrize("sp", SPACINGS, ids=["none", "2", "acdc", "aniso"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_kernel_matches_oracle(shape, sp):
    rs = np.random.RandomState(zlib.crc32(repr((shape, sp)).encode()))
    sp = _spacing(sp, len(shape))
    big = np.prod(shape) > 1e6
    pairs = [PAIRS[0], PAIRS[1], PAIRS[5]] if big else PAIRS
    for ka, kb in pairs:
        a, b = _mask(ka, shape, rs), _mask(kb, shape, rs)
        ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
        got_hd, got_asd = metric.hd95(ta, tb, voxelspacing=sp), metric.asd(a, b, voxelspacing=sp)
        want_hd, want_asd = M.hd95(a, b, sp), M.asd(a, b, sp)
        if _integer(sp):
            assert got_hd == want_hd, (ka, kb, got_hd, want_hd)
        else:
            assert got_hd == pytest.approx(want_hd, rel=1e-12, abs=0), (ka, kb)
        assert got_asd == pytest.approx(want_asd, rel=1e-12, abs=0), (ka, kb)
        assert metric.dc(ta, tb) == M.dc(a, b) and metric.jc(a, tb) == M.jc(a, b), (ka, kb)


def test_surface_metrics_on_synthetic_volumes_equals_binary_calls_and_oracle():
    cases = synthetic_acdc(30)
    _, val = fold_ids("fold1")
    sp = (10.0, 1.5625, 1.5625)
    for pid in [p for p in sorted(cases) if p in val][:4]:
        lab = cases[pid][1]
        pred = np.roll(lab, (0, 3, -2), axis=(0, 1, 2))
        pred[(pred == 3) & ~binary_erosion(pred == 3, iterations=2)] = 0
        for spacing in (None, sp):
            res = metric.surface_metrics(torch.from_numpy(pred).to(DEV), torch.from_numpy(lab).to(DEV), 4, spacing)
            for c in range(1, 4):
                r, p, g = res[c - 1], pred == c, lab == c
                assert (r.inter, r.pred, r.gt, r.union) == (np.count_nonzero(p & g), np.count_nonzero(p), np.count_nonzero(g),
                                                          np.count_nonzero(p | g))
                assert r.hd95 == metric.hd95(p, g, spacing) and r.asd == metric.asd(p, g, spacing)
                if spacing is None:
                    assert r.hd95 == M.hd95(p, g)
                else:
                    assert r.hd95 == pytest.approx(M.hd95(p, g, spacing), rel=1e-12, abs=0)
                assert r.asd == pytest.approx(M.asd(p, g, spacing), rel=1e-12, abs=0)


def test_empty_masks_connectivity_and_argument_checks():
    full, empty = np.ones((3, 8, 8), np.uint8), np.zeros((3, 8, 8), np.uint8)
    for fn in (metric.hd95, metric.asd):
        with pytest.raises(RuntimeError, match="The first supplied array does not contain any binary object."):
            fn(empty, full)
        with pytest.raises(RuntimeError, match="The second supplied array does not contain any binary object."):
            fn(full, empty)
        with pytest.raises(NotImplementedError):
            fn(full, full, connectivity=2)
        with pytest.raises(ValueError):
            fn(full, full[:, :7])
        with pytest.raises(RuntimeError, match="length"):
            fn(full, full, voxelspacing=(1.0, 2.0))
        for bad in (np.ones(8, np.uint8), np.ones((2, 2, 8, 8), np.uint8)):
            with pytest.raises(ValueError, match="rank"):
                fn(bad, bad)
    assert metric.dc(empty, empty) == 0.0
    assert metric.hd95(full * 7, full) == 0.0        # any nonzero value counts as True
    # the per-volume form flags empty classes instead of raising
    lab = np.zeros((3, 8, 8), np.uint8)
    lab[1, 2:5, 2:5] = 1
    res = metric.surface_metrics(torch.from_numpy(lab).to(DEV), torch.from_numpy(lab * 2).to(DEV), 3)
    assert (res[0].pred, res[0].gt, res[1].pred, res[1].gt) == (9, 0, 0, 9)
    assert all(np.isnan(r.hd95) and np.isnan(r.asd) for r in res)
    with pytest.raises(RuntimeError, match="classes"):
        metric.surface_metrics(torch.from_numpy(lab).to(DEV), torch.from_numpy(lab).to(DEV), 17)


def test_nonzero_values_count_as_true():
    """medpy binarises with astype(bool): 0.5 and 256 are True, not truncated or wrapped to 0 by a uint8 cast."""
    rs = np.random.RandomState(7)
    shape = (6, 40, 36)
    a = _mask("blobs", shape, rs)
    b = _mask("blobs", shape, rs)
    fa = np.where(a, 0.5, 0.0)                          # float probabilities below 1
    ib = np.where(b, 256, 0).astype(np.int64)           # a multiple of 256
    want = (M.dc(a, b), M.jc(a, b), M.hd95(a, b, 2.0), M.asd(a, b, 2.0))
    for ra, rb in ((fa, ib), (torch.from_numpy(fa), torch.from_numpy(ib).to(DEV)), (torch.from_numpy(fa).to(DEV), ib)):
        got = (metric.dc(ra, rb), metric.jc(ra, rb), metric.hd95(ra, rb, 2.0), metric.asd(ra, rb, 2.0))
        assert got[:3] == want[:3] and got[3] == pytest.approx(want[3], rel=1e-12, abs=0)


def test_sixteen_classes_fill_both_halves_of_the_surface_byte():
    """classes = 16: class 15 is the largest value the packed pred / gt surface nibbles hold."""
    rs = np.random.RandomState(11)
    shape = (9, 96, 80)
    pred = np.zeros(shape, np.uint8)
    gt = np.zeros(shape, np.uint8)
    for c in range(1, 16):
        pred[_blobs(shape, rs, 2)] = c
        gt[_blobs(shape, rs, 2)] = c
    sp = (4.0, 1.0, 2.0)
    res = metric.surface_metrics(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), 16, sp)
    assert len(res) == 15
    for c in range(1, 16):
        p, g = pred == c, gt == c
        r = res[c - 1]
        assert (r.inter, r.pred, r.gt) == (np.count_nonzero(p & g), np.count_nonzero(p), np.count_nonzero(g)), c
        if p.any() and g.any():
            assert r.hd95 == M.hd95(p, g, sp), c
            assert r.asd == pytest.approx(M.asd(p, g, sp), rel=1e-12, abs=0), c
        else:
            assert np.isnan(r.hd95), c
    assert sum(1 for c in range(1, 16) if (pred == c).any() and (gt == c).any()) >= 12


def test_two_calls_are_bit_identical():
    rs = np.random.RandomState(5)
    shape = (10, 256, 216)
    lab_a = (_mask("blobs", shape, rs) * 1 + _mask("blobs", shape, rs) * 2).astype(np.uint8)
    lab_b = (_mask("blobs", shape, rs) * 1 + _mask("faces", shape, rs) * 2).astype(np.uint8)
    ta, tb = torch.from_numpy(lab_a).to(DEV), torch.from_numpy(lab_b).to(DEV)
    r1 = metric.surface_metrics(ta, tb, 3, (10.0, 1.37, 1.41))
    r2 = metric.surface_metrics(ta, tb, 3, (10.0, 1.37, 1.41))
    assert np.array_equal(np.array(r1, np.float64), np.array(r2, np.float64), equal_nan=True)
    assert all(not np.isnan(r.hd95) for r in r1)


def test_single_volume_scores_its_prediction_like_the_host_metric(monkeypatch):
    torch.manual_seed(0)
    net = UNet(1, 4).to(DEV).set_precision("fp32")
    cases = synthetic_acdc(30)
    _, val = fold_ids("fold1")
    vols = [cases[p] for p in sorted(cases) if p in val][:3]
    vols.append((vols[0][0][2, :144, :160], vols[0][1][2, :144, :160], None))   # a 2-D slice (fed unresized): a [1,h,w] volume
    for img, lab, _ in vols:
        got = val_2D.test_single_volume(torch.from_numpy(img)[None], torch.from_numpy(lab)[None], net, 4)
        image = img[None] if img.ndim == 2 else img
        pred = val_2D._predict_volume(image, net, image.shape[1:] if img.ndim == 2 else [256, 256], 0).cpu().numpy()
        label = lab[None] if lab.ndim == 2 else lab
        want = [val_2D.calculate_metric_percase(pred == i, label == i) for i in range(1, 4)]
        assert got == want
    # the host distance transform is off the validation path
    def boom(*a, **k):
        raise AssertionError("host hd95 called")
    monkeypatch.setattr(val_2D, "hd95", boom)
    img, lab, _ = vols[0]
    assert len(val_2D.test_single_volume(torch.from_numpy(img)[None], torch.from_numpy(lab)[None], net, 4)) == 3
