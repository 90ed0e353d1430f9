"""The CPU restatement of the random-walker pseudo labels (oracle/rw_oracle.py) against closed forms and the semantics of
dataloaders/acdc_pseudo_label_random_walker.py:9-26: seeds fixed, probabilities a partition of unity, the 1-D harmonic solution,
the missing-class rule, the F17 renumbering and the rescale clipping."""
import numpy as np
import pytest

import rw_oracle as R


def _slice(seed=0, h=40, w=48):
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    rr = np.sqrt((yy - h / 2) ** 2 + (xx - w / 2) ** 2)
    lab = np.zeros((h, w), np.uint8)
    lab[rr < 16] = 1
    lab[rr < 11] = 2
    lab[rr < 6] = 3
    img = np.clip(0.15 + 0.2 * lab + 0.05 * rs.randn(h, w), 0, 1).astype(np.float32)
    scr = np.full((h, w), 4, np.uint8)
    keep = rs.rand(h, w) < 0.05
    scr[keep] = lab[keep]
    return img, lab, scr


def test_seeds_keep_their_class_and_probabilities_partition_unity():
    img, lab, scr = _slice()
    out, prob = R.random_walker(img, scr)
    seeds = scr < 4
    assert np.array_equal(out[seeds], scr[seeds])
    assert prob.min() >= -1e-12 and prob.max() <= 1 + 1e-12
    assert np.allclose(prob.sum(-1), 1.0, atol=1e-10)
    assert np.array_equal(out, np.argmax(prob, -1))
    assert (out == lab).mean() > 0.9           # well-separated intensities: the walker recovers the structure


def test_chain_matches_cumulative_resistance():
    n = 30
    d01 = np.sort(np.random.RandomState(1).rand(n))
    img = np.tile(d01, (3, 1)).astype(np.float64)          # three identical rows: vertical edges carry no current
    scr = np.full((3, n), 4, np.uint8)
    scr[:, 0], scr[:, -1] = 0, 1
    m, K = np.where(scr < 4, scr.astype(np.int64) + 1, 0), 2     # two seed classes only: the solver core, without the class check
    d = R.rescale(img)
    L = R.laplacian(*R.edge_weights(d))
    mf = m.ravel()
    U, M = np.flatnonzero(mf == 0), np.flatnonzero(mf > 0)
    onehot = np.eye(K)[mf[M] - 1]
    from scipy.sparse.linalg import spsolve
    x = np.zeros((3 * n, K))
    x[U] = np.asarray(spsolve(L[U][:, U].tocsc(), -(L[U][:, M] @ onehot))).reshape(len(U), K)
    x[M] = onehot
    p1 = x[:, 1].reshape(3, n)[1]
    # std over the whole slice equals the std of one row (rows are identical)
    want = R.chain(n, d=d[1])
    np.testing.assert_allclose(p1, want, atol=1e-9)


def test_missing_class_gives_zeros():
    img, lab, scr = _slice(2)
    for c in (1, 2, 3):
        s = scr.copy()
        s[s == c] = 4
        out, prob = R.random_walker(img, s)
        assert not out.any() and not prob.any()


def test_missing_background_renumbers_f17():
    img, lab, scr = _slice(3)
    s = scr.copy()
    s[s == 0] = 4
    m, K = R.markers(s)
    assert K == 3 and set(np.unique(m)) == {0, 1, 2, 3}
    out, prob = R.random_walker(img, s)
    seeds = s < 4
    assert np.array_equal(out[seeds], s[seeds] - 1)          # classes 1..3 come out as 0..2
    assert out.max() <= 2 and not prob[..., 3].any()
    np.testing.assert_allclose(prob[..., :3].sum(-1), 1.0, atol=1e-10)


def test_rescale_clips_to_the_input_range():
    v = np.array([-1.0, -0.35, 0.0, 0.5, 1.0, 1.35, 2.0])
    np.testing.assert_allclose(R.rescale(v), [-1.0, -1.0, 0.35 / 1.7 * 2 - 1, 0.0, 1.35 / 1.7 * 2 - 1, 1.0, 1.0], atol=1e-15)


def test_weights_follow_the_population_std():
    d = R.rescale(_slice(4)[0])
    wr, wd = R.edge_weights(d, beta=100.0)
    s = -100.0 / (10.0 * np.sqrt(((d - d.mean()) ** 2).mean()))
    np.testing.assert_allclose(wr[3, 5], np.exp(s * (d[3, 6] - d[3, 5]) ** 2) + 1e-10, rtol=1e-14)
    np.testing.assert_allclose(wd[7, 2], np.exp(s * (d[8, 2] - d[7, 2]) ** 2) + 1e-10, rtol=1e-14)
    assert wr.min() >= 1e-10


@pytest.mark.parametrize("n_classes_missing", [0, 1])
def test_ce_dice_loss_matches_a_direct_restatement(n_classes_missing):
    import torch
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    label = torch.randint(0, 4, (2, 8, 8), generator=g).to(torch.uint8)
    if n_classes_missing:
        label[label == 3] = 4                                    # ignored by CE, in no class for Dice
    got = R.ce_dice_loss(logits, label)
    ce = torch.nn.functional.cross_entropy(logits, label.long(), ignore_index=4)
    p = torch.softmax(logits, 1)
    dice = 0
    for i in range(4):
        t = (label == i).double()
        dice = dice + 1 - (2 * (p[:, i] * t).sum() + 1e-5) / ((p[:, i] ** 2).sum() + (t * t).sum() + 1e-5)
    assert torch.allclose(got, 0.5 * (ce + dice / 4), rtol=1e-12)
