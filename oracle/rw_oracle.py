"""CPU restatement of the random-walker pseudo labels of dataloaders/acdc_pseudo_label_random_walker.py:9-26
(pseudo_label_generator_acdc) and of skimage.segmentation.random_walker(data, markers, beta=100, mode='bf') as it is called
there, solved exactly (scipy.sparse + spsolve, fp64).  Test infrastructure: nothing under wsl4mis_b200/ imports it.

Steps (DESIGN §2 F17 records the unverified reading of skimage's renumbering):
  1. any of classes 1, 2, 3 absent from the scribble -> all-zero pseudo label;
  2. markers: scribble 4 -> 0 (unknown), scribble c in 0..3 -> c + 1;
  3. d = rescale_intensity(image, in_range=(-0.35, 1.35), out_range=(-1, 1));
  4. 4-neighbour edge weights w_ij = exp(-beta / (10 * std(d)) * (d_i - d_j)^2) + 1e-10 (population std over the slice);
  5. L_UU x_l = -L_UM m_l per label column; label = argmax_l x_l + 1, seeds keep their marker; pseudo = label - 1;
  6. F17: marker values are renumbered by rank when they are not consecutive (no background scribble), and the output stays
     renumbered, so every class shifts down by one.

Also ``ce_dice_step``: the step body of train_fully_supervised_2D.py / train_weakly_supervised_pCE_random_walker_2D.py:97-105,
0.5 * (CrossEntropyLoss(ignore_index=4) + DiceLoss(4)(softmax, label)), on the oracle's U-Net forward."""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.linalg import spsolve

BETA = 100.0
EPS = 1e-10


def rescale(image):
    """rescale_intensity(image, in_range=(-0.35, 1.35), out_range=(-1, 1)) in fp64 (acdc_pseudo_label_random_walker.py:22-23)"""
    d = np.clip(np.asarray(image, np.float64), -0.35, 1.35)
    return (d + 0.35) / 1.7 * 2.0 - 1.0


def edge_weights(d, beta=BETA):
    """-> (w_right [h, w-1], w_down [h-1, w]) of the 4-neighbour grid"""
    scale = -beta / (10.0 * d.std())
    wr = np.exp(scale * (d[:, 1:] - d[:, :-1]) ** 2) + EPS
    wd = np.exp(scale * (d[1:, :] - d[:-1, :]) ** 2) + EPS
    return wr, wd


def markers(scribble):
    """-> (markers int [h,w] with 0 = unknown and 1..K the rank-renumbered classes, K) or (None, 0) when a class 1..3 is absent"""
    s = np.asarray(scribble)
    present = [c for c in range(4) if (s == c).any()]
    if not all(c in present for c in (1, 2, 3)):
        return None, 0
    m = np.zeros(s.shape, np.int64)
    for rank, c in enumerate(present):          # marker c+1, renumbered by rank among the present markers (F17)
        m[s == c] = rank + 1
    return m, len(present)


def laplacian(wr, wd):
    h, w = wr.shape[0], wd.shape[1]
    idx = np.arange(h * w).reshape(h, w)
    rows = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    cols = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    vals = np.concatenate([wr.ravel(), wd.ravel()])
    A = sp.coo_matrix((vals, (rows, cols)), shape=(h * w, h * w)).tocsr()
    A = A + A.T
    return (sp.diags(np.asarray(A.sum(1)).ravel()) - A).tocsr()


def random_walker(image, scribble, beta=BETA):
    """-> (pseudo label u8 [h,w], probabilities fp64 [h,w,4] in the renumbered label order, zero where the label is all zero)"""
    m, K = markers(scribble)
    h, w = np.shape(scribble)
    prob = np.zeros((h, w, 4))
    if m is None:
        return np.zeros((h, w), np.uint8), prob
    d = rescale(image)
    L = laplacian(*edge_weights(d, beta))
    mf = m.ravel()
    U, M = np.flatnonzero(mf == 0), np.flatnonzero(mf > 0)
    onehot = np.zeros((len(M), K))
    onehot[np.arange(len(M)), mf[M] - 1] = 1.0
    rhs = -(L[U][:, M] @ onehot)
    x = spsolve(L[U][:, U].tocsc(), rhs)
    x = np.asarray(x).reshape(len(U), K)
    pf = prob.reshape(h * w, 4)
    pf[U, :K] = x
    pf[M, :K] = onehot
    lab = (np.argmax(pf[:, :K], 1)).astype(np.uint8)          # label - 1 of the renumbered markers
    return lab.reshape(h, w), prob


def chain(n, left=0.0, right=1.0, d=None, beta=BETA):
    """1-D chain of n pixels with a background seed at 0 and a class-1 seed at n-1: the probability of class 1 at pixel i is the
    cumulative resistance from the left end over the total, sum_{k<i} 1/w_k / sum_k 1/w_k (closed form of the harmonic function)."""
    d = np.linspace(left, right, n) if d is None else np.asarray(d, np.float64)
    w = np.exp(-beta / (10.0 * d.std()) * np.diff(d) ** 2) + EPS
    res = np.concatenate([[0.0], np.cumsum(1.0 / w)])
    return res / res[-1]


def ce_dice_loss(logits, label):
    """0.5 * (CrossEntropyLoss(ignore_index=4)(outputs, label) + DiceLoss(4)(softmax(outputs), label[:, None])),
    train_fully_supervised_2D.py:81-82,97-101"""
    import torch
    import wsl_oracle as O
    return 0.5 * (O.pce_loss(logits, label, 4) + O.dice_loss(torch.softmax(logits, 1), label[:, None].long()))


def ce_dice_step(p, image, label, masks=None):
    """one forward + ce_dice loss + backward of the single-head U-Net on CPU -> (loss, grads dict), like wsl_oracle.full_step"""
    import torch
    import wsl_oracle as O
    leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
    main = O.unet_forward(leaves, image, True, masks)
    loss = ce_dice_loss(main, label)
    names = [k for k, v in leaves.items() if v.requires_grad]
    gs = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), {k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(names, gs)}
