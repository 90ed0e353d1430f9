"""Random-walker pseudo labels from scribbles on the GPU (dataloaders/acdc_pseudo_label_random_walker.py:9-26 of the reference:
``pseudo_label_generator_acdc``, skimage ``random_walker(..., beta=100, mode='bf')`` per slice).

The reference runs this offline on the NIfTI volumes, one SuperLU solve per slice on the CPU; the shipped ACDC slice files carry
no ``random_walker`` dataset.  Here one launch of ``wsl_random_walker`` solves every slice of a ragged store with a batched,
matrix-free Jacobi-preconditioned CG (one persistent CTA per slice, all four label columns together), so the pseudo labels of
the ~1 900 training slices are computed in seconds when a dataset is constructed."""
import ctypes

import numpy as np
import torch

from .._lib import call


def _solve(images, scribbles, offs, shapes, beta, tol, max_iter, want_probs, ctas):
    """flat device stores -> (labels u8 [px], probs fp32 [px, 4] or None, iters int [S], resid float [S])"""
    dev = images.device
    S = len(offs)
    px = shapes[:, 0].astype(np.int64) * shapes[:, 1]
    order = np.argsort(-px, kind="stable").astype(np.int32)          # largest slices first: the last wave is short
    out2 = (ctypes.c_longlong * 2)()
    call("wsl_random_walker_workspace", int(ctas), int(px.max()), ctypes.addressof(out2))
    n_ctas = min(int(out2[0]), S)
    call("wsl_random_walker_workspace", n_ctas, int(px.max()), ctypes.addressof(out2))
    ws = torch.empty(int(out2[1]), dtype=torch.float32, device=dev)
    offs_d = torch.from_numpy(np.ascontiguousarray(offs, dtype=np.int64)).to(dev)
    shapes_d = torch.from_numpy(np.ascontiguousarray(shapes, dtype=np.int32)).to(dev)
    order_d = torch.from_numpy(order).to(dev)
    labels = torch.empty(images.numel(), dtype=torch.uint8, device=dev)
    probs = torch.empty(images.numel(), 4, dtype=torch.float32, device=dev) if want_probs else None
    iters = torch.empty(S, dtype=torch.int32, device=dev)
    resid = torch.empty(S, dtype=torch.float32, device=dev)
    call("wsl_random_walker", images, scribbles, offs_d, shapes_d, order_d, S, float(beta), float(tol), int(max_iter), ws, n_ctas,
         int(px.max()), labels, probs, iters, resid)
    return labels, probs, iters.cpu().numpy(), resid.cpu().numpy()


def random_walker_labels(images, scribbles=None, beta=100.0, tol=1e-7, max_iter=20000, probs=False, names=None, device=None, ctas=0):
    """Random-walker pseudo labels of every slice in one GPU launch.

    images: a list of 2-D fp32 images in [0, 1] (with `scribbles`: a list of u8 maps of the same shapes, 0..3 = class,
    4 = unlabelled), or a `SliceStore` built with ``scribbles=``.  Per slice: all zeros when class 1, 2 or 3 has no scribble;
    otherwise the argmax of the random-walker probabilities, seeds keeping their class (DESIGN §2 F17: without a background
    scribble every class shifts down by one, as skimage's relabelling does).  tol is the per-slice stopping rule
    max_l ||r_l|| / ||b_l|| <= tol; a loose tolerance flips labels near class boundaries, so keep the default.

    -> (labels, stats).  labels: a list of u8 [h, w] numpy arrays, or for a SliceStore a new SliceStore (same images, names and
    scribbles, the pseudo labels as its labels) that `GpuLoader` trains from.  stats: {'iters': int [S], 'resid': float [S]}
    and, with probs=True, 'probs': the per-pixel column probabilities (a list of fp32 [h, w, 4] arrays, or the flat [px, 4]
    device tensor for a SliceStore).

    Raises RuntimeError naming every slice that reached max_iter without converging; there is no fallback."""
    from .dataset import SliceStore
    if isinstance(images, SliceStore):
        store = images
        if store.scribbles is None:
            raise ValueError("random_walker_labels needs a SliceStore built with scribbles=")
        flat_i, flat_s, offs, shapes = store.images, store.scribbles, store.offs, np.asarray(store.shapes)
        names = store.names
    else:
        if scribbles is None or len(scribbles) != len(images) or len(images) == 0:
            raise ValueError("random_walker_labels needs one scribble map per image")
        store = SliceStore.from_arrays(images, scribbles, names, device)       # the scribbles ride in the label store
        flat_i, flat_s, offs, shapes = store.images, store.labels, store.offs, np.asarray(store.shapes)
        names = names if names is not None else [str(i) for i in range(len(images))]
    lab, prob, iters, resid = _solve(flat_i, flat_s, np.asarray(offs), shapes, beta, tol, max_iter, probs, ctas)
    bad = [i for i in range(len(iters)) if iters[i] < 0 or not resid[i] <= np.float32(tol)]
    if bad:
        desc = ", ".join(f"{names[i]} (slice {i}, {int(shapes[i, 0])}x{int(shapes[i, 1])}: " +
                         ("does not fit the workspace" if iters[i] < 0 else f"residual {resid[i]:.3g} after {iters[i]} iterations") + ")"
                         for i in bad[:20])
        raise RuntimeError(f"random walker did not converge to tol={tol:g} within max_iter={max_iter} for {len(bad)} slice(s): {desc}")
    stats = {"iters": iters, "resid": resid}
    if isinstance(images, SliceStore):
        if probs:
            stats["probs"] = prob
        out = SliceStore(store.images, lab, store.offs, store.shapes, np.zeros(len(store), bool), store.names)
        out.scribbles = store.scribbles          # kept for reference; no Scribble2Label prediction memory is allocated
        return out, stats
    lab_h = lab.cpu().numpy()
    prob_h = prob.cpu().numpy() if probs else None
    labels, plist = [], []
    for i in range(len(offs)):
        h, w = int(shapes[i, 0]), int(shapes[i, 1])
        labels.append(lab_h[offs[i]: offs[i] + h * w].reshape(h, w).copy())
        if probs:
            plist.append(prob_h[offs[i]: offs[i] + h * w].reshape(h, w, 4).copy())
    if probs:
        stats["probs"] = plist
    return labels, stats
