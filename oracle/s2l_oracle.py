"""CPU restatement of Scribble2Label (code/train_s2l.py, code/dataloaders/dataset_s2l.py) for the tests of the fused path.

  transform   dataset_s2l.py:103-153   rot90+flip | rotate(order 0, scipy's default cval 0 for every array, SURVEY F15), then
                                       zoom(order 0) -- the [h,w,4] weight as ONE 3-D array with class-axis factor 1, as the reference
  u_labels    train_s2l.py:128-145     the torch.where sequence, later classes overwrite earlier ones
  step_loss   train_s2l.py:123-147     CE(ignore 4) [+ 0.5 * CE(u-labels, ignore 4) from iter_num >= thr_iter]
  refresh     train_s2l.py:221-243     per slice: zoom to 256, softmax(model(img)) at batch 1 in train mode, zoom back, EMA
"""
import random

import numpy as np
import torch
import torch.nn.functional as F
from scipy import ndimage
from scipy.ndimage import zoom

import wsl_oracle as O


def transform(image, mask, scribble, weight, output_size):
    """RandomGenerator_s2l.__call__ (dataset_s2l.py:130-153) with the same random / np.random draws."""
    if random.random() > 0.5:                                          # random_rot_flip, :103-114
        k = np.random.randint(0, 4)
        image, mask, scribble, weight = (np.rot90(a, k) for a in (image, mask, scribble, weight))
        axis = np.random.randint(0, 2)
        image, mask, scribble, weight = (np.flip(a, axis=axis).copy() for a in (image, mask, scribble, weight))
    elif random.random() > 0.5:                                        # random_rotate, :117-123
        angle = np.random.randint(-20, 20)
        image, mask, scribble, weight = (ndimage.rotate(a, angle, order=0, reshape=False) for a in (image, mask, scribble, weight))
    x, y = image.shape
    fy, fx = output_size[0] / x, output_size[1] / y
    image, mask, scribble = (zoom(a, (fy, fx), order=0) for a in (image, mask, scribble))
    weight = zoom(weight, (fy, fx, 1), order=0)
    return image.astype(np.float32), mask.astype(np.uint8), scribble.astype(np.uint8), weight.astype(np.float32)


def u_labels(weight_batch, scribbles, thr_conf):
    """train_s2l.py:128-145: weight_batch [B,H,W,4] fp32, scribbles [B,H,W] -> int64 u-labels (4 = ignored)."""
    scribbles = scribbles.long()
    u = [torch.where((weight_batch[..., c] > thr_conf) & (scribbles == 4), torch.zeros_like(weight_batch[..., c]) + c,
                     4. * torch.ones_like(scribbles)) for c in range(4)]
    out = torch.ones_like(u[0]).long() * 4
    for c in range(4):
        out[u[c] == c] = c
    return out


def step_loss(outputs, scribble, weight_batch, iter_num, thr_iter=6000, thr_conf=0.8):
    """train_s2l.py:123-147 -> (loss, loss_ce, loss_u or None)."""
    loss_ce = F.cross_entropy(outputs, scribble.long(), ignore_index=4)
    if iter_num < thr_iter:
        return loss_ce, loss_ce, None
    loss_u = F.cross_entropy(outputs, u_labels(weight_batch, scribble, thr_conf), ignore_index=4)
    return loss_ce + 0.5 * loss_u, loss_ce, loss_u


def refresh(p, images, weights, alpha=0.2, masks=None, forward=None):
    """train_s2l.py:221-243 over the slices in order.  p: UNet state dict (running statistics UPDATED in place, once per slice);
    images: list of [h,w] fp32; weights: list of [h,w,4] fp32 (updated in place); masks[i] (optional): dropout keep masks of
    slice i for wsl_oracle.unet_forward.  forward(p, x, masks, new_stats) may replace the U-Net forward."""
    fwd = forward or (lambda p_, x_, m_, ns_: O.unet_forward(p_, x_, True, m_, ns_))
    for i, img0 in enumerate(images):
        h, w = img0.shape
        img = zoom(img0, (256 / h, 256 / w), order=0)
        x = torch.from_numpy(np.ascontiguousarray(img, dtype=np.float32)).unsqueeze(0).unsqueeze(0)
        new_stats = {}
        with torch.no_grad():
            pred = torch.softmax(fwd(p, x, None if masks is None else masks[i], new_stats), dim=1)
        for k, v in new_stats.items():
            p[k] = v
        for k in p:
            if k.endswith("num_batches_tracked"):
                p[k] = p[k] + 1
        pred = zoom(pred.squeeze(0).numpy(), (1, h / 256, w / 256), order=0)
        pred = torch.from_numpy(pred)
        wt = torch.from_numpy(weights[i])
        for c in range(4):
            wt[..., c] = alpha * pred[c] + (1 - alpha) * wt[..., c]
        weights[i] = wt.numpy()
    return weights
