"""GPU validation path with the reference's ``val_2D`` names (val_2D.py:7-50,90-124; SURVEY 8(f) rank 1).

The reference loops over the slices of a volume on the host: scipy ``zoom(order=0)`` to 256x256, a batch-1 forward,
argmax, ``zoom`` back, then medpy Dice / HD95 per class.  Here all slices of the volume go through the network as one
batch; both nearest-neighbour resizes, the argmax and the Dice overlap counts run on the GPU (SciPy's index rule is
reproduced bit for bit, see csrc/losses.cu).  HD95 too: surfaces, exact distance transforms and the percentile's order
statistics run in csrc/metrics.cu (``metric.surface_metrics``), one call per volume.  ``hd95`` / ``calculate_metric_percase``
below keep medpy's host algorithm on scipy (medpy is not a dependency) as the reference the GPU path is tested against.
"""
import numpy as np
import torch

from ._lib import call
from .metric import surface_metrics


def _surface_distances(result, reference):
    """Distances from the surface voxels of `result` to the surface of `reference` (the algorithm of
    medpy.metric.binary.__surface_distances with voxelspacing=None, connectivity=1)."""
    from scipy.ndimage import binary_erosion, distance_transform_edt, generate_binary_structure
    result, reference = np.atleast_1d(result.astype(bool)), np.atleast_1d(reference.astype(bool))
    if not result.any():
        raise RuntimeError('The first supplied array does not contain any binary object.')
    if not reference.any():
        raise RuntimeError('The second supplied array does not contain any binary object.')
    fp = generate_binary_structure(result.ndim, 1)
    rb = result ^ binary_erosion(result, structure=fp, iterations=1)
    fb = reference ^ binary_erosion(reference, structure=fp, iterations=1)
    dt = distance_transform_edt(~fb)
    return dt[rb]


def hd95(result, reference):
    """95th percentile of the symmetric surface distances (medpy.metric.binary.hd95)."""
    return float(np.percentile(np.hstack((_surface_distances(result, reference), _surface_distances(reference, result))), 95))


def _predict_volume(image, net, patch_size, head):
    """image: [S,h,w] array/tensor -> uint8 prediction [S,h,w] on the GPU."""
    dev = next(net.parameters()).device
    img = torch.as_tensor(np.ascontiguousarray(image), dtype=torch.float32).to(dev)
    S, h, w = img.shape
    H, W = int(patch_size[0]), int(patch_size[1])
    x = torch.empty((S, 1, H, W), dtype=torch.float32, device=dev)
    call("wsl_zoom_nearest", img, 0, S, h, w, H, W, x)
    net.eval()
    with torch.no_grad():
        out = net(x)
    logits = (out[head] if isinstance(out, (tuple, list)) else out).contiguous()
    lab = torch.empty((S, H, W), dtype=torch.uint8, device=dev)
    # argmax(softmax(x)) == argmax(x); first maximum wins like torch.argmax
    call("wsl_mix_argmax", logits, None, 1.0, 0.0, None, S, logits.shape[1], H, W, lab)
    pred = torch.empty((S, h, w), dtype=torch.uint8, device=dev)
    call("wsl_zoom_nearest", lab, 1, S, H, W, h, w, pred)
    return pred


def _metrics(pred, label, classes):
    gt = torch.as_tensor(np.ascontiguousarray(label)).to(device=pred.device, dtype=torch.uint8)
    out = []
    for m in surface_metrics(pred.contiguous(), gt.contiguous(), classes):
        if m.pred > 0:   # calculate_metric_percase (val_2D.py:7-15): (0, 0) when the prediction is empty
            if m.gt == 0:
                raise RuntimeError('The second supplied array does not contain any binary object.')
            out.append((2.0 * m.inter / float(m.pred + m.gt), m.hd95))
        else:
            out.append((0, 0))
    return out


def calculate_metric_percase(pred, gt):
    """val_2D.py:7-15 on host arrays (binary masks)."""
    pred, gt = np.asarray(pred) > 0, np.asarray(gt) > 0
    if pred.sum() > 0:
        return 2.0 * np.count_nonzero(pred & gt) / float(np.count_nonzero(pred) + np.count_nonzero(gt)), hd95(pred, gt)
    return 0, 0


def test_single_volume(image, label, net, classes, patch_size=[256, 256]):
    """val_2D.py:18-50: image/label are [1,S,h,w] (or [1,h,w]) tensors of one volume; returns [(dice, hd95)] per class."""
    image, label = image.squeeze(0).cpu().detach().numpy(), label.squeeze(0).cpu().detach().numpy()
    if image.ndim == 2:
        image, label = image[None], label[None]
        patch_size = image.shape[1:]          # the reference feeds a single 2D slice without resizing (:37-43)
    return _metrics(_predict_volume(image, net, patch_size, 0), label, classes)


def test_single_volume_cct(image, label, net, classes, patch_size=[256, 256]):
    """val_2D.py:90-124: dual-head models, metrics on the main head."""
    return test_single_volume(image, label, net, classes, patch_size)


def test_single_volume_ds(image, label, net, classes, patch_size=[256, 256]):
    """val_2D.py:53-87: deep-supervision models (four outputs), metrics on the full-resolution head (output 0)."""
    return test_single_volume(image, label, net, classes, patch_size)
