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
from .metric import VolumeSet, decode, surface_metrics

PATCH = 256        # the scripts' patch size (val_2D.py:18)


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


class ValidationSet:
    """The validation split resident on the GPU and scored in one batched pass (the trainer's every-200-iterations validation).

    Built once from ``BaseDataSets(base_dir, fold=fold, split="val")`` (ACDC h5 or ``synthetic[:N]``): every slice of every volume
    is resized to 256 x 256 (SciPy's ``zoom(order=0)`` rule, one ``wsl_zoom_nearest_ragged`` launch) into a padded batch that stays
    on the device with the packed labels, the slice and volume tables and the metrics workspace.  ``score(net, classes)`` then runs
    the network in ``eval()`` on fixed chunks of `chunk` slices (eval-mode BatchNorm uses running statistics, so a slice's logits do
    not depend on its batch), takes the argmax of head 0, resizes every label map back to its volume's own size in one launch,
    scores all (volume, class) pairs in one batched metrics launch sequence and brings the results back in one device-to-host
    copy.  It returns, per volume, what ``test_single_volume`` returns for it: ``[(dice, hd95)] * (classes - 1)``, (0, 0) for an
    empty prediction, medpy's RuntimeError (naming the case and the class) for a prediction against an empty label."""

    def __init__(self, base_dir, fold="fold1", device=None, chunk=64):
        from .dataloaders.dataset import BaseDataSets
        db = BaseDataSets(base_dir=base_dir, fold=fold, split="val")
        images, labels = [], []
        for case in db.sample_list:
            img, lab = db._read(case)
            images.append(np.asarray(img, dtype=np.float32))
            labels.append(np.asarray(lab))
        self._setup(images, labels, [c.replace(".h5", "") for c in db.sample_list], device, chunk)

    @classmethod
    def from_arrays(cls, images, labels, names=None, device=None, chunk=64):
        """the set of [S,h,w] image / label volumes given as arrays"""
        self = cls.__new__(cls)
        self._setup([np.asarray(i, dtype=np.float32) for i in images], [np.asarray(l) for l in labels],
                    names if names is not None else [str(i) for i in range(len(images))], device, chunk)
        return self

    def _setup(self, images, labels, names, device, chunk):
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.names, self.chunk = list(names), int(chunk)
        for name, im, lb in zip(self.names, images, labels):
            if im.ndim != 3 or im.shape != lb.shape:
                raise ValueError(f"ValidationSet: volume {name} must be [S,h,w] with matching image and label (got {im.shape}, "
                                 f"{lb.shape}); 2-D validation volumes are not supported")
        self.shapes = [tuple(im.shape) for im in images]
        slices = [(s, h, w) for (S, h, w) in self.shapes for s in range(S)]
        self.n_slices = len(slices)
        self.n_pad = -(-self.n_slices // self.chunk) * self.chunk
        rows, off = [], 0
        for (S, h, w) in self.shapes:
            for _ in range(S):
                rows.append((off, h, w))
                off += h * w
        self.max_hw = max(h * w for (_, h, w) in self.shapes)
        dev = self.device
        self.slice_table = torch.tensor(rows, dtype=torch.int64).to(dev)
        flat_i = torch.from_numpy(np.concatenate([im.ravel() for im in images])).to(dev)
        self.gt = torch.from_numpy(np.concatenate([lb.astype(np.uint8).ravel() for lb in labels])).to(dev)
        self.pred = torch.empty_like(self.gt)
        self.x = torch.zeros((self.n_pad, 1, PATCH, PATCH), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            call("wsl_zoom_nearest_ragged", flat_i, 0, self.slice_table, self.n_slices, self.max_hw, 0, PATCH, PATCH, self.x)
        self.lab = torch.empty((self.n_pad, PATCH, PATCH), dtype=torch.uint8, device=dev)
        self._metrics = {}            # classes -> (VolumeSet, device rows, pinned host rows, event)

    def __len__(self):
        return len(self.shapes)

    def _metric_buffers(self, classes):
        if classes not in self._metrics:
            vs = VolumeSet(self.shapes, classes, device=self.device)
            out = torch.empty((len(vs), classes - 1, 12), dtype=torch.float64, device=self.device)
            host = torch.empty(out.shape, dtype=torch.float64, pin_memory=True)
            self._metrics[classes] = (vs, out, host, torch.cuda.Event())
        return self._metrics[classes]

    @torch.no_grad()
    def predict(self, net):
        """the label maps of every volume, packed back to back in `self.pred` (uint8, device); leaves `net` in eval()"""
        net.eval()
        with torch.cuda.device(self.device):
            for c0 in range(0, self.n_pad, self.chunk):
                out = net(self.x[c0:c0 + self.chunk])
                logits = (out[0] if isinstance(out, (tuple, list)) else out).contiguous()
                # argmax(softmax(x)) == argmax(x); the first maximum wins, as in torch.argmax
                call("wsl_mix_argmax", logits, None, 1.0, 0.0, None, self.chunk, logits.shape[1], PATCH, PATCH, self.lab[c0:])
            call("wsl_zoom_nearest_ragged", self.lab, 1, self.slice_table, self.n_slices, self.max_hw, 1, PATCH, PATCH, self.pred)
        return self.pred

    def score(self, net, classes):
        """-> one ``[(dice, hd95)] * (classes - 1)`` list per volume, in dataset order (see the class docstring)"""
        vs, out, host, done = self._metric_buffers(int(classes))
        self.predict(net)
        with torch.cuda.device(self.device):
            vs(self.pred, self.gt, out)
            host.copy_(out, non_blocking=True)
            done.record()
        done.synchronize()            # the pass's one wait on the device
        res = []
        for name, rows in zip(self.names, host.numpy()):
            per = []
            for k, m in enumerate(decode(rows), start=1):
                if m.pred > 0:   # calculate_metric_percase (val_2D.py:7-15): (0, 0) when the prediction is empty
                    if m.gt == 0:
                        raise RuntimeError(f"The second supplied array does not contain any binary object. (case {name}, class {k})")
                    per.append((2.0 * m.inter / float(m.pred + m.gt), m.hd95))
                else:
                    per.append((0, 0))
            res.append(per)
        return res
