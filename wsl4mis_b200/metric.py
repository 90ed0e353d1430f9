"""medpy.metric.binary's ``dc`` / ``jc`` / ``hd95`` / ``asd`` on the GPU, and ``surface_metrics``, the per-volume form over label
maps that the validation pass uses (val_2D.py:7-15, test_2D_fully.py:74-80, utils/metrics.py:19-25).

Surfaces, the exact anisotropic distance transforms and the order statistics of HD95 run in csrc/metrics.cu; one small
device-to-host copy brings back a few doubles per class.  The last step of ``np.percentile`` (numpy's ``_lerp`` between the two
order statistics) is done here in the same float64 arithmetic, so HD95 equals medpy's value bit for bit wherever the distances do
(unit and integer spacings).
"""
import ctypes
from typing import NamedTuple

import numpy as np
import torch

from ._lib import LIB, call


class SurfaceMetrics(NamedTuple):
    """Per class: overlap counts and the surface-distance metrics.  hd95 / asd are nan when either mask is empty (medpy raises
    there; each caller applies its own rule from the counts)."""
    inter: int
    pred: int
    gt: int
    union: int
    hd95: float
    asd: float


def _spacing(voxelspacing, ndim):
    """scalar or one value per axis -> ndim floats (medpy's _ni_support._normalize_sequence)."""
    if voxelspacing is None:
        return (1.0,) * ndim
    sp = np.asarray(voxelspacing, dtype=np.float64)
    if sp.ndim == 0:
        return (float(sp),) * ndim
    if sp.shape != (ndim,):
        raise RuntimeError("sequence argument must have length equal to input rank")
    return tuple(float(v) for v in sp)


def _percentile95(lo, hi, n):
    """np.percentile(x, 95) from its two order statistics x[lo] <= x[hi] ('linear' method, numpy's _lerp)."""
    vi = (n - 1) * 0.95
    if vi >= n - 1:
        return hi
    g = vi - float(np.floor(vi))
    d = hi - lo
    return hi - d * (1 - g) if g >= 0.5 else lo + d * g


def _device_mask(x, device=None):
    """numpy array or tensor -> contiguous CUDA uint8 0/1 mask, nonzero = 1 (medpy's astype(bool)), compared in the input's own
    dtype so that 0.5 or 256 count as True."""
    m = (x != 0) if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(x) != 0))
    dev = device or (m.device if m.is_cuda else "cuda")
    return m.to(device=dev, dtype=torch.uint8).contiguous()


def surface_metrics_workspace_bytes(shape, classes):
    """device bytes `surface_metrics` needs as workspace for volumes of `shape` ([S,H,W] or [H,W])"""
    S, H, W = ((1,) + tuple(shape)) if len(shape) == 2 else tuple(shape)
    nbytes = ctypes.c_longlong(0)
    call("wsl_surface_metrics_workspace", len(shape), S, H, W, classes, ctypes.addressof(nbytes))
    return nbytes.value


def surface_metrics(pred, gt, classes, voxelspacing=None, workspace=None):
    """Counts, hd95 and asd of every class 1..classes-1 of two uint8 label volumes ([S,H,W] or [H,W], CUDA tensors) in one
    kernel sequence.  Returns [SurfaceMetrics] indexed by class - 1.  `workspace` (optional): a 256-byte aligned uint8 CUDA
    tensor of at least `surface_metrics_workspace_bytes` bytes to use instead of a fresh allocation."""
    if pred.shape != gt.shape:
        raise ValueError(f"surface_metrics: shape mismatch {tuple(pred.shape)} vs {tuple(gt.shape)}")
    if pred.dim() not in (2, 3):
        raise ValueError(f"surface_metrics: volumes must have rank 2 or 3 (got {pred.dim()})")
    if not (pred.is_cuda and gt.is_cuda and pred.device == gt.device) or pred.dtype != torch.uint8 or gt.dtype != torch.uint8:
        raise ValueError("surface_metrics: pred and gt must be uint8 tensors on the same CUDA device")
    ndim = pred.dim()
    S, H, W = ((1,) + tuple(pred.shape)) if ndim == 2 else tuple(pred.shape)
    sp = _spacing(voxelspacing, ndim)
    sz, sy, sx = ((1.0,) + sp) if ndim == 2 else sp
    with torch.cuda.device(pred.device):
        nbytes = surface_metrics_workspace_bytes(pred.shape, classes)
        if workspace is None:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=pred.device)
        else:
            if workspace.dtype != torch.uint8 or workspace.device != pred.device or workspace.numel() < nbytes:
                raise ValueError(f"surface_metrics: workspace must be a uint8 tensor of >= {nbytes} bytes on {pred.device}")
            ws = workspace
        out = torch.empty((classes - 1, 12), dtype=torch.float64, device=pred.device)
        call("wsl_surface_metrics", pred.contiguous(), gt.contiguous(), ndim, S, H, W, classes, sz, sy, sx, ws, out)
        o = out.cpu().numpy()
    return decode(o)


def decode(rows):
    """[classes-1, 12] float64 rows of the metrics kernels (see include/wsl4mis_b200.h) -> [SurfaceMetrics] indexed by class - 1"""
    res = []
    for r in rows:
        inter, npred, ngt, union, na, nb = (int(v) for v in r[:6])
        if npred and ngt:
            hd, asd = float(_percentile95(float(r[10]), float(r[11]), na + nb)), float(r[6] / na)
        else:
            hd = asd = float("nan")
        res.append(SurfaceMetrics(inter, npred, ngt, union, hd, asd))
    return res


_VOLUME = np.dtype([("voff", "<i8"), ("roff", "<i8"), ("coff", "<i8"), ("S", "<i4"), ("H", "<i4"), ("W", "<i4"), ("rank3", "<i4"),
                    ("sz", "<f8"), ("sy", "<f8"), ("sx", "<f8")])


class VolumeSet:
    """A set of V label volumes of their own shapes ([S,H,W] or [H,W]) packed back to back, scored by ONE batched metrics launch
    sequence (`wsl_surface_metrics_batched`) into [V, classes-1, 12] rows, bit-identical to V `surface_metrics` calls.  The volume
    table and the workspace are allocated once, here, on `device`; `offsets[v]` is volume v's first voxel in the packed arrays."""

    def __init__(self, shapes, classes, spacings=None, device="cuda"):
        assert LIB.load().wsl_surface_metrics_volume_bytes() == _VOLUME.itemsize, "volume table layout mismatch"
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.classes, self.device = int(classes), torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        V = len(self.shapes)
        if V == 0:
            raise ValueError("VolumeSet: no volumes")
        tab = np.zeros(V, dtype=_VOLUME)
        voff = roff = coff = 0
        for v, shape in enumerate(self.shapes):
            if len(shape) not in (2, 3):
                raise ValueError(f"VolumeSet: volume {v} has rank {len(shape)} (2 or 3)")
            S, H, W = ((1,) + shape) if len(shape) == 2 else shape
            sp = _spacing(None if spacings is None else spacings[v], len(shape))
            sz, sy, sx = ((1.0,) + sp) if len(shape) == 2 else sp
            if not all(np.isfinite(x) and x > 0 for x in (sz, sy, sx)):
                raise ValueError(f"VolumeSet: volume {v}: voxel spacing must be finite and > 0 (got {(sz, sy, sx)})")
            surface_metrics_workspace_bytes(shape, classes)          # the single-volume limits hold for every volume
            tab[v] = (voff, roff, coff, S, H, W, len(shape) == 3, sz, sy, sx)
            voff, roff, coff = voff + S * H * W, roff + S * H, coff + H * W
        self.offsets = [int(o) for o in tab["voff"]] + [voff]
        self.n, self.rows, self.cols = voff, roff, coff
        self.max_n = int(max(int(t["S"]) * int(t["H"]) * int(t["W"]) for t in tab))
        self.max_w = int(tab["W"].max())
        with torch.cuda.device(self.device):
            self.table = torch.from_numpy(tab.view(np.uint8).copy()).to(self.device)
            nbytes = ctypes.c_longlong(0)
            call("wsl_surface_metrics_batched_workspace", V, self.n, self.rows, self.classes, ctypes.addressof(nbytes))
            self.workspace = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)

    def __len__(self):
        return len(self.shapes)

    def __call__(self, pred, gt, out):
        """enqueue the metrics of packed uint8 pred / gt ([n] CUDA) into out ([V, classes-1, 12] float64 CUDA); no host sync"""
        V = len(self.shapes)
        for name, t in (("pred", pred), ("gt", gt)):
            if not (t.is_cuda and t.device == self.device and t.dtype == torch.uint8 and t.is_contiguous() and t.numel() == self.n):
                raise ValueError(f"VolumeSet: {name} must be a contiguous uint8 tensor of {self.n} voxels on {self.device}")
        if not (out.device == self.device and out.dtype == torch.float64 and tuple(out.shape) == (V, self.classes - 1, 12)):
            raise ValueError(f"VolumeSet: out must be a float64 [{V}, {self.classes - 1}, 12] tensor on {self.device}")
        with torch.cuda.device(self.device):
            call("wsl_surface_metrics_batched", pred, gt, self.table, V, self.n, self.rows, self.cols, self.max_n, self.max_w,
                 self.classes, self.workspace, out)
        return out


def _binary(result, reference, voxelspacing, connectivity):
    if connectivity != 1:
        raise NotImplementedError("only connectivity=1 (face neighbours), the value every caller uses, is implemented")
    a = _device_mask(result)
    b = _device_mask(reference, a.device)
    if a.shape != b.shape:
        raise ValueError(f"shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}")
    m = surface_metrics(a, b, 2, voxelspacing)[0]
    if m.pred == 0:
        raise RuntimeError('The first supplied array does not contain any binary object.')
    if m.gt == 0:
        raise RuntimeError('The second supplied array does not contain any binary object.')
    return m


def _counts(result, reference):
    a = _device_mask(result)
    b = _device_mask(reference, a.device)
    if a.shape != b.shape:
        raise ValueError(f"shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}")
    counts = torch.zeros(6, dtype=torch.int64, device=a.device)
    with torch.cuda.device(a.device):
        call("wsl_overlap_counts", a, b, a.numel(), 2, counts)
        inter, sa, sb = (int(v) for v in counts[3:].cpu())
    return inter, sa, sb


def dc(result, reference):
    """Dice coefficient 2|A&B| / (|A| + |B|), 0.0 when both are empty (medpy.metric.binary.dc)."""
    inter, sa, sb = _counts(result, reference)
    try:
        return 2.0 * inter / float(sa + sb)
    except ZeroDivisionError:
        return 0.0


def jc(result, reference):
    """Jaccard coefficient |A&B| / |A|B| (medpy.metric.binary.jc)."""
    inter, sa, sb = _counts(result, reference)
    return float(inter) / float(sa + sb - inter)


def hd95(result, reference, voxelspacing=None, connectivity=1):
    """95th percentile of the symmetric surface distances (medpy.metric.binary.hd95)."""
    return _binary(result, reference, voxelspacing, connectivity).hd95


def asd(result, reference, voxelspacing=None, connectivity=1):
    """Mean distance of the surface of `result` to the surface of `reference` (medpy.metric.binary.asd)."""
    return _binary(result, reference, voxelspacing, connectivity).asd
