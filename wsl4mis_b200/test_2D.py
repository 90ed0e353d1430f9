"""The reference's test step (test_2D_fully.py; test_2D_fully_sps.py for ``--model unet_cct``) with the same names, flags,
files and printed lines, run on the GPU:

    python -m wsl4mis_b200.test_2D --root_path ../data/ACDC --exp ACDC/pCE --model unet --sup_type scribble

For each fold 1-5 it loads ``../model/{exp}_{fold}/{sup_type}/iter_60000.pth``, predicts every test volume of the fold, scores
Dice / HD95 / ASD per class at the volume's voxel spacing, writes ``_pred`` / ``_img`` / ``_gt`` NIfTI files and prints the
mean Dice of the five folds.  The slices of a volume go through the network in fixed chunks of `chunk` 256x256 slices (the
last one padded), so every volume reuses one set of executor buffers; the resizes and the argmax run in csrc/losses.cu (SciPy's
``zoom(order=0)`` index rule) and all three classes' metrics come from one ``metric.surface_metrics`` call per volume.  The
per-volume device memory (image, label maps, metric workspace) is one buffer sized for the largest volume of the dataset before
the first volume runs, and ``main`` loads the five checkpoints into one network, so a five-fold pass allocates nothing after
its first volume.

``--root_path synthetic[:N]`` takes the test volumes from ``dataloaders.dataset.synthetic_acdc`` with the spacing of
``synthetic_spacing``; their "original" NIfTI files are written once per process into a temporary directory and read back
like real ones.
"""
import argparse
import atexit
import errno
import functools
import gc
import os
import re
import shutil
import tempfile

import numpy as np
import torch

from . import nifti
from ._lib import call
from .dataloaders.dataset import fold_ids, synthetic_acdc, synthetic_spacing
from .metric import surface_metrics, surface_metrics_workspace_bytes

PATCH = 256        # test_2D_fully.py:92,101
CHUNK = 16         # slices per forward

parser = argparse.ArgumentParser()
parser.add_argument('--root_path', type=str,
                    default='../data/ACDC', help='Name of Experiment')
parser.add_argument('--exp', type=str,
                    default='ACDC/WeaklySeg_pCE_MumfordShah_Loss', help='experiment_name')
parser.add_argument('--model', type=str,
                    default='unet', help='model_name')
parser.add_argument('--fold', type=str,
                    default='fold5', help='fold')
parser.add_argument('--num_classes', type=int, default=4,
                    help='output channel of network')
parser.add_argument('--sup_type', type=str, default="scribble",
                    help='label')


def get_fold_ids(fold):
    """test_2D_fully.py:34-71: [training patients, test patients] of `fold`, or the string "ERROR KEY"."""
    try:
        return list(fold_ids(fold))
    except ValueError:
        return "ERROR KEY"


def _is_synthetic(root_path):
    return str(root_path).startswith("synthetic")


@functools.lru_cache(maxsize=2)
def _synthetic_cases(root_path):
    n = int(str(root_path).split(":")[1]) if ":" in str(root_path) else 100
    return synthetic_acdc(n)


def _volume_files(root_path):
    """the file names of {root_path}/ACDC_training_volumes (os.listdir order); synthetic: one frame per patient"""
    if _is_synthetic(root_path):
        return [f"{pid}_frame01.h5" for pid in sorted(_synthetic_cases(root_path))]
    return os.listdir(root_path + "/ACDC_training_volumes")


def _h5(root_path, case):
    try:
        import h5py
    except ImportError as e:
        raise ImportError("h5py is required to read the ACDC files; pass base_dir='synthetic' for the generated stand-in") from e
    return h5py.File(root_path + "/ACDC_training_volumes/{}".format(case), 'r')


def _volume_shape(root_path, case):
    if _is_synthetic(root_path):
        return _synthetic_cases(root_path)[case.split("_")[0]][0].shape
    with _h5(root_path, case) as h5f:
        return h5f['image'].shape


def _read_volume(root_path, case):
    """-> (image, label) of one test volume (test_2D_fully.py:84-87)"""
    if _is_synthetic(root_path):
        img, lab, _ = _synthetic_cases(root_path)[case.split("_")[0]]
        return img, lab
    with _h5(root_path, case) as h5f:
        return h5f['image'][:], h5f['label'][:]


_synthetic_dir = None


def _synthetic_original(case, image):
    """the synthetic case as an 'original' NIfTI with its synthetic_spacing, written on first use"""
    global _synthetic_dir
    if _synthetic_dir is None:
        _synthetic_dir = tempfile.mkdtemp(prefix="wsl4mis_acdc_")
        atexit.register(shutil.rmtree, _synthetic_dir, True)
    path = os.path.join(_synthetic_dir, f"{case}.nii.gz")
    if not os.path.exists(path):
        nifti.write(path, image, nifti.header(image.shape, synthetic_spacing(case)))
    return path


def original_path(case, root_path, image=None):
    """The NIfTI the spacing and geometry come from: ../data/ACDC_training/{case}.nii.gz relative to the working directory, not to
    root_path (test_2D_fully.py:104).  Raises FileNotFoundError when it is missing: there is no default spacing."""
    if _is_synthetic(root_path):
        return _synthetic_original(case, image)
    path = "../data/ACDC_training/{}.nii.gz".format(case)
    if not os.path.exists(path):
        raise FileNotFoundError(errno.ENOENT, "original NIfTI of the test volume (its voxel spacing) not found", path)
    return path


def metric_spacing(spacing):
    """SimpleITK spacing (x, y, z) -> the voxelspacing the reference passes for array axes (z, y, x): (z, x, y), so rows take
    the x spacing (test_2D_fully.py:108-113; DESIGN F20)."""
    return (spacing[2], spacing[0], spacing[1])


def checkpoint_path(FLAGS):
    """test_2D_fully.py:136-137,145-146"""
    return os.path.join("../model/{}_{}/{}".format(FLAGS.exp, FLAGS.fold, FLAGS.sup_type), 'iter_60000.pth')


def predictions_dir(FLAGS):
    """test_2D_fully.py:138-139"""
    return "../model/{}_{}/{}/{}_predictions/".format(FLAGS.exp, FLAGS.fold, FLAGS.sup_type, FLAGS.model)


_ALIGN = 256      # surface_metrics' workspace alignment


def _volume_layout(shape):
    """byte offsets of (image f32, prediction u8, label u8, metric workspace, end) in the per-volume buffer"""
    n = int(np.prod(shape))
    offs, off = [], 0
    for size in (4 * n, n, n, surface_metrics_workspace_bytes(shape, 4)):
        offs.append(off)
        off += -(-size // _ALIGN) * _ALIGN
    return offs + [off]


_volume_buffers = {}


def _volume_buffer(device, nbytes):
    """the per-device buffer of the volumes' device memory, grown (never shrunk) to `nbytes`"""
    buf = _volume_buffers.get(device)
    if buf is None or buf.numel() < nbytes:
        _volume_buffers.pop(device, None)
        del buf
        buf = _volume_buffers[device] = torch.empty(nbytes, dtype=torch.uint8, device=device)
    return buf


def predict_volume(image, net, chunk=CHUNK, out=None):
    """[S,h,w] image -> uint8 label map [S,h,w] on the GPU: zoom(order=0) to 256x256, the network in eval() under no_grad,
    argmax of the first output (the main head of dual-head models, test_2D_fully_sps.py:97-100), zoom back.  The slices run in
    batches of exactly `chunk`, the last one padded with zeros; eval-mode BatchNorm uses running statistics, so the padding does
    not touch the real slices.  `out`: an [S,h,w] uint8 CUDA tensor to write the label map into."""
    dev = next(net.parameters()).device
    img = torch.as_tensor(np.ascontiguousarray(image) if isinstance(image, np.ndarray) else image, dtype=torch.float32).to(dev)
    S, h, w = img.shape
    x = torch.zeros((chunk, 1, PATCH, PATCH), dtype=torch.float32, device=dev)
    lab = torch.empty((chunk, PATCH, PATCH), dtype=torch.uint8, device=dev)
    pred = torch.empty((S, h, w), dtype=torch.uint8, device=dev) if out is None else out
    net.eval()
    for s0 in range(0, S, chunk):
        n = min(chunk, S - s0)
        call("wsl_zoom_nearest", img[s0:], 0, n, h, w, PATCH, PATCH, x)
        if n < chunk:
            x[n:].zero_()
        with torch.no_grad():
            out = net(x)
        logits = (out[0] if isinstance(out, (tuple, list)) else out).contiguous()
        # argmax(softmax(x)) == argmax(x); the first maximum wins, as in torch.argmax
        call("wsl_mix_argmax", logits, None, 1.0, 0.0, None, n, logits.shape[1], PATCH, PATCH, lab)
        call("wsl_zoom_nearest", lab, 1, n, PATCH, PATCH, h, w, pred[s0:])
    return pred


def _medpy_check(m, where):
    """medpy's surface distances raise on an empty mask; asd(pred, gt) checks the prediction first (test_2D_fully.py:78)"""
    if m.pred == 0:
        raise RuntimeError(f"The first supplied array does not contain any binary object. ({where})")
    if m.gt == 0:
        raise RuntimeError(f"The second supplied array does not contain any binary object. ({where})")


def _dc(m):
    """medpy.metric.binary.dc: 2|A&B| / (|A| + |B|), 0 when both masks are empty"""
    return 2.0 * m.inter / float(m.pred + m.gt) if m.pred + m.gt else 0.0


def calculate_metric_percase(pred, gt, spacing):
    """test_2D_fully.py:74-80: (dice, hd95, asd) of two binary masks at voxel spacing `spacing` (one value per axis)."""
    p = torch.from_numpy(np.ascontiguousarray(np.asarray(pred) != 0)).to("cuda", torch.uint8)
    g = torch.from_numpy(np.ascontiguousarray(np.asarray(gt) != 0)).to("cuda", torch.uint8)
    m = surface_metrics(p, g, 2, spacing)[0]
    _medpy_check(m, "calculate_metric_percase")
    return _dc(m), m.hd95, m.asd


def test_single_volume(case, net, test_save_path, FLAGS, chunk=CHUNK):
    """test_2D_fully.py:83-124: predict one test volume, score classes 1-3 at the original's spacing, write _pred / _img / _gt.
    Returns three (dice, hd95, asd) tuples."""
    image, label = _read_volume(FLAGS.root_path, case)
    dev = next(net.parameters()).device
    S, h, w = image.shape
    o_img, o_pred, o_gt, o_ws, end = _volume_layout(image.shape)
    buf = _volume_buffer(dev, end)
    img = buf[o_img:o_pred].view(torch.float32)[:S * h * w].view(S, h, w)
    img.copy_(torch.from_numpy(np.ascontiguousarray(image, dtype=np.float32)))
    gt = buf[o_gt:o_gt + S * h * w].view(S, h, w)
    gt.copy_(torch.from_numpy(np.ascontiguousarray(label)).to(torch.uint8))
    pred = predict_volume(img, net, chunk, out=buf[o_pred:o_pred + S * h * w].view(S, h, w))
    case = case.replace(".h5", "")
    org = nifti.read(original_path(case, FLAGS.root_path, image))
    res = []
    for k, m in enumerate(surface_metrics(pred, gt, 4, metric_spacing(org.spacing), workspace=buf[o_ws:end]), start=1):
        _medpy_check(m, f"case {case}, class {k}")
        res.append((_dc(m), m.hd95, m.asd))
    nifti.write(test_save_path + case + "_pred.nii.gz", pred.cpu().numpy().astype(np.float32), org.header)
    nifti.write(test_save_path + case + "_img.nii.gz", np.asarray(image).astype(np.float32), org.header)
    nifti.write(test_save_path + case + "_gt.nii.gz", np.asarray(label).astype(np.float32), org.header)
    return tuple(res)


def Inference(FLAGS, chunk=CHUNK, net=None):
    """test_2D_fully.py:127-165: score the fold's test volumes with ../model/{exp}_{fold}/{sup_type}/iter_60000.pth; returns the
    mean Dice over classes 1-3 and volumes.  `net` (optional): a network of FLAGS.model to load the checkpoint into instead of a
    new one."""
    from .networks.net_factory import net_factory
    train_ids, test_ids = get_fold_ids(FLAGS.fold)
    all_volumes = _volume_files(FLAGS.root_path)
    image_list = []
    for ids in test_ids:
        image_list.extend([x for x in all_volumes if re.match('{}.*'.format(ids), x) is not None])
    test_save_path = predictions_dir(FLAGS)
    if os.path.exists(test_save_path):
        shutil.rmtree(test_save_path)
    os.makedirs(test_save_path)
    own_net = net is None
    if own_net:
        net = net_factory(net_type=FLAGS.model, in_chns=1, class_num=FLAGS.num_classes)
    save_mode_path = checkpoint_path(FLAGS)
    # read on the host and copied into the parameters: changing folds allocates no device memory
    net.load_state_dict(torch.load(save_mode_path, map_location="cpu"))
    print("init weight from {}".format(save_mode_path))
    net.eval()
    # every fold lists the same volumes: size the volume buffer for the largest once
    _volume_buffer(next(net.parameters()).device, max(_volume_layout(_volume_shape(FLAGS.root_path, v))[-1] for v in all_volumes))

    first_total = 0.0
    second_total = 0.0
    third_total = 0.0
    for case in image_list:
        print(case)
        first_metric, second_metric, third_metric = test_single_volume(case, net, test_save_path, FLAGS, chunk)
        first_total += np.asarray(first_metric)
        second_total += np.asarray(second_metric)
        third_total += np.asarray(third_metric)
    avg_metric = [first_total / len(image_list), second_total / len(image_list), third_total / len(image_list)]
    print(avg_metric)
    print((avg_metric[0] + avg_metric[1] + avg_metric[2]) / 3)
    if own_net:      # the network and its executor reference each other: collect them now and release their memory
        del net
        gc.collect()
    return ((avg_metric[0] + avg_metric[1] + avg_metric[2]) / 3)[0]


def main(argv=None):
    """test_2D_fully.py:168-177: folds 1-5, then the mean of the five mean Dice values"""
    from .networks.net_factory import net_factory
    FLAGS = parser.parse_args(argv)
    net = net_factory(net_type=FLAGS.model, in_chns=1, class_num=FLAGS.num_classes)    # one network, five checkpoints
    total = 0.0
    for i in [1, 2, 3, 4, 5]:
        FLAGS.fold = "fold{}".format(i)
        print("Inference fold{}".format(i))
        mean_dice = Inference(FLAGS, net=net)
        total += mean_dice
    print(total / 5.0)
    return total / 5.0


if __name__ == '__main__':
    main()
