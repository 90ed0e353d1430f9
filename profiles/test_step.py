"""Cost of the test step (wsl4mis_b200/test_2D.py) on one GPU: ``Inference`` over fold 1 of synthetic:100 (UNet, bf16) against the
reference's host loop restated in the same run (test_2D_fully.py:83-124: per-slice scipy zoom, a batch-1 forward, softmax +
argmax, zoom back, Dice / HD95 / ASD per class with scipy at the volume's spacing, the three NIfTI files).  The checkpoint
comes from --train-steps captured ce_dice steps (batch 12), so the predictions have the shape of a real run's.  Both arms
write their files into a temporary directory.  Prints one JSON line with the times, whether the two arms agree, the device
name and its power limit.

    python profiles/test_step.py [--patients 100] [--train-steps 400]
"""
import argparse
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.ndimage import zoom  # noqa: E402

import _metric_oracle as M  # noqa: E402
from s2l_step import device_info  # noqa: E402
import wsl4mis_b200.test_2D as T  # noqa: E402
from wsl4mis_b200 import nifti  # noqa: E402
from wsl4mis_b200.dataloaders.dataset import GpuLoader, SliceStore, fold_ids, synthetic_acdc  # noqa: E402
from wsl4mis_b200.engine import TrainStep  # noqa: E402
from wsl4mis_b200.networks.net_factory import net_factory  # noqa: E402
from wsl4mis_b200.networks.unet import UNet  # noqa: E402


def host_loop(FLAGS, image_list, out):
    """test_2D_fully.py:127-165 with the per-slice body of :83-124 (scipy for zoom and the metrics, this package's writer for
    SimpleITK's)"""
    net = net_factory(net_type=FLAGS.model, in_chns=1, class_num=FLAGS.num_classes)
    net.load_state_dict(torch.load(T.checkpoint_path(FLAGS)))
    net.eval()
    total = [0.0, 0.0, 0.0]
    for case in image_list:
        image, label = T._read_volume(FLAGS.root_path, case)
        prediction = np.zeros_like(label)
        for ind in range(image.shape[0]):
            x, y = image.shape[1:]
            sl = zoom(image[ind], (256 / x, 256 / y), order=0)
            with torch.no_grad():
                o = net(torch.from_numpy(sl).unsqueeze(0).unsqueeze(0).float().cuda())
                o = torch.argmax(torch.softmax(o, dim=1), dim=1).squeeze(0).cpu().numpy()
            prediction[ind] = zoom(o, (x / 256, y / 256), order=0)
        case = case.replace(".h5", "")
        org = nifti.read(T.original_path(case, FLAGS.root_path, image))
        sp = T.metric_spacing(org.spacing)
        for k in range(1, 4):
            p, g = prediction == k, label == k
            total[k - 1] += np.asarray((M.dc(p, g), M.hd95(p, g, sp), M.asd(p, g, sp)))
        for name, a in (("_pred", prediction), ("_img", image), ("_gt", label)):
            nifti.write(out + case + name + ".nii.gz", a.astype(np.float32), org.header)
    avg = [t / len(image_list) for t in total]
    return ((avg[0] + avg[1] + avg[2]) / 3)[0]


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patients", type=int, default=100)
    ap.add_argument("--train-steps", type=int, default=400)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/test_step.py measures on a GPU"
    root = f"synthetic:{a.patients}"
    cases = synthetic_acdc(a.patients)
    train, test = fold_ids("fold1")
    torch.manual_seed(0)
    net = UNet(1, 4).cuda()
    ims = [im for p in sorted(cases) if p in train for im in cases[p][0]]
    labs = [lb for p in sorted(cases) if p in train for lb in cases[p][1]]
    step = TrainStep(net, "ce_dice", graph=True)
    loader, done = GpuLoader(SliceStore.from_arrays(ims, labs, device="cuda"), 12, drop_last=True), 0
    while done < a.train_steps:
        for batch in loader:
            step(batch["image"], batch["label"])
            done += 1
            if done == a.train_steps:
                break
    tmp = tempfile.mkdtemp(prefix="wsl4mis_test_step_")
    work = os.path.join(tmp, "work")
    os.makedirs(os.path.join(tmp, "model", "ACDC", "prof_fold1", "label"))
    os.makedirs(work)
    torch.save(net.state_dict(), os.path.join(tmp, "model", "ACDC", "prof_fold1", "label", "iter_60000.pth"))
    del net, step
    os.chdir(work)
    FLAGS = T.parser.parse_args(["--root_path", root, "--exp", "ACDC/prof", "--fold", "fold1", "--sup_type", "label"])
    image_list = [f"{p}_frame01.h5" for p in sorted(cases) if p in test]
    host_out = os.path.join(tmp, "host") + "/"
    os.makedirs(host_out)
    vox = int(sum(cases[c.split("_")[0]][1].size for c in image_list))
    res = {"device": device_info(), "volumes": len(image_list), "voxels": vox, "slices": int(sum(cases[c.split("_")[0]][1].shape[0]
                                                                                           for c in image_list)),
           "train_steps": done}
    wall(lambda: T.Inference(FLAGS))                 # warm-up: library load, executor buffers, original NIfTI files
    wall(lambda: host_loop(FLAGS, image_list[:2], host_out))
    g1, tg1 = wall(lambda: T.Inference(FLAGS))
    h, th = wall(lambda: host_loop(FLAGS, image_list, host_out))
    g2, tg2 = wall(lambda: T.Inference(FLAGS))
    res["fold_gpu_s"] = round(min(tg1, tg2), 3)
    res["fold_gpu_s_runs"] = [round(tg1, 3), round(tg2, 3)]
    res["fold_host_loop_s"] = round(th, 3)
    res["mean_dice_gpu"], res["mean_dice_host"] = float(g1), float(h)
    res["max_abs_diff_mean_dice"] = abs(float(g1) - float(h))
    # the GPU arm without its file writes: prediction + metrics only
    net = net_factory(net_type="unet", in_chns=1, class_num=4)
    net.load_state_dict(torch.load(T.checkpoint_path(FLAGS)))
    vols = [T._read_volume(root, c) for c in image_list]
    sps = [T.metric_spacing(nifti.read(T.original_path(c.replace(".h5", ""), root, v[0])).spacing) for c, v in zip(image_list, vols)]

    def predict_and_score():
        for (img, lab), sp in zip(vols, sps):
            pred = T.predict_volume(img, net)
            T.surface_metrics(pred, torch.from_numpy(lab).cuda(), 4, sp)

    predict_and_score()
    _, tp = wall(predict_and_score)
    res["fold_gpu_predict_and_metrics_s"] = round(tp, 3)
    # the 3 x volumes .nii.gz writes alone

    def write_all():
        for c, (img, lab) in zip(image_list, vols):
            hdr = nifti.read(T.original_path(c.replace(".h5", ""), root, img)).header
            for name, arr in (("_pred", lab), ("_img", img), ("_gt", lab)):
                nifti.write(host_out + c.replace(".h5", "") + name + ".nii.gz", arr.astype(np.float32), hdr)

    _, tw = wall(write_all)
    res["fold_nifti_read_write_s"] = round(tw, 3)
    res["cpu_cores"] = os.cpu_count()
    os.chdir(ROOT)
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
