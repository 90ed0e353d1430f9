"""Validation-pass cost on one GPU: val_2D.test_single_volume over the fold-1 validation volumes of synthetic:100 (UNet, bf16) with
HD95 on the GPU (wsl4mis_b200.metric.surface_metrics), after --train-steps captured ce_dice steps (batch 12) so that the
predictions have the shape of a real run's, against the same predictions scored by the host calculate_metric_percase
(scipy distance transforms); the metric alone per volume with CUDA events; and the largest ACDC case, a 21x512x428 volume at
spacing (10, 1.5625, 1.5625), on the GPU and with scipy; and at that shape the layout that costs the outward distance scans the
most: a one-voxel gt line along x in the first slice (features in every x-plane, none within reach of most voxels along y), scored
against a full prediction.  Prints one JSON line with the numbers, the device name and its power
limit.

    python profiles/val_metrics.py [--patients 100] [--reps 20] [--train-steps 400]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _metric_oracle as M  # noqa: E402
from s2l_step import device_info  # noqa: E402
from wsl4mis_b200 import val_2D  # noqa: E402
from wsl4mis_b200.dataloaders.dataset import GpuLoader, SliceStore, fold_ids, synthetic_acdc  # noqa: E402
from wsl4mis_b200.engine import TrainStep  # noqa: E402
from wsl4mis_b200.metric import surface_metrics  # noqa: E402
from wsl4mis_b200.networks.unet import UNet  # noqa: E402


def host_pass(vols, net):
    out = []
    for img, lab in vols:
        pred = val_2D._predict_volume(img, net, [256, 256], 0).cpu().numpy()
        out.append([val_2D.calculate_metric_percase(pred == i, lab == i) for i in range(1, 4)])
    return out


def gpu_pass(vols, net):
    return [val_2D.test_single_volume(torch.from_numpy(img)[None], torch.from_numpy(lab)[None], net, 4) for img, lab in vols]


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def largest_case():
    """ACDC's largest volume shape with three nested classes and a shifted, resized prediction."""
    S, H, W = 21, 512, 428
    z, y, x = np.mgrid[:S, :H, :W].astype(np.float32)
    gt = np.zeros((S, H, W), np.uint8)
    pred = np.zeros_like(gt)
    for c, r in ((1, 90.0), (2, 60.0), (3, 35.0)):
        rr = r * (1.0 - np.abs(z - S / 2) / S)
        gt[(y - 250) ** 2 + (x - 210) ** 2 < rr ** 2] = c
        pred[(y - 254) ** 2 + ((x - 207) * 1.05) ** 2 < (rr * 1.03) ** 2] = c
    return pred, gt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patients", type=int, default=100)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--train-steps", type=int, default=400)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/val_metrics.py measures on a GPU"
    cases = synthetic_acdc(a.patients)
    train, val = fold_ids("fold1")
    vols = [(cases[p][0], cases[p][1]) for p in sorted(cases) if p in val]
    torch.manual_seed(0)
    net = UNet(1, 4).cuda()                      # bf16 (the default execution mode)
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
    res = {"device": device_info(), "volumes": len(vols), "voxels": int(sum(v[1].size for v in vols)), "train_steps": done}
    gpu_pass(vols[:2], net)                      # warm-up: library load, allocator, every kernel
    host_pass(vols[:2], net)
    g1, tg1 = wall(lambda: gpu_pass(vols, net))
    h, th = wall(lambda: host_pass(vols, net))
    g2, tg2 = wall(lambda: gpu_pass(vols, net))
    res["val_pass_gpu_metric_s"] = round(min(tg1, tg2), 4)
    res["val_pass_gpu_metric_s_runs"] = [round(tg1, 4), round(tg2, 4)]
    res["val_pass_host_metric_s"] = round(th, 4)
    res["same_results"] = bool(g1 == h and g2 == h)
    res["empty_predictions"] = int(sum(d == (0, 0) for r in h for d in r))
    # the metric alone: one surface_metrics call per volume (kernels + the result copy), CUDA events
    preds = [val_2D._predict_volume(img, net, [256, 256], 0) for img, _ in vols]
    gts = [torch.from_numpy(lab).cuda() for _, lab in vols]
    for p, g in zip(preds, gts):
        surface_metrics(p, g, 4)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(a.reps):
        for p, g in zip(preds, gts):
            surface_metrics(p, g, 4)
    e.record()
    torch.cuda.synchronize()
    res["metric_ms_per_volume_gpu"] = round(s.elapsed_time(e) / (a.reps * len(vols)), 3)
    t0 = time.perf_counter()
    for p, g in zip(preds, gts):
        ph, gh = p.cpu().numpy(), g.cpu().numpy()
        for i in range(1, 4):
            if (ph == i).any():
                val_2D.hd95(ph == i, gh == i)
    res["metric_ms_per_volume_host"] = round((time.perf_counter() - t0) * 1000 / len(vols), 1)
    # the largest ACDC volume with its voxel spacing
    sp = (10.0, 1.5625, 1.5625)
    pred, gt = largest_case()
    tp, tgt = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    surface_metrics(tp, tgt, 4, sp)
    s.record()
    for _ in range(5):
        big = surface_metrics(tp, tgt, 4, sp)
    e.record()
    torch.cuda.synchronize()
    res["largest_shape"] = list(pred.shape)
    res["largest_metric_ms_gpu"] = round(s.elapsed_time(e) / 5, 2)
    t0 = time.perf_counter()
    ref = [(M.hd95(pred == i, gt == i, sp), M.asd(pred == i, gt == i, sp)) for i in range(1, 4)]
    res["largest_metric_s_host_scipy"] = round(time.perf_counter() - t0, 2)
    res["largest_max_rel_diff"] = max(abs(r.hd95 - h_) / h_ + abs(r.asd - a_) / a_ for r, (h_, a_) in zip(big, ref))
    # the slow layout of the y scan: every voxel scans O(H) rows
    line = np.zeros_like(gt)
    line[0, 0, :] = 1
    full = np.ones_like(gt)
    tl, tf = torch.from_numpy(line).cuda(), torch.from_numpy(full).cuda()
    surface_metrics(tf, tl, 2, sp)
    s.record()
    for _ in range(3):
        adv = surface_metrics(tf, tl, 2, sp)[0]
    e.record()
    torch.cuda.synchronize()
    res["line_metric_ms_gpu"] = round(s.elapsed_time(e) / 3, 2)
    t0 = time.perf_counter()
    ref_h, ref_a = M.hd95(full, line, sp), M.asd(full, line, sp)
    res["line_metric_s_host_scipy"] = round(time.perf_counter() - t0, 2)
    res["line_max_rel_diff"] = abs(adv.hd95 - ref_h) / ref_h + abs(adv.asd - ref_a) / ref_a
    res["cpu_cores"] = os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
