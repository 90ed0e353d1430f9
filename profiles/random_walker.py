"""pCE + Random Walker on one GPU: the batched random-walker pseudo labels (wsl_random_walker) for every fold-1 training slice of
synthetic:100 with thin line (arc) scribbles -- GPU wall time, iteration counts -- against scipy's spsolve of the same system per
slice on the host (oracle/rw_oracle.py, a sample of slices), and the captured ce_dice step (train_fully_supervised_2D.py:97-105;
UNet, bf16, graph=True) at batch 12 and 64.  Prints one JSON line with the numbers, the device name and its power limit.

    python profiles/random_walker.py [--patients 100] [--cpu-sample 6] [--steps 50]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from s2l_step import device_info, timed  # noqa: E402
from wsl4mis_b200.dataloaders import random_walker_labels  # noqa: E402
from wsl4mis_b200.dataloaders.dataset import GpuLoader, SliceStore, fold_ids, synthetic_acdc  # noqa: E402
from wsl4mis_b200.engine import TrainStep  # noqa: E402
from wsl4mis_b200.networks.unet import UNet  # noqa: E402


def arcs(lab, rs):
    """one-pixel arcs over ~90 degrees of each class's median radius (few seeds: the slow case for the solver)"""
    scr = np.full(lab.shape, 4, np.uint8)
    for c in range(4):
        ys, xs = np.nonzero(lab == c)
        if len(ys) == 0:
            continue
        cy, cx = ys.mean(), xs.mean()
        rr = np.sqrt((ys - cy) ** 2 + (xs - cx) ** 2)
        ang = np.arctan2(ys - cy, xs - cx)
        sel = (np.abs(rr - np.median(rr)) < 0.5) & (((ang - rs.rand() * 2 * np.pi) % (2 * np.pi)) < 1.6)
        scr[ys[sel], xs[sel]] = c
    return scr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patients", type=int, default=100)
    ap.add_argument("--cpu-sample", type=int, default=6)
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/random_walker.py measures on a GPU"
    cases = synthetic_acdc(a.patients)
    train, _ = fold_ids("fold1")
    rs = np.random.RandomState(0)
    ims, scrs, labs = [], [], []
    for pid in sorted(cases):
        if pid not in train:
            continue
        img, lab, _ = cases[pid]
        for z in range(img.shape[0]):
            ims.append(img[z])
            labs.append(lab[z])
            scrs.append(arcs(lab[z], rs))
    res = {"device": device_info(), "slices": len(ims), "pixels": int(sum(im.size for im in ims))}
    store = SliceStore.from_arrays(ims, labs, device="cuda", scribbles=scrs)
    random_walker_labels(store)                                  # warm-up (library load, allocator)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out, st = random_walker_labels(store)
    torch.cuda.synchronize()
    res["gpu_wall_s_all_slices"] = round(time.perf_counter() - t0, 3)
    it = np.asarray(st["iters"])
    res["iters_mean"], res["iters_max"], res["iters_min"] = round(float(it.mean()), 1), int(it.max()), int(it.min())
    res["resid_max"] = float(np.max(st["resid"]))
    import rw_oracle as R
    pick = np.linspace(0, len(ims) - 1, a.cpu_sample).astype(int)
    t0 = time.perf_counter()
    for i in pick:
        R.random_walker(ims[i], scrs[i])
    res["cpu_spsolve_s_per_slice"] = round((time.perf_counter() - t0) / len(pick), 3)
    res["cpu_sample_slices"] = len(pick)
    res["cpu_cores"] = os.cpu_count()
    res["cpu_note"] = "scipy spsolve (SuperLU, one core) of the fp64 system, 4 right-hand sides, including matrix assembly"
    res["cpu_estimate_s_all_slices"] = round(res["cpu_spsolve_s_per_slice"] * len(ims), 1)
    for B in (12, 64):
        step = TrainStep(UNet(1, 4).cuda(), "ce_dice", graph=True)
        batch = next(iter(GpuLoader(out, B, drop_last=True)))
        for _ in range(5):
            step(batch["image"], batch["label"])
        res[f"ce_dice_step_ms_b{B}"] = round(timed(lambda: step(batch["image"], batch["label"]), a.steps), 3)
        res[f"ce_dice_images_per_s_b{B}"] = round(B * 1000.0 / res[f"ce_dice_step_ms_b{B}"], 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
