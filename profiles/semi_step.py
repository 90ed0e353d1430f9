"""Mean teacher (train_mean_teacher_2D.py:138-180) and entropy minimisation (train_entropy_minimization_2D.py:121-150) on one GPU.

At 6 + 6 (the scripts' default --batch_size 12) and 32 + 32, per-iteration time of three bodies on the same UNet modules (bf16),
timed in alternating windows: the script's autograd body (model(x_l), model(x_u), torch softmax / CrossEntropyLoss / DiceLoss /
entropy_loss, torch.optim.SGD with the poly LR), the eager fused step and the graph-captured fused step; and the launches the fused
step issues per iteration.  Then three synthetic epochs of the two-stream loop zip(cycle(labelled), unlabelled) at 6 + 6 in graph
mode, short last batches included: per epoch the iterations, time and graphs held (a shape is captured on its third occurrence),
and the device memory the short shapes' graphs and buffers add.
Prints one JSON line with the device name and its power limit read in the same run.

    python profiles/semi_step.py [--steps 20] [--reps 5] [--data synthetic:100]
"""
import argparse
import itertools
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from wsl4mis_b200.dataloaders.dataset import GpuLoader  # noqa: E402
from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets  # noqa: E402
from wsl4mis_b200.engine import EntropyMinStep, MeanTeacherStep  # noqa: E402
from wsl4mis_b200.networks.unet import UNet  # noqa: E402
from wsl4mis_b200.utils import losses, ramps  # noqa: E402


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                       # pragma: no cover - informational only
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {type(e).__name__})"
    return q


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def make_step(method, graph, precision):
    torch.manual_seed(0)
    s = UNet(1, 4).cuda().set_precision(precision)
    if method == "mt":
        return MeanTeacherStep(s, UNet(1, 4).cuda().set_precision(precision), graph=graph)
    return EntropyMinStep(s, graph=graph)


class ScriptBody:
    """the script's step body through autograd on the package's modules, as the unchanged script runs it"""

    def __init__(self, method, precision, base_lr=0.01, max_iterations=30000):
        torch.manual_seed(0)
        self.method, self.base_lr, self.max_iterations = method, base_lr, max_iterations
        self.model = UNet(1, 4).cuda().set_precision(precision)
        self.ema_model = UNet(1, 4).cuda().set_precision(precision) if method == "mt" else None
        self.opt = torch.optim.SGD(self.model.parameters(), lr=base_lr, momentum=0.9, weight_decay=0.0001)
        self.ce_loss, self.dice_loss = torch.nn.CrossEntropyLoss(), losses.DiceLoss(4)
        self.iter_num = 0

    def __call__(self, volume_batch, label_batch, unlabeled_volume_batch):
        if self.method == "mt":
            noise = torch.clamp(torch.randn_like(unlabeled_volume_batch) * 0.1, -0.2, 0.2)
            ema_inputs = unlabeled_volume_batch + noise
        outputs = self.model(volume_batch)
        outputs_soft = torch.softmax(outputs, dim=1)
        outputs_unlabeled = self.model(unlabeled_volume_batch)
        outputs_unlabeled_soft = torch.softmax(outputs_unlabeled, dim=1)
        loss_ce = self.ce_loss(outputs, label_batch[:].long())
        loss_dice = self.dice_loss(outputs_soft, label_batch.unsqueeze(1))
        supervised_loss = 0.5 * (loss_dice + loss_ce)
        consistency_weight = 0.1 * ramps.sigmoid_rampup(self.iter_num // 300, 200.0)
        if self.method == "mt":
            with torch.no_grad():
                ema_output_soft = torch.softmax(self.ema_model(ema_inputs), dim=1)
            consistency_loss = torch.mean((outputs_unlabeled_soft - ema_output_soft) ** 2)
        else:
            consistency_loss = losses.entropy_loss(outputs_unlabeled_soft, C=4)
        loss = supervised_loss + consistency_weight * consistency_loss
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        lr_ = self.base_lr * (1.0 - self.iter_num / self.max_iterations) ** 0.9
        for param_group in self.opt.param_groups:
            param_group["lr"] = lr_
        self.iter_num += 1
        return loss


def step_times(method, B, a):
    x = torch.rand(2 * B, 1, 256, 256, device="cuda")
    y = torch.randint(0, 4, (B, 256, 256), device="cuda", dtype=torch.uint8)
    args = (x[:B], y, x[B:])
    bodies = {"autograd_script": ScriptBody(method, a.precision), "eager_step": make_step(method, False, a.precision),
              "graph_step": make_step(method, True, a.precision)}
    for fn in bodies.values():
        for _ in range(3):                      # graph step: two eager warm-up steps, then the capture
            fn(*args)
    ms = {k: [] for k in bodies}
    for _ in range(a.reps):                     # alternate the three bodies, window by window
        for k, fn in bodies.items():
            ms[k].append(timed(lambda: fn(*args), a.steps))
    res = {f"{k}_ms": round(statistics.median(v), 3) for k, v in ms.items()}
    res.update({f"{k}_ms_spread": [round(min(v), 3), round(max(v), 3)] for k, v in ms.items()})
    res["launches_per_step"] = bodies["eager_step"].launches_per_step
    res["graph_speedup_vs_autograd"] = round(res["autograd_script_ms"] / res["graph_step_ms"], 2)
    res["graph_speedup_vs_eager"] = round(res["eager_step_ms"] / res["graph_step_ms"], 2)
    del bodies
    torch.cuda.empty_cache()
    return res


def epochs(method, a, n_epochs=3):
    """epochs of zip(cycle(GpuLoader(labelled, 6)), GpuLoader(unlabelled, 6)) in graph mode, after the full-shape graph exists"""
    torch.manual_seed(1)
    L = BaseDataSets(base_dir=a.data, labeled_type="labeled", fold="fold1", split="train").to_slice_store()
    U = BaseDataSets(base_dir=a.data, labeled_type="unlabeled", fold="fold1", split="train").to_slice_store()
    loader_l, loader_u = GpuLoader(L, 6), GpuLoader(U, 6)
    step = make_step(method, True, a.precision)
    b = next(iter(loader_l))
    for _ in range(3):                          # the full 6 + 6 shape: warm-up and capture
        step(b["image"], b["label"], b["image"])
    torch.cuda.synchronize()
    alloc0, reserved0 = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
    shapes, per_epoch = set(), []
    for _ in range(n_epochs):
        n, t0 = 0, time.perf_counter()
        for bl, bu in zip(itertools.cycle(loader_l), loader_u):
            shapes.add((bl["image"].shape[0], bu["image"].shape[0]))
            step(bl["image"], bl["label"], bu["image"])
            n += 1
        torch.cuda.synchronize()
        per_epoch.append({"iterations": n, "seconds": round(time.perf_counter() - t0, 3), "graphs": len(step._graphs)})
    extra = len(step._graphs) - 1
    d_alloc, d_res = torch.cuda.memory_allocated() - alloc0, torch.cuda.memory_reserved() - reserved0
    return {"labelled_batches": len(loader_l), "unlabelled_batches": len(loader_u), "batch_shapes": sorted(shapes),
            "epochs": per_epoch, "extra_allocated_mib": round(d_alloc / 2**20, 1), "extra_reserved_mib": round(d_res / 2**20, 1),
            "extra_reserved_mib_per_extra_shape": round(d_res / 2**20 / max(extra, 1), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--data", default="synthetic:100")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/semi_step.py measures on a GPU"
    res = {"device": device_info(), "precision": a.precision, "steps_per_window": a.steps, "windows": a.reps}
    for method in ("mt", "em"):
        for B in (6, 32):
            res[f"{method}_b{B}+{B}"] = step_times(method, B, a)
        res[f"{method}_epochs"] = epochs(method, a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
