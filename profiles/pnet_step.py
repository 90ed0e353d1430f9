"""PNet2D (net_factory('pnet'), bf16) on one GPU: the captured training steps against the eager autograd module path.

At the recipes' batches -- 12 for TrainStep('pce') (train_weakly_supervised_pCE_2D.py with --batch_size 12) and 12 + 12 for UAMTStep
(train_uncertainty_aware_mean_teacher_2D.py's two streams at --batch_size 24) -- per-iteration time of the graph-captured fused step
and of the module path the way tests/test_gpu_pnet.py::test_pnet_step_time_at_256 times it (m(x), CrossEntropyLoss(ignore_index=4),
torch.optim.SGD; for UAMT the script's body: two student forwards, five no-grad teacher forwards on noisy inputs, CE + Dice and the
uncertainty-masked consistency), timed in alternating windows with CUDA events.  Also the peak device memory of one resident
validation pass at chunk 64.  Prints one JSON line with the device name and its power limit read in the same run.

    python profiles/pnet_step.py [--steps 10] [--reps 3]
"""
import argparse
import gc
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from wsl4mis_b200.engine import TrainStep, UAMTStep  # noqa: E402
from wsl4mis_b200.networks.net_factory import net_factory  # noqa: E402
from wsl4mis_b200.utils import losses, ramps  # noqa: E402


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                       # pragma: no cover - informational only
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {type(e).__name__})"
    return q


def timed(fn, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def batch(n, seed, dense=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 1, 256, 256, generator=g)
    y = torch.randint(0, 4, (n, 256, 256), generator=g, dtype=torch.uint8)
    if not dense:
        y = torch.where(torch.rand(n, 256, 256, generator=g) < 0.05, y, torch.full_like(y, 4))
    return x.cuda(), y.cuda()


def pce_bodies(B):
    x, y = batch(B, 1)
    torch.manual_seed(0)
    fused = TrainStep(net_factory("pnet", 1, 4), "pce", graph=True)
    torch.manual_seed(0)
    m = net_factory("pnet", 1, 4)
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    ce = torch.nn.CrossEntropyLoss(ignore_index=4)
    m.train()

    def module():
        loss = ce(m(x), y.long())
        opt.zero_grad()
        loss.backward()
        opt.step()
    return {"captured": lambda: fused(x, y), "module": module}, fused


def uamt_bodies(B):
    x_l, y_l = batch(B, 2, dense=True)
    x_u, _ = batch(B, 3)
    torch.manual_seed(0)
    fused = UAMTStep(net_factory("pnet", 1, 4), net_factory("pnet", 1, 4), graph=True)
    torch.manual_seed(0)
    s, t = net_factory("pnet", 1, 4), net_factory("pnet", 1, 4)
    for p in t.parameters():
        p.detach_()
    opt = torch.optim.SGD(s.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    dice = losses.DiceLoss(4)
    state = {"it": 0}

    def module():
        s.train()
        t.train()
        out_l, out_u = s(x_l), s(x_u)
        with torch.no_grad():
            ema = t(x_u + torch.clamp(torch.randn_like(x_u) * 0.1, -0.2, 0.2))
            rep = x_u.repeat(2, 1, 1, 1)
            preds = torch.cat([t(rep + torch.clamp(torch.randn_like(rep) * 0.1, -0.2, 0.2)) for _ in range(4)], 0)
            preds = F.softmax(preds, 1).reshape(8, B, 4, 256, 256).mean(0)
            unc = -(preds * torch.log(preds + 1e-6)).sum(1, keepdim=True)
        sup = 0.5 * (dice(torch.softmax(out_l, 1), y_l.unsqueeze(1)) + F.cross_entropy(out_l, y_l.long()))
        w = 0.1 * ramps.sigmoid_rampup(state["it"] // 300, 200.0)
        thr = (0.75 + 0.25 * ramps.sigmoid_rampup(state["it"], 30000)) * math.log(2)
        mask = (unc < thr).float()
        dist = (torch.softmax(out_u, 1) - torch.softmax(ema, 1)) ** 2
        loss = sup + w * (mask * dist).sum() / (2 * mask.sum() + 1e-16)
        opt.zero_grad()
        loss.backward()
        opt.step()
        state["it"] += 1
    return {"captured": lambda: fused(x_l, y_l, x_u), "module": module}, fused


def measure(bodies, steps, reps):
    for fn in bodies.values():                   # warm-up: graph capture, allocator, module loading
        for _ in range(3):
            fn()
    ms = {k: [] for k in bodies}
    for _ in range(reps):
        for k, fn in bodies.items():
            ms[k].append(timed(fn, steps))
    return {k: round(statistics.median(v), 2) for k, v in ms.items()}, {k: round(max(v) - min(v), 2) for k, v in ms.items()}


def validation_peak():
    from wsl4mis_b200 import val_2D
    rs = np.random.RandomState(5)
    shapes = [(40, 220, 200)] * 3
    vs = val_2D.ValidationSet.from_arrays([rs.rand(*s).astype(np.float32) for s in shapes],
                                          [rs.randint(0, 4, s).astype(np.uint8) for s in shapes])
    net = net_factory("pnet", 1, 4)
    gc.collect()                    # the timed steps' networks and executors reference each other
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    vs.score(net, 4)
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), vs.chunk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    out = {"device": device_info()}
    for name, make, B in (("pce", pce_bodies, 12), ("uamt", uamt_bodies, 12)):
        bodies, fused = make(B)
        med, spread = measure(bodies, a.steps, a.reps)
        out[name] = {"batch": B if name == "pce" else f"{B}+{B}", "ms_per_iteration": med, "spread_ms": spread,
                     "speedup": round(med["module"] / med["captured"], 2), "fused_launches_per_step": fused.launches_per_step}
        del bodies, fused
        gc.collect()
        torch.cuda.empty_cache()
    peak, chunk = validation_peak()
    out["validation_peak_GiB"] = {"chunk": chunk, "peak_allocated": peak}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
