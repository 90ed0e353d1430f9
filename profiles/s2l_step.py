"""Scribble2Label on one GPU: the captured step (train_s2l.py:119-157; UNet, bf16, graph=True) at batch 12 and 64 after thr_iter
(both CE terms), and the ensemble refresh (:214-243) over ~1 500 ACDC-shaped synthetic ragged slices -- batched per-sample-BatchNorm
forwards in chunks of 64 versus one slice per forward (the reference's batch-1 loop on the same kernels).  Prints one JSON line with
the times, the device name and its power limit.

    python profiles/s2l_step.py [--slices 1500] [--steps 50]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from wsl4mis_b200.dataloaders.dataset import S2LLoader, SliceStore  # noqa: E402
from wsl4mis_b200.engine import S2LStep  # noqa: E402
from wsl4mis_b200.networks.unet import UNet  # noqa: E402


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


def ragged_store(n, seed=0):
    rs = np.random.RandomState(seed)
    shapes = [(256, 216), (216, 256), (224, 154), (232, 256), (174, 208)]
    ims, labs, scrs = [], [], []
    for i in range(n):
        h, w = shapes[rs.randint(len(shapes))]
        ims.append(rs.rand(h, w).astype(np.float32))
        labs.append(rs.randint(0, 4, (h, w)).astype(np.uint8))
        scrs.append(np.where(rs.rand(h, w) < 0.03, labs[-1], 4).astype(np.uint8))
    return SliceStore.from_arrays(ims, labs, device="cuda", scribbles=scrs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", type=int, default=1500)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--precision", default="bf16")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/s2l_step.py measures on a GPU"
    torch.manual_seed(0)
    store = ragged_store(a.slices)
    store.weight_live.uniform_(0.0, 1.0)
    res = {"device": device_info(), "precision": a.precision, "slices": a.slices}
    for B in (12, 64):
        step = S2LStep(UNet(1, 4).cuda().set_precision(a.precision), thr_iter=0, graph=True)
        batch = next(iter(S2LLoader(store, B, drop_last=True)))
        args = (batch["image"], batch["scribble"], batch["weight"])
        for _ in range(5):
            step(*args)
        res[f"step_ms_b{B}"] = round(timed(lambda: step(*args), a.steps), 3)
        res[f"images_per_s_b{B}"] = round(B * 1000.0 / res[f"step_ms_b{B}"], 1)
    model = UNet(1, 4).cuda().set_precision(a.precision)
    step = S2LStep(model, graph=False)
    for chunk, key in ((64, "refresh_ms_batched64"), (1, "refresh_ms_batch1_loop")):
        step.refresh(store, chunk=chunk)                 # warm-up: buffers for this shape
        res[key] = round(timed(lambda: step.refresh(store, chunk=chunk), 2), 1)
    res["refresh_speedup"] = round(res["refresh_ms_batch1_loop"] / res["refresh_ms_batched64"], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
