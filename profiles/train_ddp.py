"""Data-parallel scaling of the native trainer (wsl4mis_b200/train.py) and of the Scribble2Label refresh, at W = 1, 2, 4, 8 ranks
(as many as the box has GPUs), one process per GPU over NCCL as torchrun starts them.

    python profiles/train_ddp.py [--iters 400] [--out results/train_ddp.json]

* trainer: BASELINE config 3 (train_weakly_supervised_segmentation_pCE_ours_proposed.py, DMPLS, unet_cct, global batch 128) and
  config 5 (train_uncertainty_aware_mean_teacher_2D.py, UAMT, global batch 256) on fold 1 of synthetic:100, `--iters` iterations,
  validation and logging included.  The steady-state rate is taken on rank 0 between the validation points at 200 and `--iters`
  (every batch shape is captured before 200; the other ranks meet rank 0 at every step's all-reduce); images/s counts the global
  batch, and the scaling factor is images/s over the W = 1 run's.
* refresh: one `S2LStep.refresh` over fold 1's 626 training slices of synthetic:100 (chunks of 64), median of three after a warm-up
  pass, in one process and split over the most ranks the box has.

Prints one JSON line with the device name and its power limit read in the same run.
"""
import argparse
import json
import os
import socket
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

CONFIGS = (("config3_dmpls", "train_weakly_supervised_segmentation_pCE_ours_proposed.py", 128),
           ("config5_uamt", "train_uncertainty_aware_mean_teacher_2D.py", 256))


def _port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _env(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))


def _trainer_worker(rank, world, port, script, bs, iters, out):
    _env(rank, world, port)
    import wsl4mis_b200.train as TR
    marks = {}
    orig = TR.Trainer._validate

    def validate(self, iter_num, best):
        res = orig(self, iter_num, best)
        torch.cuda.synchronize()
        marks[iter_num] = time.perf_counter()
        return res
    TR.Trainer._validate = validate
    work = tempfile.mkdtemp(prefix="wsl4mis_train_ddp_")
    os.makedirs(os.path.join(work, "code"))
    os.chdir(os.path.join(work, "code"))
    TR.train([script, "--root_path", "synthetic:100", "--exp", "prof/ddp", "--fold", "fold1", "--max_iterations", str(iters),
              "--batch_size", str(bs)])
    if rank == 0:
        dt = marks[iters] - marks[200]
        with open(out, "w") as f:
            json.dump({"ms_per_iter": round(1e3 * dt / (iters - 200), 3), "images_per_s": round(bs * (iters - 200) / dt, 1)}, f)


def _refresh_worker(rank, world, port, out):
    import torch.distributed as dist
    _env(rank, world, port)
    torch.cuda.set_device(rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from wsl4mis_b200.dataloaders.dataset import BaseDataSets_s2l
        from wsl4mis_b200.engine import S2LStep
        from wsl4mis_b200.networks.unet import UNet
        torch.manual_seed(2022)
        step = S2LStep(UNet(1, 4).cuda(), world_size=world)
        store = BaseDataSets_s2l(base_dir="synthetic:100", fold="fold1").to_slice_store()
        times = []
        for rep in range(4):
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            step.refresh(store, alpha=0.2)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        if rank == 0:
            with open(out, "w") as f:
                json.dump({"slices": len(store), "ms": round(1e3 * sorted(times[1:])[1], 2)}, f)
    finally:
        if world > 1:
            dist.destroy_process_group()


def _spawn(fn, world, *args):
    import torch.multiprocessing as mp
    out = tempfile.mktemp(suffix=".json")
    mp.spawn(fn, args=(world, _port()) + args + (out,), nprocs=world, join=True)
    with open(out) as f:
        return json.load(f)


def main():
    from train_run import _card
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert a.iters > 200 and torch.cuda.is_available(), "needs a GPU and --iters > 200"
    gpus = torch.cuda.device_count()
    worlds = [w for w in (1, 2, 4, 8) if w <= gpus]
    res = {"device": _card(), "gpus": gpus, "iters": a.iters, "root": "synthetic:100 fold1", "trainer": {}, "refresh": {}}
    for name, script, bs in CONFIGS:
        rows = {}
        for w in worlds:
            rows[w] = _spawn(_trainer_worker, w, script, bs, a.iters)
            rows[w]["scaling"] = round(rows[w]["images_per_s"] / rows[1]["images_per_s"], 3)
        res["trainer"][name] = {"global_batch": bs, "by_world_size": rows}
    res["refresh"]["one_process"] = _spawn(_refresh_worker, 1)
    if worlds[-1] > 1:
        res["refresh"][f"{worlds[-1]}_ranks"] = _spawn(_refresh_worker, worlds[-1])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
