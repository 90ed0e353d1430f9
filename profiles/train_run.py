"""Wall time of the native trainer (wsl4mis_b200/train.py) and of one validation pass, batched against per-volume.

    python profiles/train_run.py [--iters 3000] [--out results/train_run.json]

* trainer: pCE + GatedCRF and mean teacher at batch 12 on fold 1 of synthetic:100, `--iters` iterations each, validation every 200
  and logging included; the steady-state rate is taken between the validation points at 200 and `--iters` (the graphs are captured
  before 200), the total includes set-up and capture.
* validation: `ValidationSet.score` against the per-volume `val_2D.test_single_volume` loop, median of `--reps` passes each, on
  fold 1 of synthetic:100 (20 volumes) and on 20 volumes of ACDC's largest shape, 21 x 512 x 428.

Prints one JSON line with the device name and its power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:                     # pragma: no cover
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {type(e).__name__})"
    return q


def _trainer(script, iters):
    import wsl4mis_b200.train as TR
    marks = {}
    orig = TR.Trainer._validate

    def validate(self, iter_num, best):
        out = orig(self, iter_num, best)
        torch.cuda.synchronize()
        marks[iter_num] = time.perf_counter()
        return out
    TR.Trainer._validate = validate
    work = tempfile.mkdtemp(prefix="wsl4mis_train_run_")
    os.makedirs(os.path.join(work, "code"))
    cwd = os.getcwd()
    os.chdir(os.path.join(work, "code"))
    try:
        t0 = time.perf_counter()
        TR.train([script, "--root_path", "synthetic:100", "--exp", "prof/run", "--fold", "fold1", "--max_iterations", str(iters),
                  "--batch_size", "12"])
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        os.chdir(cwd)
        TR.Trainer._validate = orig
    steady = (marks[iters] - marks[200]) / (iters - 200)
    return {"script": script, "iterations": iters, "batch": 12, "total_s": round(total, 2),
            "ms_per_iteration_200_to_end": round(1e3 * steady, 3), "images_per_s": round(12 / steady, 1)}


def _median(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def _validation(reps):
    import wsl4mis_b200.val_2D as V
    from wsl4mis_b200.dataloaders.dataset import BaseDataSets
    from wsl4mis_b200.networks.net_factory import net_factory
    torch.manual_seed(0)
    net = net_factory("unet", 1, 4)
    out = {}
    db = BaseDataSets(base_dir="synthetic:100", fold="fold1", split="val")
    vols = [db._read(c) for c in db.sample_list]
    rs = np.random.RandomState(0)
    big = []
    for _ in range(20):                       # ACDC's largest shape; every class present in the label
        img = rs.rand(21, 512, 428).astype(np.float32)
        lab = np.zeros((21, 512, 428), np.uint8)
        lab[:, 100:400, 100:300] = 1
        lab[:, 150:350, 150:250] = 2
        lab[:, 200:300, 180:220] = 3
        big.append((img, lab))
    for name, data in (("synthetic:100 fold1", vols), ("20 x 21x512x428", big)):
        vset = V.ValidationSet.from_arrays([d[0] for d in data], [d[1] for d in data])
        batched = vset.score(net, 4)
        tb = _median(lambda: vset.score(net, 4), reps)
        tens = [(torch.from_numpy(np.asarray(i, np.float32))[None], torch.from_numpy(np.asarray(l))[None]) for i, l in data]
        per = [V.test_single_volume(i, l, net, 4) for i, l in tens]
        assert per == batched, "batched and per-volume validation disagree"
        tp = _median(lambda: [V.test_single_volume(i, l, net, 4) for i, l in tens], reps)
        out[name] = {"volumes": len(data), "batched_s": round(tb, 4), "per_volume_s": round(tp, 4), "speedup": round(tp / tb, 2)}
        del vset
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": _card(), "validation": _validation(a.reps),
           "trainer": [_trainer(s, a.iters) for s in ("train_weakly_supervised_pCE_GatedCRFLoss_2D.py", "train_mean_teacher_2D.py")],
           "run_py_unchanged_script": "not measured"}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
