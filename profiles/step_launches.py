"""The C-ABI launch sequence of every training step class, for comparing two versions of the step code.

Each configuration builds its models from fixed seeds, runs two eager steps at iterations where the ramps are non-zero, and keeps
every launch in order as (entry point, scalar arguments, names of the pointer arguments passed as NULL).  Pointer values are left
out, so two versions that allocate their buffers differently give the same trace.  The configurations:
  - every TrainStep variant on UNet and UNet_CCT (dmpls on UNet_CCT only), in bf16 and fp32;
  - S2LStep before and after thr_iter;
  - UAMTStep, MeanTeacherStep and EntropyMinStep with a full and a short unlabelled batch;
  - USTMStep with rot90 counts 0-3;
  - DANStep at 256 x 256 with a full and a short unlabelled batch.
Each configuration also records the step's `segments`, `n_trained` and `launches_per_step`, and a separate table records
`segments` and `n_trained` of every step class on UNet, UNet_CCT, UNet_DS, UNet_CCT_3H and PNet2D (or the error a construction
raises).  Writes one JSON file; two such files from two versions should be equal.

    python profiles/step_launches.py --out /tmp/launches.json
"""
import argparse
import ctypes
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from wsl4mis_b200 import _lib  # noqa: E402
from wsl4mis_b200.engine import (DANStep, EntropyMinStep, MeanTeacherStep, S2LStep, TrainStep, UAMTStep, USTMStep,  # noqa: E402
                                 VARIANTS)
from wsl4mis_b200.networks.discriminator import FCDiscriminator  # noqa: E402
from wsl4mis_b200.networks.pnet import PNet2D  # noqa: E402
from wsl4mis_b200.networks.unet import UNet, UNet_CCT, UNet_CCT_3H, UNet_DS  # noqa: E402

DEV = torch.device("cuda", 0)
MODELS = {"unet": lambda: UNet(1, 4), "unet_cct": lambda: UNet_CCT(1, 4), "unet_ds": lambda: UNet_DS(1, 4),
          "unet_cct_3h": lambda: UNet_CCT_3H(1, 4), "pnet": lambda: PNet2D(1, 4, 64, [1, 2, 4, 8, 16])}


class OrderedRecorder:
    """Stands in for _lib.PROFILE: runs every C-ABI call as call() does (a nonzero return code raises) and appends it to `trace`."""

    def __init__(self):
        self.trace = []

    def record(self, name, fn, vals):
        rc = fn(*vals)
        if rc != 0:
            raise RuntimeError(f"{name} failed ({rc}): {_lib.LIB.last_error()}")
        args = [(nm, ty, v) for (ty, nm), v in zip(_lib.LIB.protos[name][1], vals) if nm != "stream"]
        scalars = [[nm, v if isinstance(v, (int, float)) else repr(v)] for nm, ty, v in args if ty is not ctypes.c_void_p]
        nulls = [nm for nm, ty, v in args if ty is ctypes.c_void_p and v is None]
        self.trace.append([name, scalars, nulls])


def batch(B, hw, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(B, 1, hw, hw, generator=g)
    lab = torch.randint(0, 4, (B, hw, hw), generator=g, dtype=torch.uint8)
    return img.to(DEV), lab.to(DEV)


def scribbles(lab, seed):
    """keep ~10 % of the labels, the rest unlabelled (4)"""
    g = torch.Generator().manual_seed(seed)
    keep = (torch.rand(tuple(lab.shape), generator=g) < 0.1).to(DEV)
    return torch.where(keep, lab, torch.full_like(lab, 4))


def record(step, calls):
    rec = OrderedRecorder()
    _lib.PROFILE = rec
    try:
        for args, kw in calls:
            step(*args, **kw)
        torch.cuda.synchronize()
    finally:
        _lib.PROFILE = None
    return {"trace": rec.trace, "segments": [list(s) for s in step.segments], "n_trained": step.n_trained,
            "launches_per_step": step.launches_per_step}


def configurations():
    """name -> () -> (step, [(args, kwargs) per step])"""
    cfg = {}
    for model in ("unet", "unet_cct"):
        for variant in VARIANTS:
            if variant == "dmpls" and model == "unet":
                continue
            for prec in ("bf16", "fp32"):
                def make(model=model, variant=variant, prec=prec):
                    torch.manual_seed(11)
                    random.seed(12)
                    step = TrainStep(MODELS[model]().to(DEV).set_precision(prec), variant, graph=False)
                    step.iter_num = 900
                    img, lab = batch(2, 32, 13)
                    return step, [((img, scribbles(lab, 14)), {})] * 2
                cfg[f"train/{model}/{variant}/{prec}"] = make
    for phase, it in (("before", 0), ("after", 10)):
        def make(it=it):
            torch.manual_seed(15)
            step = S2LStep(UNet(1, 4).to(DEV), thr_iter=5, graph=False)
            step.iter_num = it
            img, lab = batch(2, 32, 16)
            weight = torch.softmax(torch.rand(2, 32, 32, 4, generator=torch.Generator().manual_seed(17)), -1).to(DEV)
            return step, [((img, scribbles(lab, 18), weight), {})] * 2
        cfg[f"s2l/{phase}_thr_iter"] = make
    for method in ("uamt", "mt", "em"):
        for bu in (2, 1):
            def make(method=method, bu=bu):
                torch.manual_seed(19)
                s = UNet(1, 4).to(DEV)
                if method == "em":
                    step = EntropyMinStep(s)
                else:
                    step = (UAMTStep if method == "uamt" else MeanTeacherStep)(s, UNet(1, 4).to(DEV))
                step.iter_num = 900
                img_l, lab_l = batch(2, 32, 20)
                img_u, _ = batch(bu, 32, 21)
                return step, [((img_l, lab_l, img_u), {})] * 2
            cfg[f"{method}/bu{bu}"] = make
    for k in range(4):
        def make(k=k):
            torch.manual_seed(22)
            step = USTMStep(UNet(1, 4).to(DEV), UNet(1, 4).to(DEV))
            step.iter_num = 5000
            img, lab = batch(2, 32, 23)
            return step, [((img, scribbles(lab, 24)), {"rot_times": k})] * 2
        cfg[f"ustm/rot{k}"] = make
    for bu in (2, 1):
        def make(bu=bu):
            torch.manual_seed(25)
            step = DANStep(UNet(1, 4).to(DEV), FCDiscriminator(4).to(DEV), graph=False)
            step.iter_num = 900
            img_l, lab_l = batch(2, 256, 26)
            img_u, _ = batch(bu, 256, 27)
            return step, [((img_l, lab_l, img_u), {})] * 2
        cfg[f"dan/bu{bu}"] = make
    return cfg


def segment_table():
    """(step, model) -> {segments, n_trained} or the error its construction raises"""
    ctors = {f"train/{v}": (lambda m, t, v=v: TrainStep(m, v, graph=False)) for v in VARIANTS}
    ctors.update({
        "s2l": lambda m, t: S2LStep(m, graph=False),
        "uamt": lambda m, t: UAMTStep(m, t),
        "mt": lambda m, t: MeanTeacherStep(m, t),
        "em": lambda m, t: EntropyMinStep(m),
        "ustm": lambda m, t: USTMStep(m, t),
        "dan": lambda m, t: DANStep(m, FCDiscriminator(4).to(DEV)),
    })
    out = {}
    for sname, ctor in ctors.items():
        for mname, mk in MODELS.items():
            torch.manual_seed(0)
            try:
                step = ctor(mk().to(DEV), mk().to(DEV))
                out[f"{sname}/{mname}"] = {"segments": [list(s) for s in step.segments], "n_trained": step.n_trained}
            except Exception as e:
                out[f"{sname}/{mname}"] = {"error": type(e).__name__}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    res = {}
    for name, make in configurations().items():
        step, calls = make()
        res[name] = record(step, calls)
        print(f"{name}: {len(res[name]['trace'])} launches over {len(calls)} steps", flush=True)
    res["segments_by_model"] = segment_table()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=0, sort_keys=True)
    print(json.dumps({"configurations": len(res) - 1, "launches": sum(len(v["trace"]) for k, v in res.items() if "trace" in v)}))


if __name__ == "__main__":
    main()
