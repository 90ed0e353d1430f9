"""Time every row-kernel launch (conv_row_kernel behind wsl_conv_tc2) of the benchmark's training step in isolation.

    python profiles/conv_row.py [--precision bf16|fp16] [--batch 64] [--reps 200]

One eager step of bench.py's workload (unet_cct, pCE + GatedCRF, N x 1 x 256 x 256) runs with a recorder in place of
wsl4mis_b200._lib.PROFILE, which keeps every wsl_conv_tc2 call the dispatcher sends to the row kernel (3x3, CoutP 16 or 32,
W % 128 == 0, H % 16 == 0, C0 + C1 <= 64) and how often the step makes it.  Each distinct launch is then replayed on seeded
operands of its shape, timed with CUDA events over --reps launches after warm-up.  Algorithmic bytes per launch are
(input + output channels) x pixels x 2 B, 4 B per output channel for the fp32 NCHW logits.  The card name and power limit are
read in the same run."""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEV = torch.device("cuda", 0)
HBM_GBS = 3350.0        # H100 SXM data sheet (700 W)
T16 = {0: torch.bfloat16, 2: torch.float16}


def card():
    name = torch.cuda.get_device_name(DEV)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[DEV.index or 0]
    except Exception as e:      # the timing does not depend on it; say so instead
        q = f"power limit not readable ({e})"
    return f"{name}, {q}"


def is_row(a):
    return (a["ksize"] == 3 and a["CoutP"] in (16, 32) and a["W"] % 128 == 0 and a["H"] % 16 == 0 and a["C0"] + a["C1"] <= 64)


class RowRecorder:
    """stands in for _lib.PROFILE: runs every call and counts the distinct row-kernel launches of wsl_conv_tc2"""

    def __init__(self):
        self.meta = None
        self.launches = {}

    def record(self, name, fn, vals):
        from wsl4mis_b200._lib import LIB
        rc = fn(*vals)
        if rc != 0:
            raise RuntimeError(f"{name} failed ({rc}): {LIB.last_error()}")
        if name != "wsl_conv_tc2":
            return
        args = [(nm, ty, v) for (ty, nm), v in zip(LIB.protos[name][1], vals) if nm != "stream"]
        a = {nm: v for nm, ty, v in args if ty is not ctypes.c_void_p}
        if not is_row(a):
            return
        null = tuple(nm for nm, ty, v in args if ty is ctypes.c_void_p and v is None)
        key = (tuple(sorted(a.items())), null)
        self.launches[key] = self.launches.get(key, 0) + 1


def harvest(precision, batch):
    from wsl4mis_b200 import _lib
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet_CCT
    sys.path.insert(0, ROOT)
    import bench
    torch.manual_seed(2022)
    model = UNet_CCT(1, 4).to(DEV).set_precision(precision)
    step = TrainStep(model, "pce_gatedcrf", graph=False, world_size=1)
    step.ex.multi_stream = False
    img, lab = bench.synth(batch, 2022)
    img, lab = img.to(DEV), lab.to(DEV)
    step(img, lab)
    torch.cuda.synchronize()
    rec, saved = RowRecorder(), _lib.PROFILE
    _lib.PROFILE = rec
    try:
        step(img, lab)
        torch.cuda.synchronize()
    finally:
        _lib.PROFILE = saved
    del step, model
    torch.cuda.empty_cache()
    return rec.launches


def time_launch(a, null, reps, warm):
    from wsl4mis_b200._lib import call
    g = torch.Generator(device=DEV).manual_seed(1234)
    C0, C1, N, H, W = a["C0"], a["C1"], a["N"], a["H"], a["W"]
    CoutP, Cs, dt, mode = a["CoutP"], a["CoutStore"], a["dtype"], a["out_mode"]
    s0 = torch.randn(N, H, W, C0, device=DEV, generator=g).to(T16[dt])
    s1 = torch.randn(N, H, W, C1, device=DEV, generator=g).to(T16[dt]) if C1 else None
    wpk = (torch.randn(9 * (C0 + C1) * CoutP, device=DEV, generator=g) * 0.05).to(T16[dt])
    bias = None if "bias" in null else torch.randn(CoutP, device=DEV, generator=g)
    out = torch.empty((N, Cs, H, W) if mode == 1 else (N, H, W, Cs), device=DEV, dtype=torch.float32 if mode == 1 else T16[dt])
    parts = None if "stat_partials" in null else torch.empty(2048 * 2 * CoutP, device=DEV)
    rows = ctypes.c_int(0)

    def run():
        call("wsl_conv_tc2", s0, C0, s1, C1, wpk, bias, out, mode, N, H, W, CoutP, Cs, 3, dt, parts, ctypes.addressof(rows))
    for _ in range(warm):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / reps * 1e3
    px = N * H * W
    nbytes = px * ((C0 + C1) * 2 + Cs * (4 if mode == 1 else 2))
    return us, nbytes, rows.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    print(f"card: {card()}")
    print(f"workload: unet_cct pCE+GatedCRF {args.precision}, {args.batch}x1x256x256; row-kernel launches of one training step")
    launches = harvest(args.precision, args.batch)
    print(f"{'shape':<24} {'C0+C1->Cout':<12} {'mode':<5} {'bias':<5} {'stats':<5} {'per step':>8} {'grid':>5} {'us':>9} "
          f"{'GB/s':>7} {'of 3.35 TB/s':>12}")
    tot_us = tot_bytes = 0.0
    n_launch = 0
    for (items, null), count in sorted(launches.items(), key=lambda kv: kv[0]):
        a = dict(items)
        us, nbytes, grid = time_launch(a, null, args.reps, args.warmup)
        gbs = nbytes / (us * 1e-6) / 1e9
        tot_us += us * count
        tot_bytes += nbytes * count
        n_launch += count
        print(f"{a['N']}x{a['H']}x{a['W']:<14} {a['C0']}+{a['C1']}->{a['CoutStore']:<6} {a['out_mode']:<5} "
              f"{'no' if 'bias' in null else 'yes':<5} {'no' if 'stat_partials' in null else 'yes':<5} {count:>8} {grid:>5} "
              f"{us:>9.1f} {gbs:>7.0f} {gbs / HBM_GBS:>12.3f}")
    gbs = tot_bytes / (tot_us * 1e-6) / 1e9
    print(f"per step: {n_launch} row launches, {tot_us / 1e3:.3f} ms, {tot_bytes / 1e9:.2f} GB algorithmic, {gbs:.0f} GB/s = "
          f"{gbs / HBM_GBS:.3f} of 3.35 TB/s")


if __name__ == "__main__":
    main()
