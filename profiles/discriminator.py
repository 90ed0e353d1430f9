"""Time FCDiscriminator at the DAN script's shapes (train_deep_adversarial_network_2D.py:107-178) with CUDA events after warm-up.

    python profiles/discriminator.py [--reps 20]

Rows: phase 1 (B = 6, eval, gradients w.r.t. the map and the parameters), phase 2 (2B = 12, train, parameter gradients only) and
train-mode batches of 32 and 64, each forward + backward, for this repository's discriminator in bf16 and fp32 mode and for the
reference class (staged by oracle/stage_semi.py) on cuDNN at torch defaults and under bf16 autocast, on the same inputs.  Useful
TFLOP/s counts the 4x4 / stride-2 convolutions' own work; the tensor cores execute 36/16 = 2.25x that (structured 3x3 weights).
Then one full DAN iteration (both phases, this repository's UNet as the student) with each discriminator.  The card name and power
limit are read in the same run."""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import dan_oracle as D  # noqa: E402

DEV = torch.device("cuda", 0)


def conv_flops(n, ndf=64, cin=5, hw=256):
    """useful forward FLOPs of the five convolutions per batch: [first layer (conv0 + conv1), conv2, conv3, conv4]"""
    out, c, h = [], cin, hw
    for cout in (ndf, 2 * ndf, 4 * ndf, 8 * ndf):
        h //= 2
        out.append(2.0 * n * h * h * cout * c * 16)
        c = cout
    return out


def step_flops(n, input_grad):
    f = conv_flops(n)
    return sum(f) + sum(f) + sum(f[1:]) + (f[0] if input_grad else 0.0)     # forward + weight gradients + data gradients


def card():
    name = torch.cuda.get_device_name(DEV)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[DEV.index or 0]
    except Exception as e:      # the timing does not depend on it; say so instead
        q = f"power limit not readable ({e})"
    return f"{name}, {q}"


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def disc_step(model, mp, feat, tgt, input_grad, autocast=False):
    def run():
        model.zero_grad(set_to_none=True)
        m = mp.detach().requires_grad_(input_grad)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = model(m, feat)
        F.cross_entropy(out.float(), tgt).backward()
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/discriminator.py measures on a GPU"
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    import stage_semi
    ref_mod = stage_semi.load_reference_discriminator()
    torch.backends.cudnn.benchmark = True
    print(f"card: {card()}")
    p = D.synth_params(101)
    impls = {}
    for prec in ("bf16", "fp32"):
        m = FCDiscriminator(4)
        m.load_state_dict(p)
        impls["ours " + prec] = (m.to(DEV).set_precision(prec), False)
    if ref_mod is not None:
        r = ref_mod.FCDiscriminator(4)
        r.load_state_dict(p)
        r = r.to(DEV)
        impls["cuDNN fp32"] = (r, False)
        impls["cuDNN bf16 autocast"] = (r, True)
    else:
        print("reference discriminator not staged: cuDNN rows not measured")
    rows = [("phase 1", 6, False, True), ("phase 2", 12, True, False), ("train 32", 32, True, False), ("train 64", 64, True, False)]
    print(f"{'shape':10s} {'impl':20s} {'ms':>9s} {'img/s':>8s} {'useful TFLOP/s':>15s} {'MMA TFLOP/s':>12s}")
    for label, n, training, input_grad in rows:
        mp, feat = D.synth_inputs(5, n)
        mp, feat = mp.to(DEV), feat.to(DEV)
        tgt = torch.tensor([1, 0] * (n // 2), device=DEV)
        fl = step_flops(n, input_grad)
        for name, (model, ac) in impls.items():
            model.train(training)
            reps = max(2, args.reps // 10) if name == "ours fp32" else args.reps
            ms = timed(disc_step(model, mp, feat, tgt, input_grad, ac), reps, warm=1 if name == "ours fp32" else 3)
            mma = f"{fl * 2.25 / ms / 1e9:12.1f}" if name == "ours bf16" else f"{'':12s}"
            print(f"{label:10s} {name:20s} {ms:9.3f} {n * 1e3 / ms:8.0f} {fl / ms / 1e9:15.1f} {mma}")
    dan_iteration(impls)


def dan_iteration(impls, B=6, reps=10):
    """train_deep_adversarial_network_2D.py:138-178 with this repository's UNet as the student, per discriminator"""
    import wsl_oracle as O
    from wsl4mis_b200.networks.unet import UNet
    from wsl4mis_b200.utils import losses
    student = UNet(1, 4)
    student.load_state_dict(O.synth_params(1, 4, ("decoder",), 7))
    student = student.to(DEV)
    opt = torch.optim.SGD(student.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    xl, yl = O.synth_batch(B, 256, 256, seed=3, dense=True)
    xl, yl = xl.to(DEV), yl.to(DEV)
    xu = xl.flip(3).contiguous()
    dice = losses.DiceLoss(4)
    tgt = torch.tensor([1] * B + [0] * B, device=DEV)
    print(f"\nfull DAN iteration (B = {B} labelled + {B} unlabelled, student UNet bf16, SGD + Adam):")
    for name, (disc, ac) in impls.items():
        if name == "ours fp32":
            continue
        dopt = torch.optim.Adam(disc.parameters(), lr=1e-4, betas=(0.9, 0.99))

        def it():
            student.train()
            disc.eval()
            ol, ou = student(xl), student(xu)
            sl = torch.softmax(ol, 1)
            sup = 0.5 * (dice(sl, yl.unsqueeze(1)) + F.cross_entropy(ol, yl.long()))
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
                do = disc(torch.softmax(ou, 1), xu)
            loss = sup + 0.1 * F.cross_entropy(do.float(), tgt[:B])
            opt.zero_grad()
            loss.backward()
            opt.step()
            student.eval()
            disc.train()
            with torch.no_grad():
                maps = torch.softmax(torch.cat([student(xl), student(xu)], 0), 1)
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
                do = disc(maps, torch.cat([xl, xu], 0))
            dl = F.cross_entropy(do.float(), tgt)
            dopt.zero_grad()
            dl.backward()
            dopt.step()
        ms = timed(it, reps)
        print(f"  {name:20s} {ms:8.2f} ms / iteration  ({2 * B * 1e3 / ms:.0f} labelled + unlabelled images/s)")


if __name__ == "__main__":
    main()
