"""The fused per-step body (wsl4mis_b200.engine.TrainStep) against the CPU oracle's step for every hot-path script
variant: loss value, and the SGD update direction of every parameter; CUDA-graph replay == eager launch sequence."""
import copy

import numpy as np
import pytest
import torch

import wsl_oracle as O
from _gpu_util import chan_masks, cosine, elem_masks_nchw, ENC_MASK_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT


def _setup(cct, n, hw, seed=3):
    torch.manual_seed(seed)
    m = (UNet_CCT if cct else UNet)(1, 4)          # reference default init (bit-identical to the reference's)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    em = elem_masks_nchw(5, n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    ck = None
    if cct:
        ck = chan_masks(9, n)
        m.channel_keep = [c.to(DEV) for c in ck]
    image, label = O.synth_batch(n, hw, hw, seed=11, frac=0.05)
    return m, p, {k: e for k, e in zip(ENC_MASK_KEYS, em)}, ck, image, label


@pytest.mark.parametrize("variant,cct", [("pce", False), ("pce_gatedcrf", False), ("pce_gatedcrf", True), ("pce_ms", False),
                                         ("pce_tv", False), ("dmpls", True), ("pce_entropy", False), ("pce_variance", False)])
def test_step_matches_oracle(variant, cct):
    n, hw = 4, 64
    m, p, om, ock, image, label = _setup(cct, n, hw)
    step = TrainStep(m, variant, base_lr=0.01, graph=False)
    import random
    random.seed(123)
    ovariant = variant
    if variant == "pce_variance":
        from wsl4mis_b200.utils import ramps
        step.iter_num = 4500                   # a non-trivial ramp weight
        ovariant = f"pce_variance:{0.1 * ramps.sigmoid_rampup(4500 // 150, 200.0)}"
    loss = step(image.to(DEV), label.to(DEV))
    torch.cuda.synchronize()
    beta = getattr(step, "beta", 0.5)
    O.QUANT = True                                        # oracle emulating bf16 storage (see test_gpu_unet.py)
    try:
        if variant == "pce_gatedcrf" and cct:
            # single-head script on a two-head model: loss on main_seg only (SURVEY F7)
            leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
            main, _ = O.unet_cct_forward(leaves, image, True, om, ock)
            ref_loss = O.step_loss_pce_gatedcrf(main, image, label)[0]
            names = [k for k, v in leaves.items() if v.requires_grad]
            gs = torch.autograd.grad(ref_loss, [leaves[k] for k in names], allow_unused=True)
            grads = {k: g for k, g in zip(names, gs)}
        else:
            ref_loss, grads, _ = O.full_step(p, image, label, ovariant, cct, om, ock, beta)
    finally:
        O.QUANT = None
    assert abs(loss.item() - ref_loss.item()) < 0.02 * abs(ref_loss.item()) + 1e-4, (loss.item(), ref_loss.item())
    # SGD first step: delta = -lr * (g + wd*w); compare directions parameter by parameter
    named = dict(m.named_parameters())
    worst = 1.0
    for k, g in grads.items():
        new = named[k].detach().cpu()
        if g is None:                                      # untouched aux decoder: skipped by the optimiser
            assert torch.equal(new, p[k]), k
            continue
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue                                       # zero-gradient biases in front of BatchNorm
        delta, ref_delta = new - p[k], -0.01 * (g + 1e-4 * p[k])
        c = cosine(delta, ref_delta)
        worst = min(worst, c)
        assert c > 0.9, (variant, k, c)
        assert abs(delta.norm().item() - ref_delta.norm().item()) < 0.35 * ref_delta.norm().item() + 1e-9, k
    print(f"[{variant} cct={cct}] loss {loss.item():.5f} (oracle {ref_loss.item():.5f}), worst update cosine {worst:.4f}")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_uamt_step_matches_oracle(precision):
    """BASELINE config 5 (train_uncertainty_aware_mean_teacher_2D.py:138-197): student on labelled + unlabelled halves,
    never-updated teacher with T = 8 noisy passes, uncertainty-masked consistency.  Noise and dropout masks injected."""
    from wsl4mis_b200.engine import UAMTStep
    B, hw = 2, 32
    torch.manual_seed(21)
    student, teacher = UNet(1, 4), UNet(1, 4)
    ps = {k: v.clone() for k, v in student.state_dict().items()}
    pt = {k: v.clone() for k, v in teacher.state_dict().items()}
    student, teacher = student.to(DEV).set_precision(precision), teacher.to(DEV).set_precision(precision)
    ones = [torch.ones(B, O.FT[i], hw >> i, hw >> i, dtype=torch.uint8) for i in range(5)]
    for m in (student, teacher):
        m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(ones)}
    om = {k: e for k, e in zip(ENC_MASK_KEYS, ones)}
    om2 = {k: e.repeat(2, 1, 1, 1) for k, e in om.items()}
    g = torch.Generator().manual_seed(5)
    img_l, img_u = torch.rand(B, 1, hw, hw, generator=g), torch.rand(B, 1, hw, hw, generator=g)
    lab_l = torch.randint(0, 4, (B, hw, hw), generator=g, dtype=torch.uint8)
    noises = [torch.clamp(torch.randn(B, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2)] + \
             [torch.clamp(torch.randn(2 * B, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2) for _ in range(4)]
    step = UAMTStep(student, teacher, base_lr=0.01, max_iterations=30000)
    step.iter_num = 900                       # non-trivial consistency weight / threshold
    loss = step(img_l.to(DEV), lab_l.to(DEV), img_u.to(DEV), [n.to(DEV) for n in noises])
    torch.cuda.synchronize()
    # ---- oracle ----
    if precision == "bf16":
        O.QUANT = True
    try:
        leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in ps.items()}
        out_l = O.unet_forward(leaves, img_l, True, om)
        out_u = O.unet_forward(leaves, img_u, True, om)
        with torch.no_grad():
            ema_out = O.unet_forward(pt, img_u + noises[0], True, om)
            mc = torch.cat([O.unet_forward(pt, img_u.repeat(2, 1, 1, 1) + noises[1 + i], True, om2) for i in range(4)], 0)
        ref_loss, sup, cons, mask, cw, thr = O.uamt_losses(out_l, out_u, ema_out, mc, lab_l, 900, 30000)
        names = [k for k, v in leaves.items() if v.requires_grad]
        grads = dict(zip(names, torch.autograd.grad(ref_loss, [leaves[k] for k in names], allow_unused=True)))
    finally:
        O.QUANT = None
    tol = 1e-4 if precision == "fp32" else 0.03
    assert abs(step.parts["weight"] - cw) < 1e-9 and abs(step.parts["threshold"] - thr) < 1e-9
    assert abs(loss.item() - ref_loss.item()) < tol * abs(ref_loss.item()) + 1e-5, (loss.item(), ref_loss.item())
    agree = (step.parts["mask"].cpu().float() == mask[:, 0]).float().mean().item()
    assert agree > (0.9999 if precision == "fp32" else 0.97), agree
    named = dict(student.named_parameters())
    worst = 1.0
    for k, gr in grads.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        delta = named[k].detach().cpu() - ps[k]
        ref_delta = -0.01 * (gr + 1e-4 * ps[k])
        c = cosine(delta, ref_delta)
        worst = min(worst, c)
        assert c > (0.999 if precision == "fp32" else 0.85), (k, c)
    print(f"[uamt {precision}] loss {loss.item():.6f} (oracle {ref_loss.item():.6f}), mask agreement {agree:.4f}, worst update cosine {worst:.5f}")


def _lockstep(eager, captured, calls, state):
    """Step an eager and a graph-captured stepper side by side on the same inputs and compare EVERY step's loss and weights, then
    copy the eager state over the captured one.  (The fp32 cross-check mode accumulates weight gradients with atomics; run to run
    that is 1e-8 of noise which training amplifies ~4x per step, so a comparison of final weights after many free-running steps cannot tell a stale ramp from noise.  One step from
    identical state can: noise stays ~1e-9, a wrong EMA factor or ramp value is >= 1e-4.)"""
    worst = 0.0
    for i, call_args in enumerate(calls):
        le, lg = eager(*call_args[0], **call_args[1]).item(), captured(*call_args[0], **call_args[1]).item()
        torch.cuda.synchronize()
        assert abs(le - lg) < 1e-4 * abs(le), (i, le, lg)
        for name in state:
            a, b = getattr(captured, name), getattr(eager, name)
            d = ((a - b).norm() / b.norm().clamp_min(1e-30)).item()
            worst = max(worst, d)
            assert d < 1e-5, (i, name, d)
            a.copy_(b)
    return worst


def test_uamt_graph_replay_equals_eager():
    """UAMTStep(graph=True): the captured body (7 network passes, losses, two backwards, SGD) with the ramps read from device
    memory takes the same steps as the eager body -- across the iteration where the consistency weight changes (:183 uses
    iter_num // 300)."""
    from wsl4mis_b200.engine import UAMTStep
    B, hw = 2, 64
    g = torch.Generator().manual_seed(8)
    img_l, img_u = torch.rand(B, 1, hw, hw, generator=g).to(DEV), torch.rand(B, 1, hw, hw, generator=g).to(DEV)
    lab_l = torch.randint(0, 4, (B, hw, hw), generator=g, dtype=torch.uint8).to(DEV)
    steps = {}
    for graph in (False, True):
        torch.manual_seed(33)
        student, teacher = UNet_CCT(1, 4).to(DEV).set_precision("fp32"), UNet_CCT(1, 4).to(DEV).set_precision("fp32")
        steps[graph] = UAMTStep(student, teacher, base_lr=0.01, max_iterations=30000, graph=graph)
        steps[graph].iter_num = 297
    worst = _lockstep(steps[False], steps[True], [((img_l, lab_l, img_u), {})] * 6, ("flat", "mom"))
    e, c = steps[False], steps[True]
    assert list(c._graphs) == [0] and c.launches_per_step > 500 and c.iter_num == e.iter_num == 303
    assert e.parts["weight"] == c.parts["weight"] and e.parts["threshold"] == c.parts["threshold"]
    w0 = 0.1 * c.ramps.sigmoid_rampup(0, 200.0)
    assert c.parts["weight"] != w0                    # the ramp weight changed at iteration 300, inside the captured steps
    print(f"[uamt graph] worst single-step weight difference captured vs eager {worst:.2e}")


def test_ustm_graph_replay_equals_eager():
    """USTMStep(graph=True): one captured graph per rot90 count (a kernel argument, :123); threshold, weight and the EMA factor
    (which changes every step below iteration 99) come from device memory."""
    from wsl4mis_b200.engine import USTMStep
    B, hw = 2, 64
    img, lab = O.synth_batch(B, hw, hw, seed=12, frac=0.1)
    img, lab = img.to(DEV), lab.to(DEV)
    steps = {}
    for graph in (False, True):
        torch.manual_seed(35)
        student, teacher = UNet(1, 4).to(DEV).set_precision("fp32"), UNet(1, 4).to(DEV).set_precision("fp32")
        steps[graph] = USTMStep(student, teacher, base_lr=0.01, max_iterations=60000, graph=graph)
    ks = [0, 1, 2, 3, 1, 2, 0, 3]
    worst = _lockstep(steps[False], steps[True], [((img, lab), {"rot_times": k}) for k in ks], ("flat", "mom", "tflat"))
    c = steps[True]
    assert sorted(c._graphs) == [0, 1, 2, 3] and c.iter_num == 8      # steps 0, 1 are the eager warm-up; 2.. capture / replay
    print(f"[ustm graph] worst single-step weight difference captured vs eager {worst:.2e}")


def test_clamped_noise_kernel_statistics():
    from wsl4mis_b200._lib import call
    x = torch.zeros(1 << 20, device=DEV)
    out = torch.empty(2 << 20, device=DEV)
    call("wsl_add_clamped_noise", x, x.numel(), 2, 0.1, 0.2, 7, None, out)
    torch.cuda.synchronize()
    o = out.cpu()
    assert o.abs().max().item() <= 0.2 + 1e-6 and abs(o.mean().item()) < 1e-3
    assert abs(o.std().item() - 0.0954) < 3e-3          # std of N(0, 0.1) clamped at 2 sigma
    assert not torch.equal(o[: 1 << 20], o[1 << 20:])   # the repeated copies draw different noise


def test_graph_replay_equals_eager():
    n, hw = 4, 64
    img, lab = O.synth_batch(n, hw, hw, seed=5, frac=0.05)
    img, lab = img.to(DEV), lab.to(DEV)
    losses = {}
    finals = {}
    for graph in (False, True):
        torch.manual_seed(7)
        m = UNet_CCT(1, 4).to(DEV)
        step = TrainStep(m, "pce_gatedcrf", graph=graph)
        ls = [step(img, lab).item() for _ in range(6)]
        torch.cuda.synchronize()
        losses[graph] = ls
        finals[graph] = step.flat.clone()
        assert step.iter_num == 6
    assert np.allclose(losses[False], losses[True], rtol=2e-3), (losses[False], losses[True])
    assert cosine(finals[False], finals[True]) > 0.999999
    assert losses[True][-1] < losses[True][0]


def test_dmpls_graph_follows_host_beta():
    """DMPLS inside a captured graph: the per-step beta of Python's `random` reaches the kernels through device memory."""
    import random
    n, hw = 4, 64
    img, lab = O.synth_batch(n, hw, hw, seed=5, frac=0.05)
    img, lab = img.to(DEV), lab.to(DEV)
    res = {}
    for graph in (False, True):
        torch.manual_seed(7)
        random.seed(99)
        m = UNet_CCT(1, 4).to(DEV)
        step = TrainStep(m, "dmpls", graph=graph)
        ls, betas = [], []
        for _ in range(6):
            ls.append(step(img, lab).item())
            betas.append(step.beta)
        res[graph] = (ls, betas)
    assert res[False][1] == res[True][1] and len(set(res[True][1])) == 6
    assert np.allclose(res[False][0], res[True][0], rtol=5e-3), res


def test_lr_schedule_follows_the_script():
    torch.manual_seed(0)
    m = UNet(1, 4).to(DEV)
    step = TrainStep(m, "pce", base_lr=0.03, max_iterations=100, graph=False)
    img, lab = O.synth_batch(2, 32, 32, seed=1, frac=0.1)
    for it in range(3):
        step(img.to(DEV), lab.to(DEV))
        assert abs(step.lr_dev.item() - O.poly_lr(0.03, it, 100)) < 1e-8


def test_rot90_and_ema_kernels():
    from wsl4mis_b200._lib import call
    x = torch.randn(3, 4, 16, 16, device=DEV)
    for k in range(4):
        out = torch.empty_like(x)
        call("wsl_rot90", x, 12, 16, k, 0, out)
        assert torch.equal(out, torch.rot90(x, k, [2, 3]).contiguous())
    acc = torch.ones_like(x)
    call("wsl_rot90", x, 12, 16, 3, 1, acc)
    assert torch.allclose(acc, 1 + torch.rot90(x, 3, [2, 3]))
    e, p = torch.randn(1000, device=DEV), torch.randn(1000, device=DEV)
    ref = e * 0.75 + 0.25 * p
    call("wsl_ema_update", e, p, 1000, 0.75)
    assert torch.allclose(e, ref, atol=1e-7)


@pytest.mark.parametrize("rot", [0, 1, 3])
def test_ustm_step_matches_oracle(rot):
    """train_weakly_supervised_ustm_2D.py:113-170 in fp32 parity mode: loss, SGD update and the EMA teacher update."""
    from wsl4mis_b200.engine import USTMStep
    B, hw = 2, 32
    torch.manual_seed(33)
    student, teacher = UNet(1, 4), UNet(1, 4)
    ps = {k: v.clone() for k, v in student.state_dict().items()}
    pt = {k: v.clone() for k, v in teacher.state_dict().items()}
    student, teacher = student.to(DEV).set_precision("fp32"), teacher.to(DEV).set_precision("fp32")
    ones = [torch.ones(B, O.FT[i], hw >> i, hw >> i, dtype=torch.uint8) for i in range(5)]
    for m in (student, teacher):
        m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(ones)}
    om = {k: e for k, e in zip(ENC_MASK_KEYS, ones)}
    om2 = {k: e.repeat(2, 1, 1, 1) for k, e in om.items()}
    img, lab = O.synth_batch(B, hw, hw, seed=8, frac=0.1)
    g = torch.Generator().manual_seed(6)
    noises = [torch.clamp(torch.randn(B, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2)] + \
             [torch.clamp(torch.randn(2 * B, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2) for _ in range(4)]
    step = USTMStep(student, teacher, base_lr=0.03, max_iterations=60000)
    step.iter_num = 5000
    loss = step(img.to(DEV), lab.to(DEV), [n.to(DEV) for n in noises], rot_times=rot)
    torch.cuda.synchronize()
    leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in ps.items()}
    out = O.unet_forward(leaves, img, True, om)
    rimg = torch.rot90(img, rot, [2, 3])
    with torch.no_grad():
        ema_out = O.unet_forward(pt, rimg + noises[0], True, om)
        mc = torch.cat([O.unet_forward(pt, rimg.repeat(2, 1, 1, 1) + noises[1 + i], True, om2) for i in range(4)], 0)
    ref_loss, ce, cons, mask, cw, thr = O.ustm_losses(out, ema_out, mc, lab, rot, 5000, 60000)
    assert abs(loss.item() - ref_loss.item()) < 1e-4 * abs(ref_loss.item()), (loss.item(), ref_loss.item())
    names = [k for k, v in leaves.items() if v.requires_grad]
    grads = dict(zip(names, torch.autograd.grad(ref_loss, [leaves[k] for k in names])))
    new_s = {k: ps[k] - 0.03 * (grads[k] + 1e-4 * ps[k]) for k in names}
    named, tnamed = dict(student.named_parameters()), dict(teacher.named_parameters())
    alpha = min(1 - 1 / (5000 + 1), 0.99)
    for k in names:
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        assert cosine(named[k].detach().cpu() - ps[k], new_s[k] - ps[k]) > 0.999, k
        ref_t = pt[k] * alpha + (1 - alpha) * named[k].detach().cpu()
        assert torch.allclose(tnamed[k].detach().cpu(), ref_t, atol=1e-6), k


def test_training_is_bit_reproducible_run_to_run():
    """Two runs of three fused steps from the same weights / batch / seeds end with bit-identical parameters and losses: every
    reduction on the path has a fixed order (BatchNorm statistics, loss sums, split-K weight gradients via per-CTA partial tiles
    and a fixed-order finalize, bias gradients, the first layer's fused weight gradient)."""
    import random
    outs = []
    for rep in range(2):
        torch.manual_seed(3)
        random.seed(3)
        m = UNet_CCT(1, 4).to(DEV)
        # 256 x 256: every layer runs on the tensor-core kernels (maps smaller than one 16 x 8 tile fall back to the CUDA-core
        # weight gradient, which still accumulates with atomics)
        image, label = O.synth_batch(2, 256, 256, seed=11, frac=0.05)
        step = TrainStep(m, "dmpls", graph=False)
        losses = [float(step(image.to(DEV), label.to(DEV))) for _ in range(3)]
        torch.cuda.synchronize()
        outs.append((step.flat.detach().clone(), losses))
    assert outs[0][1] == outs[1][1], (outs[0][1], outs[1][1])
    assert torch.equal(outs[0][0], outs[1][0])
