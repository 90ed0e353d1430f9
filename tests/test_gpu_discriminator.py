"""FCDiscriminator on the H100 (reference networks/discriminator.py:58-101): the space-to-depth packers bit for bit against the CPU
oracle, every convolution launch of the plan (tensor-core in bf16, CUDA-core in fp32) at the DAN script's shapes against fp64 on the
same operands, both modes against the oracle, and one full DAN iteration (train_deep_adversarial_network_2D.py:138-178) in fp32
mode."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dan_oracle as D
from _conv_check import (SLACK_16, UNIT_ROUNDOFF, check_output, check_wgrad, describe, direct_slack, direct_u, reference,
                         wgrad_reference)
from _gpu_util import ENC_MASK_KEYS, elem_masks_nchw, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _model(precision, pseed=101):
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    m = FCDiscriminator(4)
    m.load_state_dict(D.synth_params(pseed))
    return m.to(DEV).set_precision(precision)


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def test_packers_and_gathers_bit_exact():
    from wsl4mis_b200._lib import call
    g = torch.Generator().manual_seed(7)
    N, H = 2, 32
    mp, feat = torch.rand(N, 4, H, H, generator=g), torch.rand(N, 1, H, H, generator=g)
    for dt, tdt in ((0, torch.bfloat16), (1, torch.float32)):
        T = torch.empty(N, H // 2, H // 2, 32, dtype=tdt, device=DEV)
        call("wsl_disc_pack_input", mp.to(DEV), 4, feat.to(DEV), 1, N, H, H, 32, T, dt)
        assert torch.equal(T.cpu(), D.s2d(torch.cat([mp, feat], 1), 32).to(tdt))
        dmap, dfeat = torch.empty(N, 4, H, H, device=DEV), torch.empty(N, 1, H, H, device=DEV)
        call("wsl_disc_unpack_input_grad", T, dt, N, H, H, 32, 4, 1, dmap, dfeat)
        back = D.d2s(T.cpu().float(), 5)
        assert torch.equal(dmap.cpu(), back[:, :4]) and torch.equal(dfeat.cpu(), back[:, 4:])
        C = 24
        y = torch.randn(N, H, H, C, generator=g).to(tdt)
        keep = (torch.rand(N, C, generator=g) >= 0.5).float()
        for slope, cs in ((1.0, None), (0.2, keep * 2.0)):
            out = torch.empty(N, H // 2, H // 2, 4 * C, dtype=tdt, device=DEV)
            call("wsl_s2d_act_fwd", y.to(DEV), dt, N, H, H, C, slope, None if cs is None else cs.to(DEV), out)
            a = F.leaky_relu(y.float(), slope) * (1.0 if cs is None else cs[:, None, None, :])
            assert torch.equal(out.cpu(), D.s2d(a.permute(0, 3, 1, 2)).to(tdt))
            dT = torch.randn(N, H // 2, H // 2, 4 * C, generator=g).to(tdt)
            dy = torch.empty(N, H, H, C, dtype=tdt, device=DEV)
            call("wsl_d2s_act_bwd", dT.to(DEV), None if cs is None else y.to(DEV), dt, N, H, H, C, slope, None if cs is None else cs.to(DEV), dy)
            r = D.d2s(dT.float(), C).permute(0, 2, 3, 1)
            if cs is not None:
                r = r * cs[:, None, None, :] * torch.where(y.float() > 0, 1.0, slope)
            assert torch.equal(dy.cpu(), r.to(tdt))
    w0, w1 = torch.randn(64, 4, 4, 4, generator=g), torch.randn(64, 1, 4, 4, generator=g)
    b0, b1 = torch.randn(64, generator=g), torch.randn(64, generator=g)
    w3, bias = torch.empty(64 * 32 * 9, device=DEV), torch.empty(64, device=DEV)
    call("wsl_disc_scatter_weights", w0.to(DEV), b0.to(DEV), 4, w1.to(DEV), b1.to(DEV), 1, 64, 32, w3, bias)
    assert torch.equal(w3.cpu().view(64, 32, 3, 3), D.scatter(torch.cat([w0, w1], 1), 32))
    assert torch.equal(bias.cpu(), b0 + b1)
    dw3 = torch.randn(64, 32, 3, 3, generator=g)
    d0, d1 = torch.empty(64, 4, 4, 4, device=DEV), torch.empty(64, 1, 4, 4, device=DEV)
    call("wsl_disc_gather_wgrad", dw3.to(DEV), 64, 32, 4, 1, d0, d1)
    ref = D.gather(dw3, 5)
    assert torch.equal(d0.cpu(), ref[:, :4]) and torch.equal(d1.cpu(), ref[:, 4:])


@pytest.mark.parametrize("N", [6, 12])
def test_tensor_core_launches_against_fp64(N):
    """forward, data gradient and weight gradient of every layer on the bf16 tensor-core kernels, with the operands the executor
    produced at the DAN script's batch sizes (phase 1: B = 6, phase 2: 2B = 12)"""
    _layer_launches_against_fp64(N, "bf16")


@pytest.mark.parametrize("N", [6, 12])
def test_direct_kernel_launches_against_fp64(N):
    """the same in fp32 mode, on the CUDA-core wsl_conv_direct / wsl_wgrad_direct: the last layer reads 1024 channels (K = 9216
    sequential FMAs per output, and 2048 weight-gradient CTAs)"""
    _layer_launches_against_fp64(N, "fp32")


def _layer_launches_against_fp64(N, precision):
    m = _model(precision)
    m.train()
    mp, feat = D.synth_inputs(5, N)
    m.channel_keep = D.chan_keep(6, N)
    ex = m.executor
    logits, rec = ex.forward(mp.to(DEV), feat.to(DEV), True, True, True, m.channel_keep)
    g = torch.Generator(device=DEV).manual_seed(N)
    f32 = precision == "fp32"
    u = direct_u(torch.float32) if f32 else UNIT_ROUNDOFF[torch.bfloat16]
    for i, L in enumerate(ex.layers):
        fwd, dgr, bias = rec["packs"][i]
        T, y = rec["Ts"][i], rec["ys"][i]
        if f32:       # 'wf' pack [taps][CinP][CoutP] -> torch layout
            w3 = fwd.view(9, L.CP, L.Cout).permute(2, 1, 0).reshape(L.Cout, L.CP, 3, 3).double()
        else:         # wgmma B operand [taps][Cout][Cin] -> torch layout
            w3 = fwd.view(9, L.Cout, L.CP).permute(1, 2, 0).reshape(L.Cout, L.CP, 3, 3).double()
        ref, S = reference(_nchw(T), w3, bias.double())
        rep = check_output(_nchw(y), ref, S, u, direct_slack(9 * L.CP) if f32 else SLACK_16)
        assert rep["bad"] == 0, f"layer {i} forward (N={N}): {describe(rep)}"
        fw = rep["worst"]
        dy = torch.randn(y.shape, generator=g, device=DEV) * 0.1
        dy = dy if f32 else dy.to(torch.bfloat16)
        dT = ex._dgrad(L, dy, dgr, N)
        ref, S = reference(_nchw(dy), w3.flip(2, 3).transpose(0, 1), None)
        rep = check_output(_nchw(dT), ref, S, u, direct_slack(9 * L.Cout) if f32 else SLACK_16)
        assert rep["bad"] == 0, f"layer {i} data gradient (N={N}): {describe(rep)}"
        dws, db = ex._wgrad(L, T, dy, N)
        dw_ref = D.gather(wgrad_reference(_nchw(T), _nchw(dy), 3), L.C)
        rw = check_wgrad(torch.cat(dws, 1), dw_ref, 64, L.C)
        assert not rw["bad"], f"layer {i} weight gradient (N={N}): {rw}"
        assert rel_l2(db, _nchw(dy).sum((0, 2, 3))) < 1e-5, f"layer {i} bias gradient"
        print(f"[disc {precision} N={N}] layer {i} ({L.CP} -> {L.Cout} at {L.h}x{L.h}): error / bound forward {fw:.3g}, data gradient "
              f"{rep['worst']:.3g}; wgrad rel-L2 {rw['rel']:.2e}")


def _oracle_run(p, mp, feat, training, keep, quant=None, dtype=torch.float64):
    pp = {k: v.to(DEV, dtype).requires_grad_(True) for k, v in p.items()}
    m, f = mp.to(DEV, dtype).requires_grad_(True), feat.to(DEV, dtype).requires_grad_(True)
    logits = D.forward(pp, m, f, training, [k.to(DEV) for k in keep], quant)
    F.cross_entropy(logits, torch.tensor([1, 0] * (mp.shape[0] // 2), device=DEV)).backward()
    return logits.detach(), m.grad, f.grad, [pp[k].grad for k in pp]


def _ours(precision, mp, feat, training, keep):
    m = _model(precision)
    m.train(training)
    m.channel_keep = keep
    mg, fg = mp.to(DEV).requires_grad_(True), feat.to(DEV).requires_grad_(True)
    logits = m(mg, fg)
    F.cross_entropy(logits, torch.tensor([1, 0] * (mp.shape[0] // 2), device=DEV)).backward()
    return logits.detach(), mg.grad, fg.grad, [q.grad for q in m.parameters()]


@pytest.mark.parametrize("training", [False, True])
def test_fp32_mode_against_fp64_oracle(training):
    mp, feat = D.synth_inputs(202, 2)
    keep = D.chan_keep(303, 2)
    lo, dmo, dfo, go = _ours("fp32", mp, feat, training, keep)
    lr, dmr, dfr, gr = _oracle_run(D.synth_params(101), mp, feat, training, keep)
    err = (lo.double() - lr).abs().max().item() / lr.abs().max().item()
    assert err < 1e-5, err
    assert rel_l2(dmo, dmr) < 1e-4 and rel_l2(dfo, dfr) < 1e-4, (rel_l2(dmo, dmr), rel_l2(dfo, dfr))
    errs = {k: rel_l2(a, b) for k, a, b in zip(D.param_shapes(), go, gr)}
    assert max(errs.values()) < 1e-4, errs
    print(f"[disc fp32 training={training}] logits {err:.2e} of scale, map grad {rel_l2(dmo, dmr):.2e}, worst param grad "
          f"{max(errs.values()):.2e}")


@pytest.mark.parametrize("training", [False, True])
def test_bf16_mode_against_bf16_emulating_oracle(training):
    """the oracle rounds what the executor stores in the forward (inputs, weights, conv outputs, activations); gradients travel in
    bf16 in the executor and in fp32 in the oracle, which the gradient bound absorbs"""
    mp, feat = D.synth_inputs(202, 2)
    keep = D.chan_keep(303, 2)
    lo, dmo, dfo, go = _ours("bf16", mp, feat, training, keep)
    lr, dmr, dfr, gr = _oracle_run(D.synth_params(101), mp, feat, training, keep, quant=torch.bfloat16, dtype=torch.float32)
    err = (lo.double() - lr.double()).abs().max().item() / lr.abs().max().item()
    errs = {k: rel_l2(a, b) for k, a, b in zip(D.param_shapes(), go, gr)}
    print(f"[disc bf16 training={training}] logits {err:.2e} of scale, map grad {rel_l2(dmo, dmr):.2e}, worst param grad "
          f"{max(errs.values()):.2e}")
    assert err < 5e-3, err
    assert rel_l2(dmo, dmr) < 4e-2, rel_l2(dmo, dmr)
    assert max(errs.values()) < 4e-2, errs


def test_dan_iteration_fp32_mode_matches_oracle():
    """train_deep_adversarial_network_2D.py:138-178 for the unlabelled half: phase 1 (student train, D eval) back-propagates the
    adversarial cross entropy through D, the softmax and the student; phase 2 (D train on 2B no-grad maps) takes one Adam step"""
    import wsl_oracle as O
    from wsl4mis_b200.networks.unet import UNet
    B, HW = 2, 256
    ps = O.synth_params(1, 4, ("decoder",), 7)
    student = UNet(1, 4)
    student.load_state_dict(ps)
    student = student.to(DEV).set_precision("fp32")
    student.train()
    em = elem_masks_nchw(11, B, HW, HW)
    student.dropout_masks = {i: em[i].permute(0, 2, 3, 1).contiguous().to(DEV) for i in range(5)}
    x, _ = O.synth_batch(B, HW, HW, seed=3)
    x = x.to(DEV)
    disc = _model("fp32")
    disc.eval()
    # phase 1: ours
    out = student(x)
    loss1 = F.cross_entropy(disc(torch.softmax(out, 1), x), torch.ones(B, dtype=torch.long, device=DEV))
    loss1.backward()
    g_student = [q.grad.clone() for q in student.parameters()]
    # phase 1: oracle (fp64)
    names = [k for k, _ in student.named_parameters()]
    pso = {k: v.to(DEV, torch.float64 if v.is_floating_point() else v.dtype) for k, v in ps.items()}
    for k in names:
        pso[k].requires_grad_(True)
    pdo = {k: v.to(DEV, torch.float64) for k, v in D.synth_params(101).items()}
    masks = {k: em[i].to(DEV) for i, k in enumerate(ENC_MASK_KEYS)}
    out_o = O.unet_forward(pso, x.double(), True, masks)
    lo = F.cross_entropy(D.forward(pdo, torch.softmax(out_o, 1), x.double(), False), torch.ones(B, dtype=torch.long, device=DEV))
    lo.backward()
    assert abs(loss1.item() - lo.item()) <= 1e-5 * abs(lo.item()), (loss1.item(), lo.item())
    # a conv bias that feeds training-mode BatchNorm has an exactly-zero gradient in the executor (rounding noise in the oracle)
    feeds_bn = lambda k: ".conv_conv." in k and k.endswith((".0.bias", ".4.bias"))
    errs = {k: rel_l2(g, pso[k].grad) for k, g in zip(names, g_student) if not feeds_bn(k)}
    assert all(g_student[names.index(k)].abs().max().item() == 0.0 for k in names if feeds_bn(k))
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"[DAN phase 1 fp32] loss {loss1.item():.6f} / oracle {lo.item():.6f}; worst student gradient {worst}")
    # The bound is the student's, not D's (D's own gradients are checked at 1e-4 above).  The adversarial term reaches the student as one
    # small scalar's gradient, and the BatchNorm backward turns it into sums of dz * xhat over 131 k pixels per channel that largely
    # cancel, so the student executor's fp32 accumulation noise is large relative to these gradients (BatchNorm affine gradients: 4e-3
    # relative L2 on an H100).
    assert worst[1] < 1e-2, worst
    # phase 2: D in train mode on 2B no-grad maps with injected masks, one Adam step
    with torch.no_grad():
        student.eval()
        maps = torch.softmax(torch.cat([student(x), student(x.flip(3))], 0), 1)
    imgs = torch.cat([x, x.flip(3)], 0)
    tgt = torch.tensor([1] * B + [0] * B, device=DEV)
    keep = D.chan_keep(17, 2 * B)
    disc.train()
    disc.channel_keep = keep
    opt = torch.optim.Adam(disc.parameters(), lr=1e-4, betas=(0.9, 0.99))
    before = [q.detach().clone() for q in disc.parameters()]
    opt.zero_grad()
    F.cross_entropy(disc(maps, imgs), tgt).backward()
    opt.step()
    pd = {k: v.clone().requires_grad_(True) for k, v in pdo.items()}
    F.cross_entropy(D.forward(pd, maps.double(), imgs.double(), True, [k.to(DEV) for k in keep]), tgt).backward()
    opt_o = torch.optim.Adam(list(pd.values()), lr=1e-4, betas=(0.9, 0.99))
    opt_o.step()
    for (k, ref), got, b in zip(pd.items(), disc.parameters(), before):
        step_o, step = (ref.detach() - b.double()), (got.detach().double() - b.double())
        diff = (step - step_o).abs()
        # Adam's first step is lr * g / (|g| + eps): only where the gradient is near 0 (below 1e-3 of the tensor's largest) can the sign
        # differ, by up to 2 lr; elsewhere the steps agree up to the fp32 rounding of the stored parameter
        g = ref.grad.abs()
        near_zero = g <= 1e-3 * g.max()
        tol = 1e-3 * 1e-4 + 2 * torch.finfo(torch.float32).eps * b.double().abs()
        assert diff.max().item() <= 2e-4 + 1e-7, k
        assert bool(((diff <= tol) | near_zero).all()), (k, diff[~near_zero].max().item())
