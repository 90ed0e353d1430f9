"""Whole-network parity: UNet / UNet_CCT on the fused executor vs the reference-generated golden fixtures
and vs the CPU oracle on the same seeded inputs and weights.

The reference computes in fp32; the executor stores activations in bf16 (8-bit mantissa) with fp32
accumulation, statistics and master weights.  Tolerances are therefore stated relative to the logit /
gradient scale and were chosen from the measured error (see DESIGN.md 'Precision'), not from the 1e-3
north-star target, which bf16 storage cannot meet (reported, not hidden)."""
import os

import numpy as np
import pytest
import torch

import wsl_oracle as O
from _gpu_util import chan_masks, cosine, elem_masks_nchw, rel_l2, ENC_MASK_KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200 import functional as Fn
    from wsl4mis_b200.networks.net_factory import net_factory
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT
    from wsl4mis_b200.utils import losses as L
    from wsl4mis_b200.utils.gate_crf_loss import ModelLossSemsegGatedCRF

# Tolerances.  Two references are used:
#  * the fp32 reference fixtures -> what bf16 STORAGE costs (8-bit mantissa through 23 BN-normalised layers on a 2-image
#    batch: measured 1.3 % of the logit scale in eval, 5.5 % in train mode; the oracle's own bf16-storage emulation
#    (wsl_oracle.QUANT) shows the same 4.5 % / gradient cosine 0.85 against fp32, so this is precision, not a kernel bug);
#  * the oracle with bf16-storage emulation -> kernel correctness, tight.
EVAL_TOL_FP32 = 0.03
TRAIN_TOL_FP32 = 0.09
LOGIT_TOL_Q = 0.06    # vs bf16-emulating oracle (2-image BN at a 2x2 bottleneck amplifies 1-ulp rounding differences; measured 0.035-0.045)
GRAD_COS_Q = 0.93     # vs bf16-emulating oracle: cosine of every weight gradient (measured >= 0.97)
GRAD_COS_FP32 = 0.70  # vs fp32 oracle (bf16 storage noise on a 2-image batch)


def _model(cct, g, use_tc=True):
    decs = ("main_decoder", "aux_decoder1") if cct else ("decoder",)
    p = O.synth_params(1, 4, decs, int(g["pseed"]))
    m = (UNet_CCT if cct else UNet)(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV)
    m.executor.use_tc = use_tc
    return m, p


def _set_masks(m, g, cct):
    n, hw = int(g["n"]), int(g["hw"])
    em = elem_masks_nchw(int(g["mseed"]), n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    ck = None
    if cct:
        ck = chan_masks(int(g["cseed"]), n)
        m.channel_keep = [c.to(DEV) for c in ck]
    return {k: e for k, e in zip(ENC_MASK_KEYS, em)}, ck


@pytest.mark.parametrize("use_tc", [True, False])
@pytest.mark.parametrize("cct", [False, True])
def test_forward_matches_golden(golden_dir, cct, use_tc):
    g = np.load(os.path.join(golden_dir, "unet_cct_dmpls.npz" if cct else "unet_pce_gatedcrf.npz"))
    m, _ = _model(cct, g, use_tc)
    _set_masks(m, g, cct)
    x = torch.from_numpy(g["image"]).to(DEV)
    m.eval()
    with torch.no_grad():
        o = m(x)
    main = o[0] if cct else o
    ref = torch.from_numpy(g["eval_main"])
    err = (main.cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < EVAL_TOL_FP32, ("eval", err)
    if cct:
        ra = torch.from_numpy(g["eval_aux"])
        assert (o[1].cpu() - ra).abs().max().item() / ra.abs().max().item() < EVAL_TOL_FP32
    m.train()
    with torch.no_grad():
        o = m(x)
    main = o[0] if cct else o
    ref = torch.from_numpy(g["train_main"])
    err = (main.cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < TRAIN_TOL_FP32, ("train", err)
    # label maps: bit-exact wherever the reference's top-2 margin exceeds the measured logit error
    top2 = ref.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * TRAIN_TOL_FP32 * ref.abs().max()
    assert torch.equal(main.cpu().argmax(1)[sure], ref.argmax(1)[sure])
    assert sure.float().mean().item() > 0.3
    # kernel correctness: against the oracle emulating bf16 storage at the same points
    n, hw = int(g["n"]), int(g["hw"])
    p = O.synth_params(1, 4, ("main_decoder", "aux_decoder1") if cct else ("decoder",), int(g["pseed"]))
    om = {k: e for k, e in zip(ENC_MASK_KEYS, elem_masks_nchw(int(g["mseed"]), n, hw, hw))}
    ock = chan_masks(int(g["cseed"]), n) if cct else None
    O.QUANT = True
    try:
        with torch.no_grad():
            img = torch.from_numpy(g["image"])
            q = O.unet_cct_forward(p, img, True, om, ock)[0] if cct else O.unet_forward(p, img, True, om)
    finally:
        O.QUANT = None
    errq = (main.cpu() - q).abs().max().item() / q.abs().max().item()
    print(f"[cct={cct} tc={use_tc}] logits vs fp32 ref: {err:.4f}; vs bf16-emulating oracle: {errq:.4f}")
    assert errq < LOGIT_TOL_Q, errq


@pytest.mark.parametrize("cct", [False, True])
def test_backward_matches_oracle_and_golden(golden_dir, cct):
    g = np.load(os.path.join(golden_dir, "unet_cct_dmpls.npz" if cct else "unet_pce_gatedcrf.npz"))
    m, p = _model(cct, g)
    om, ock = _set_masks(m, g, cct)
    x = torch.from_numpy(g["image"]).to(DEV)
    lab = torch.from_numpy(g["label"]).to(DEV)
    m.train()
    if cct:
        beta = float(g["beta"])
        o1, o2 = m(x)
        ce1, s1 = Fn.softmax_pce(o1, lab)
        ce2, s2 = Fn.softmax_pce(o2, lab)
        pseudo = Fn.mix_argmax(s1, s2, beta)
        pdl = L.pDLoss(4, 4)
        loss = 0.5 * (ce1 + ce2) + 0.5 * 0.5 * (pdl(s1, pseudo.unsqueeze(1)) + pdl(s2, pseudo.unsqueeze(1)))
    else:
        o = m(x)
        ce, s = Fn.softmax_pce(o, lab)
        loss = ce + 0.1 * ModelLossSemsegGatedCRF()(s, [{"weight": 1, "xy": 6, "rgb": 0.1}], 5, x, 32, 32)["loss"]
    loss.backward()
    torch.cuda.synchronize()
    ref_loss = float(g["loss"])
    assert abs(loss.item() - ref_loss) < 0.02 * abs(ref_loss), (loss.item(), ref_loss)
    # oracle gradients on the same inputs: fp32 and bf16-storage emulation (CPU)
    args = (p, torch.from_numpy(g["image"]), torch.from_numpy(g["label"]), "dmpls" if cct else "pce_gatedcrf", cct, om, ock,
            float(g["beta"]) if cct else 0.5)
    _, grads, _ = O.full_step(*args)
    O.QUANT = True
    try:
        _, gradsq, _ = O.full_step(*args)
    finally:
        O.QUANT = None
    keys = [str(k) for k in g["grad_keys"]]
    stats = g["grad_stats"]
    named = dict(m.named_parameters())
    worst = worstq = 1.0
    for k, (_, _, l2) in zip(keys, stats):
        mine = named[k].grad.detach().cpu()
        ref = grads[k]
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            # conv bias directly before BatchNorm: the true gradient is 0, both sides hold rounding noise
            assert mine.abs().max().item() < 1e-3 * max(1.0, stats[:, 1].max())
            continue
        c, cq = cosine(mine, ref), cosine(mine, gradsq[k])
        worst, worstq = min(worst, c), min(worstq, cq)
        assert cq > GRAD_COS_Q, (k, cq, c)
        assert c > GRAD_COS_FP32, (k, c)
        assert abs(mine.double().norm().item() - gradsq[k].double().norm().item()) < 0.35 * gradsq[k].norm().item() + 1e-6, k  # BN affine grads are cancelling sums: noisy in bf16
    print(f"[cct={cct}] worst gradient cosine vs fp32 oracle {worst:.4f}, vs bf16-emulating oracle {worstq:.4f}")
    # running statistics were updated in place like nn.BatchNorm2d does
    if not cct:
        sd = m.state_dict()
        for k in [f for f in g.files if f.startswith("stat:")]:
            assert np.allclose(sd[k[5:]].cpu().numpy(), g[k], rtol=5e-2, atol=1e-2), k   # bf16 conv outputs feed the batch mean
        assert int(sd["encoder.in_conv.conv_conv.1.num_batches_tracked"]) == 1


@pytest.mark.parametrize("cct", [False, True])
def test_fp32_parity_mode_meets_the_north_star_tolerance(golden_dir, cct):
    """precision='fp32' (activations and gradients stored in fp32, CUDA-core convolutions): logits within 1e-3 of the
    reference (north_star's bar; measured ~1e-6), label maps bit-exact, every gradient within 1e-3 relative L2."""
    g = np.load(os.path.join(golden_dir, "unet_cct_dmpls.npz" if cct else "unet_pce_gatedcrf.npz"))
    decs = ("main_decoder", "aux_decoder1") if cct else ("decoder",)
    p = O.synth_params(1, 4, decs, int(g["pseed"]))
    m = (UNet_CCT if cct else UNet)(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV).set_precision("fp32")
    om, ock = _set_masks(m, g, cct)
    x = torch.from_numpy(g["image"]).to(DEV)
    lab = torch.from_numpy(g["label"]).to(DEV)
    m.eval()
    with torch.no_grad():
        o = m(x)
    for mine, key in ((o[0] if cct else o, "eval_main"),) + (((o[1], "eval_aux"),) if cct else ()):
        ref = torch.from_numpy(g[key])
        assert (mine.cpu() - ref).abs().max().item() / ref.abs().max().item() < 1e-3, key
    m.train()
    if cct:
        beta = float(g["beta"])
        o1, o2 = m(x)
        ce1, s1 = Fn.softmax_pce(o1, lab)
        ce2, s2 = Fn.softmax_pce(o2, lab)
        pseudo = Fn.mix_argmax(s1, s2, beta)
        assert np.array_equal(pseudo.cpu().numpy(), g["pseudo"])          # bit-exact dynamically mixed pseudo labels
        pdl = L.pDLoss(4, 4)
        loss = 0.5 * (ce1 + ce2) + 0.5 * 0.5 * (pdl(s1, pseudo.unsqueeze(1)) + pdl(s2, pseudo.unsqueeze(1)))
        main = o1
    else:
        main = m(x)
        ce, s = Fn.softmax_pce(main, lab)
        loss = ce + 0.1 * ModelLossSemsegGatedCRF()(s, [{"weight": 1, "xy": 6, "rgb": 0.1}], 5, x, 32, 32)["loss"]
    ref = torch.from_numpy(g["train_main"])
    err = (main.detach().cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-3, err
    assert torch.equal(main.detach().cpu().argmax(1), ref.argmax(1))      # bit-exact label maps
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - float(g["loss"])) < 1e-4 * abs(float(g["loss"]))
    _, grads, _ = O.full_step(p, torch.from_numpy(g["image"]), torch.from_numpy(g["label"]), "dmpls" if cct else "pce_gatedcrf",
                              cct, om, ock, float(g["beta"]) if cct else 0.5)
    named = dict(m.named_parameters())
    worst = 0.0
    for k, (_, _, l2) in zip([str(k) for k in g["grad_keys"]], g["grad_stats"]):
        mine = named[k].grad.detach().cpu()
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            assert mine.abs().max().item() < 1e-4          # true gradient is zero (conv bias in front of BatchNorm)
            continue
        e = rel_l2(mine, grads[k])
        worst = max(worst, e)
        assert e < 1e-3, (k, e)
        assert abs(mine.double().norm().item() - l2) < 2e-3 * l2 + 1e-7, k
    print(f"[fp32 cct={cct}] logits err {err:.2e} of scale, worst gradient rel-L2 {worst:.2e}")


def test_script_style_step_with_torch_optimizer():
    """The per-step body of train_weakly_supervised_pCE_GatedCRFLoss_2D.py:111-126 written exactly as the
    script does (torch CrossEntropyLoss, torch.softmax, optim.SGD) on net_factory's model: loss decreases."""
    torch.manual_seed(2022)
    model = net_factory("unet", in_chns=1, class_num=4)
    assert net_factory("nope") is None
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    ce_loss = torch.nn.CrossEntropyLoss(ignore_index=4)
    crf = ModelLossSemsegGatedCRF()
    img, lab = O.synth_batch(4, 64, 64, seed=1, frac=0.05)
    img, lab = img.to(DEV), lab.to(DEV)
    model.train()
    hist = []
    for it in range(12):
        out = model(img)
        soft = torch.softmax(out, dim=1)
        l_ce = ce_loss(out, lab[:].long())
        l_crf = crf(soft, [{"weight": 1, "xy": 6, "rgb": 0.1}], 5, img, 64, 64)["loss"]
        loss = l_ce + 0.1 * l_crf
        opt.zero_grad()
        loss.backward()
        opt.step()
        hist.append(l_ce.item())
    assert hist[-1] < hist[0] - 0.05, hist


def test_rng_dropout_is_fresh_each_step_and_eval_is_deterministic():
    torch.manual_seed(0)
    m = UNet(1, 4).to(DEV)
    x = torch.rand(2, 1, 32, 32, device=DEV)
    m.train()
    with torch.no_grad():
        a, b = m(x), m(x)
    assert not torch.equal(a, b)
    m.eval()
    with torch.no_grad():
        c, d = m(x), m(x)
    assert torch.equal(c, d)


def test_wide_rows_take_the_row_kernel_and_match_the_oracle():
    """2 x 1 x 32 x 128: rows of 128 pixels route the full-resolution 16-channel layers (forward with fused statistics, data
    gradients, out_conv) through conv_row; the whole step is checked against the bf16-storage-emulating oracle."""
    torch.manual_seed(5)
    N, H, W = 2, 32, 128
    p = O.synth_params(1, 4, ("main_decoder", "aux_decoder1"), 21)
    m = UNet_CCT(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV)
    m.dropout_masks = {i: torch.ones(N, H >> i, W >> i, O.FT[i], dtype=torch.uint8, device=DEV) for i in range(5)}
    keep = [(torch.arange(c) % 3 != 0).to(torch.uint8).repeat(N, 1) for c in O.FT]
    m.channel_keep = [k.to(DEV) for k in keep]
    image, label = O.synth_batch(N, H, W, seed=12, frac=0.05)
    m.train()
    o1, o2 = m(image.to(DEV))
    ce1, s1 = Fn.softmax_pce(o1, label.to(DEV))
    ce2, s2 = Fn.softmax_pce(o2, label.to(DEV))
    loss = 0.5 * (ce1 + ce2)
    loss.backward()
    torch.cuda.synchronize()
    names = ["encoder.in_conv.conv_conv.3"] + [f"encoder.down{j}.maxpool_conv.1.conv_conv.3" for j in range(1, 5)]
    masks = {k: torch.ones(N, O.FT[i], H >> i, W >> i, dtype=torch.uint8) for i, k in enumerate(names)}

    def oracle():
        leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
        a, b = O.unet_cct_forward(leaves, image, True, masks, keep)
        l = 0.5 * (O.pce_loss(a, label) + O.pce_loss(b, label))
        ks = [k for k, v in leaves.items() if v.requires_grad]
        return a.detach(), b.detach(), l.detach(), dict(zip(ks, torch.autograd.grad(l, [leaves[k] for k in ks])))

    O.QUANT = True
    try:
        a, b, lq, gq = oracle()
    finally:
        O.QUANT = None
    for mine, ref in ((o1, a), (o2, b)):
        err = (mine.detach().float().cpu() - ref).abs().max().item() / ref.abs().max().item()
        assert err < LOGIT_TOL_Q, err
    assert abs(loss.item() - lq.item()) < 0.03 * abs(lq.item())
    named = dict(m.named_parameters())
    worst = {}
    for k, ref in gq.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        worst[k] = cosine(named[k].grad.detach().cpu(), ref)
    # convolution weights: tight; BatchNorm affine gradients are cancelling sums over a 2-image batch and sit at 0.90-0.93 on
    # this input, so they get the looser bound
    bad = {k: round(v, 4) for k, v in worst.items() if v <= (GRAD_COS_Q if named[k].dim() == 4 else 0.85)}
    print("worst cosines:", sorted(worst.items(), key=lambda kv: kv[1])[:6])
    assert not bad, bad


def _ds_case(golden_dir, precision):
    g = np.load(os.path.join(golden_dir, "unet_heads.npz"))
    n, hw = int(g["n"]), int(g["hw"])
    p = O.synth_params(1, 4, ("decoder",), int(g["pseed"]), ds=True)
    from wsl4mis_b200.networks.unet import UNet_DS
    m = UNet_DS(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV)
    if precision == "fp32":
        m.set_precision("fp32")
    em = elem_masks_nchw(int(g["mseed"]), n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    return g, p, m, {k: e for k, e in zip(ENC_MASK_KEYS, em)}


def test_unet_ds_fp32_mode_matches_the_reference_fixture(golden_dir):
    """UNet_DS (SURVEY 8(f) rank 4): four outputs, loss = sum of the heads' pCE, every parameter gradient, in the fp32 parity
    mode against the fixture generated from the unmodified reference class."""
    g, p, m, _ = _ds_case(golden_dir, "fp32")
    x, lab = torch.from_numpy(g["image"]).to(DEV), torch.from_numpy(g["label"]).to(DEV)
    m.train()
    outs = m(x)
    assert len(outs) == 4
    for i, o in enumerate(outs):
        ref = torch.from_numpy(g[f"ds:out{i}"])
        err = (o.detach().cpu() - ref).abs().max().item() / ref.abs().max().item()
        assert err < 1e-3, (i, err)
        assert torch.equal(o.detach().cpu().argmax(1), ref.argmax(1)) or err < 1e-5
    loss = sum(Fn.softmax_pce(o, lab)[0] for o in outs)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - float(g["ds:loss"])) < 1e-3 * abs(float(g["ds:loss"]))
    named = dict(m.named_parameters())
    keys = [str(k) for k in g["ds:grad_keys"]]
    errs = {}
    for k, (_, asum, l2) in zip(keys, g["ds:grad_stats"]):
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        assert named[k].grad is not None, k
        errs[k] = abs(named[k].grad.double().norm().item() - l2) / (l2 + 1e-12)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    print("[unet_ds fp32] worst gradient-norm errors:", [(k, f"{v:.2e}") for k, v in worst])
    # convolution weights: 2e-3; BatchNorm affine gradients (cancelling sums, formed from raw moments in bn_bwd_reduce): 1e-2
    bad = {k: v for k, v in errs.items() if v > (2e-3 if named[k].dim() == 4 else 1e-2)}
    assert not bad, bad
    for k in (str(k) for k in g["ds:no_grad_keys"]):        # out_conv_dp4 never runs: no gradient, exactly like autograd
        assert named[k].grad is None, k


def test_unet_ds_bf16_path_matches_the_quant_oracle(golden_dir):
    g, p, m, om = _ds_case(golden_dir, "bf16")
    x = torch.from_numpy(g["image"])
    m.train()
    with torch.no_grad():
        outs = m(x.to(DEV))
    O.QUANT = True
    try:
        with torch.no_grad():
            ref = O.unet_ds_forward(p, x, True, om)
    finally:
        O.QUANT = None
    for i, (o, r) in enumerate(zip(outs, ref)):
        err = (o.cpu() - r).abs().max().item() / r.abs().max().item()
        assert err < LOGIT_TOL_Q, (i, err)


def test_unet_ds_wide_input_runs_the_tensor_core_heads():
    """64 x 128 input: the dp1 / dp2 heads take the wgmma kernels; outputs against the bf16-emulating oracle, backward runs."""
    from wsl4mis_b200.networks.unet import UNet_DS
    N, H, W = 2, 64, 128
    p = O.synth_params(1, 4, ("decoder",), 41, ds=True)
    m = UNet_DS(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV)
    m.dropout_masks = {i: torch.ones(N, H >> i, W >> i, O.FT[i], dtype=torch.uint8, device=DEV) for i in range(5)}
    image, label = O.synth_batch(N, H, W, seed=14, frac=0.05)
    m.train()
    outs = m(image.to(DEV))
    loss = sum(Fn.softmax_pce(o, label.to(DEV))[0] for o in outs)
    loss.backward()
    torch.cuda.synchronize()
    masks = {k: torch.ones(N, O.FT[i], H >> i, W >> i, dtype=torch.uint8) for i, k in enumerate(ENC_MASK_KEYS)}
    O.QUANT = True
    try:
        leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
        ref = O.unet_ds_forward(leaves, image, True, masks)
        lq = sum(O.pce_loss(r, label) for r in ref)
        ks = [k for k, v in leaves.items() if v.requires_grad and "dp4" not in k]
        gq = dict(zip(ks, torch.autograd.grad(lq, [leaves[k] for k in ks])))
    finally:
        O.QUANT = None
    for i, (o, r) in enumerate(zip(outs, ref)):
        err = (o.detach().cpu() - r.detach()).abs().max().item() / r.detach().abs().max().item()
        assert err < LOGIT_TOL_Q, (i, err)
    named = dict(m.named_parameters())
    for k, r in gq.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        if named[k].dim() == 4:
            assert cosine(named[k].grad.detach().cpu(), r) > GRAD_COS_Q, k


def _3h_case(golden_dir, precision):
    from torch.distributions.uniform import Uniform
    from wsl4mis_b200.networks.unet import UNet_CCT_3H
    g = np.load(os.path.join(golden_dir, "unet_heads.npz"))
    n, hw = int(g["n"]), int(g["hw"])
    p = O.synth_params(1, 4, ("main_decoder", "aux_decoder1", "aux_decoder2"), int(g["pseed"]))
    m = UNet_CCT_3H(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV).set_precision(precision)
    em = elem_masks_nchw(int(g["mseed"]), n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    m.channel_keep = [c.to(DEV) for c in chan_masks(int(g["cseed"]), n)]
    torch.manual_seed(int(g["nseed"]))               # the reference's FeatureNoise draws, in feature order (unet.py:369)
    m.feature_noise = [Uniform(-0.3, 0.3).sample((O.FT[i], hw >> i, hw >> i)) for i in range(5)]
    return g, m


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
def test_unet_cct_3h_matches_the_reference_fixture(golden_dir, precision):
    """UNet_CCT_3H (SURVEY 8(f) rank 4): three outputs -- main, aux_decoder1 on channel-dropped features, aux_decoder1 AGAIN on
    FeatureNoise'd features (unet.py:363-371) -- loss = sum of the heads' pCE, every parameter gradient (aux_decoder1 accumulates both
    passes, aux_decoder2 gets none), against the fixture generated from the unmodified reference class."""
    g, m = _3h_case(golden_dir, precision)
    x, lab = torch.from_numpy(g["image"]).to(DEV), torch.from_numpy(g["label"]).to(DEV)
    m.train()
    outs = m(x)
    assert len(outs) == 3
    for i, o in enumerate(outs):
        ref = torch.from_numpy(g[f"3h:out{i}"])
        err = (o.detach().cpu() - ref).abs().max().item() / ref.abs().max().item()
        assert err < 1e-3, (i, err)
    loss = sum(Fn.softmax_pce(o, lab)[0] for o in outs)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - float(g["3h:loss"])) < 1e-3 * abs(float(g["3h:loss"]))
    named = dict(m.named_parameters())
    errs = {}
    for k, (_, asum, l2) in zip([str(k) for k in g["3h:grad_keys"]], g["3h:grad_stats"]):
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        assert named[k].grad is not None, k
        errs[k] = abs(named[k].grad.double().norm().item() - l2) / (l2 + 1e-12)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print(f"[unet_cct_3h {precision}] worst gradient-norm errors:", [(k, f"{v:.2e}") for k, v in worst])
    bad = {k: v for k, v in errs.items() if v > (2e-3 if named[k].dim() == 4 else 1e-2)}
    assert not bad, bad
    for k in (str(k) for k in g["3h:no_grad_keys"]):        # aux_decoder2 never runs: no gradient, exactly like autograd
        assert named[k].grad is None, k


def test_unet_cct_3h_bf16_runs_with_its_own_noise():
    """default mode, no injected randomness: three finite outputs, a backward pass, fresh FeatureNoise every forward"""
    from wsl4mis_b200.networks.net_factory import net_factory
    torch.manual_seed(3)
    m = net_factory("unet_cct_3h", in_chns=1, class_num=4)
    x = torch.rand(2, 1, 64, 64, device=DEV)
    m.train()
    a = m(x)
    b = m(x)
    assert len(a) == 3 and all(torch.isfinite(o).all() for o in a)
    assert not torch.equal(a[2], b[2])
    sum(o.float().mean() for o in a).backward()
    assert next(m.aux_decoder1.parameters()).grad is not None and next(m.aux_decoder2.parameters()).grad is None
