"""Execution modes vs the fp32 reference (north_star: logits within 1e-3, label maps bit-exact).

  * at the reference-generated fixtures (2 x 1 x 32 x 32): every mode against the reference's own outputs;
  * at the BASELINE shape (N x 1 x 256 x 256, N = 4): every mode against the CPU oracle (pinned to the reference by
    tests/test_oracle_golden.py) -- the dispatcher picks the real-size kernel templates there (conv_row, conv_tc2 with MT up
    to 4, split-K weight gradients over every SM), but on a 132-SM H100 the full-resolution conv_row launches (128 row items)
    and the 64 x 64 x 64 conv_tc2 layer (128 tiles) give each CTA a single work item, and these bounds are network-level;
    tests/test_gpu_conv_at_scale.py checks every convolution launch of the training step per element against fp64 at
    N = 12 and 64, where CTAs walk several tiles;
  * at 64 x 1 x 256 x 256 on the device only: tensor-core executor vs the CUDA-core fp32 executor, layer by layer outputs are
    not exposed, so the check is on logits and on every parameter gradient.
Measured errors are printed; the asserted bounds keep <= 2x headroom over the measurements recorded in DESIGN.md section 5."""
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
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT
    from wsl4mis_b200.utils import losses as L
    from wsl4mis_b200.utils.gate_crf_loss import ModelLossSemsegGatedCRF

# logit error bounds (fraction of max |reference logit|), train-mode forward: {mode: (fixture 2x32x32, N x 256 x 256)}.
# The north-star bar is 1e-3: fp16x3 (and fp32) meet it, the 16-bit storage modes do not.
LOGIT_TOL = {"bf16": (0.09, 0.2), "fp16": (0.012, 0.025), "fp16x3": (1e-3, 1e-3), "fp32": (1e-3, 1e-3)}
# Worst relative-L2 error over the convolution weight gradients at N x 256 x 256 (fp32-accurate modes).  The yardstick is the
# oracle evaluated in fp64: the reference's own fp32 arithmetic (the fp32 oracle = torch CPU fp32) is 0.7 - 1.0e-2 away from it on
# the encoder gradients at this shape (sums of 10^5..10^6 cancelling terms behind every BatchNorm), so two correct fp32
# implementations differ by that much; measured here: fp16x3 8e-3 .. 1.0e-2 vs the fp32 oracle, 9e-3 vs the CUDA-core executor.
GRAD_TOL = {"fp16x3": 2.5e-2, "fp32": 2.5e-2}
# 16-bit storage modes: every convolution weight gradient against the oracle that rounds to the same type at the same tensors
# (kernel correctness, separated from what the storage format costs); cosine, since rounding-order noise decorrelates
GRAD_COS_EMU = {"bf16": 0.90, "fp16": 0.97}


def _build(cct, pseed, precision):
    decs = ("main_decoder", "aux_decoder1") if cct else ("decoder",)
    p = O.synth_params(1, 4, decs, pseed)
    m = (UNet_CCT if cct else UNet)(1, 4)
    m.load_state_dict(p)
    m = m.to(DEV).set_precision(precision)
    return m, p


@pytest.mark.parametrize("precision", ["fp16", "fp16x3"])
@pytest.mark.parametrize("cct", [False, True])
def test_modes_against_the_reference_fixture(golden_dir, cct, precision):
    g = np.load(os.path.join(golden_dir, "unet_cct_dmpls.npz" if cct else "unet_pce_gatedcrf.npz"))
    m, p = _build(cct, int(g["pseed"]), precision)
    n, hw = int(g["n"]), int(g["hw"])
    em = elem_masks_nchw(int(g["mseed"]), n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    if cct:
        m.channel_keep = [c.to(DEV) for c in chan_masks(int(g["cseed"]), n)]
    x = torch.from_numpy(g["image"]).to(DEV)
    errs = {}
    for mode, key in ((False, "eval_main"), (True, "train_main")):
        m.train(mode)
        with torch.no_grad():
            o = m(x)
        main = o[0] if cct else o
        ref = torch.from_numpy(g[key])
        errs[key] = (main.cpu() - ref).abs().max().item() / ref.abs().max().item()
    print(f"[{precision} cct={cct}] fixture logits: eval {errs['eval_main']:.2e}, train {errs['train_main']:.2e} of scale")
    assert errs["train_main"] < LOGIT_TOL[precision][0], errs
    assert errs["eval_main"] < LOGIT_TOL[precision][0], errs
    if precision == "fp16x3":
        assert torch.equal(main.cpu().argmax(1), ref.argmax(1))      # bit-exact label maps in the fp32-accurate tensor-core mode


REAL_N, REAL_HW = 4, 256


def _real_case(cct, variant, precision):
    """one training step at N x 1 x 256 x 256 through the script-style API, and the oracle's step on the same inputs"""
    m, p = _build(cct, 31 if cct else 29, precision)
    image, label = O.synth_batch(REAL_N, REAL_HW, REAL_HW, seed=5, frac=0.03)
    ones = [torch.ones(REAL_N, REAL_HW >> i, REAL_HW >> i, O.FT[i], dtype=torch.uint8, device=DEV) for i in range(5)]
    m.dropout_masks = dict(enumerate(ones))                      # dropout off on both sides (keep-all masks)
    keep = [(torch.arange(c) % 3 != 0).to(torch.uint8).repeat(REAL_N, 1) for c in O.FT] if cct else None
    if cct:
        m.channel_keep = [k.to(DEV) for k in keep]
    x, lab = image.to(DEV), label.to(DEV)
    m.train()
    if cct:
        o1, o2 = m(x)
        ce1, s1 = Fn.softmax_pce(o1, lab)
        ce2, s2 = Fn.softmax_pce(o2, lab)
        pseudo = Fn.mix_argmax(s1, s2, 0.37)
        pdl = L.pDLoss(4, 4)
        loss = 0.5 * (ce1 + ce2) + 0.5 * 0.5 * (pdl(s1, pseudo.unsqueeze(1)) + pdl(s2, pseudo.unsqueeze(1)))
        main = o1
    else:
        main = m(x)
        ce, s = Fn.softmax_pce(main, lab)
        loss = ce + 0.1 * ModelLossSemsegGatedCRF()(s, [{"weight": 1, "xy": 6, "rgb": 0.1}], 5, x, REAL_HW, REAL_HW)["loss"]
    loss.backward()
    torch.cuda.synchronize()
    return m, p, image, label, keep, main.detach().float().cpu(), loss.item()


_ORACLE_CACHE = {}


def _oracle(cct, p, image, label, keep, quant=None):
    """fp32 oracle step (quant None) or the storage-emulating one (quant 'bf16' / 'fp16')"""
    if (cct, quant) not in _ORACLE_CACHE:
        masks = {k: torch.ones(REAL_N, O.FT[i], REAL_HW >> i, REAL_HW >> i, dtype=torch.uint8) for i, k in enumerate(ENC_MASK_KEYS)}
        torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
        if quant == "fp64":
            p, image = {k: (v.double() if v.is_floating_point() else v) for k, v in p.items()}, image.double()
        else:
            O.QUANT, O.QUANT_SCALE = quant, float(2 ** (round(np.log2(REAL_N * REAL_HW * REAL_HW)) - 1))
        try:
            loss, grads, (main, _) = O.full_step(p, image, label, "dmpls" if cct else "pce_gatedcrf", cct, masks, keep, 0.37)
        finally:
            O.QUANT, O.QUANT_SCALE = None, 1.0
        grads, main = {k: v.float() for k, v in grads.items()}, main.float()
        _ORACLE_CACHE[(cct, quant)] = (loss.item(), grads, main)
    return _ORACLE_CACHE[(cct, quant)]


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16x3"])
@pytest.mark.parametrize("cct", [False, True])
def test_training_step_at_the_baseline_shape_against_the_oracle(cct, precision):
    """unet + pCE + GatedCRF (config 2's step) and unet_cct + DMPLS (config 3's step) at 4 x 1 x 256 x 256."""
    m, p, image, label, keep, main, loss = _real_case(cct, "dmpls" if cct else "pce_gatedcrf", precision)
    ref_loss, grads, ref = _oracle(cct, p, image, label, keep)
    scale = ref.abs().max().item()
    err = (main - ref).abs().max().item() / scale
    mism = (main.argmax(1) != ref.argmax(1)).float().mean().item()
    top2 = ref.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * LOGIT_TOL[precision][1] * scale
    named = dict(m.named_parameters())
    worst_w, worst_k, worst_aff = 0.0, None, 0.0
    for k, gr in grads.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        if named[k].grad is None:
            continue
        e = rel_l2(named[k].grad.detach().cpu(), gr)
        if named[k].dim() == 4:
            if e > worst_w:
                worst_w, worst_k = e, k
        else:
            worst_aff = max(worst_aff, e)
    print(f"[{precision} cct={cct}] 4x256x256: logits {err:.2e} of scale, label mismatch {mism:.2e}, loss {loss:.6f} vs {ref_loss:.6f}, "
          f"worst conv-weight gradient rel-L2 {worst_w:.2e} ({worst_k}), worst BN/bias gradient rel-L2 {worst_aff:.2e}")
    assert err < LOGIT_TOL[precision][1], err
    assert torch.equal(main.argmax(1)[sure], ref.argmax(1)[sure])
    if precision == "fp16x3":
        assert mism < 1e-5, mism                       # ties closer than fp32 rounding may flip; nothing else
    assert abs(loss - ref_loss) < (2e-4 if precision == "fp16x3" else 0.02) * abs(ref_loss)
    if precision in GRAD_TOL:
        _, g64, m64 = _oracle(cct, p, image, label, keep, "fp64")
        w64 = max(rel_l2(named[k].grad.detach().cpu(), g) for k, g in g64.items() if named[k].grad is not None and named[k].dim() == 4)
        r64 = max(rel_l2(grads[k], g) for k, g in g64.items() if named[k].grad is not None and named[k].dim() == 4)
        print(f"[{precision} cct={cct}] vs the fp64 oracle: logits {(main - m64).abs().max().item() / scale:.2e} of scale, worst conv-weight gradient "
              f"rel-L2 {w64:.2e} (the fp32 oracle itself: {r64:.2e})")
        assert worst_w < GRAD_TOL[precision], (worst_k, worst_w)
        assert w64 < GRAD_TOL[precision] and w64 < 3 * r64 + 1e-3, (w64, r64)
        assert worst_aff < 2 * GRAD_TOL[precision], worst_aff
    else:
        _, gq, mq = _oracle(cct, p, image, label, keep, precision)
        errq = (main - mq).abs().max().item() / mq.abs().max().item()
        cosw = {k: cosine(named[k].grad.detach().cpu(), g) for k, g in gq.items() if named[k].grad is not None and named[k].dim() == 4}
        kmin = min(cosw, key=cosw.get)
        print(f"[{precision} cct={cct}] vs the {precision}-storage emulating oracle: logits {errq:.2e} of scale, worst conv-weight gradient "
              f"cosine {cosw[kmin]:.4f} ({kmin})")
        assert errq < LOGIT_TOL[precision][1], errq
        assert cosw[kmin] > GRAD_COS_EMU[precision], (kmin, cosw[kmin])


def test_tensor_core_executor_against_the_cuda_core_executor_at_full_size():
    """64 x 1 x 256 x 256 (BASELINE config 2's per-GPU batch), device only: bf16 / fp16 / fp16x3 tensor-core steps against the
    fp32 CUDA-core executor (itself pinned to the reference at 1e-5) -- logits and every convolution weight gradient."""
    N = 64
    image, label = O.synth_batch(N, 256, 256, seed=9, frac=0.03)
    x, lab = image.to(DEV), label.to(DEV)
    ones = [torch.ones(N, 256 >> i, 256 >> i, O.FT[i], dtype=torch.uint8, device=DEV) for i in range(5)]
    res = {}
    for precision in ("fp32", "bf16", "fp16", "fp16x3"):
        m, _ = _build(False, 29, precision)
        m.dropout_masks = dict(enumerate(ones))
        m.train()
        main = m(x)
        ce, s = Fn.softmax_pce(main, lab)
        loss = ce + 0.1 * ModelLossSemsegGatedCRF()(s, [{"weight": 1, "xy": 6, "rgb": 0.1}], 5, x, 256, 256)["loss"]
        loss.backward()
        torch.cuda.synchronize()
        res[precision] = (main.detach().float(), {k: v.grad.detach().clone() for k, v in m.named_parameters() if v.grad is not None and v.dim() == 4})
        del m
        torch.cuda.empty_cache()
    ref, gref = res["fp32"]
    scale = ref.abs().max().item()
    for precision in ("bf16", "fp16", "fp16x3"):
        main, gr = res[precision]
        err = (main - ref).abs().max().item() / scale
        worst = max(rel_l2(gr[k], gref[k]) for k in gref)
        mism = (main.argmax(1) != ref.argmax(1)).float().mean().item()
        print(f"[{precision}] 64x256x256 vs CUDA-core fp32: logits {err:.2e} of scale, label mismatch {mism:.2e}, worst conv-weight gradient rel-L2 {worst:.2e}")
        assert err < LOGIT_TOL[precision][1], (precision, err)
        if precision in GRAD_TOL:
            assert worst < GRAD_TOL[precision], (precision, worst)
            assert mism < 1e-5, mism
