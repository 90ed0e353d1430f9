"""Every loss-head launch of the training steps (wsl4mis_b200/csrc/losses.cu: softmax + pCE, the logit-gradient head, Gated CRF,
Mumford-Shah, Dice, TV, entropy, class variance, the mean-teacher consistency and its teacher noise, rot90, the EMA update,
mixed pseudo labels and the Scribble2Label head), replayed at the steps' own shapes and checked per element against fp64
(tests/_loss_check.py states the references and the bounds).

The launches are harvested as tests/test_gpu_netops_at_scale.py harvests its own: one eager step per configuration runs with a
LaunchRecorder in place of wsl4mis_b200._lib.PROFILE, which keeps each distinct (entry point, scalar arguments, NULL pointer
arguments) of the losses.cu entry points.  The configurations follow profiles/step_launches.py at the scripts' sizes: every
TrainStep variant on UNet_CCT at 12 x 256 x 256 in bf16, fp16 (loss scale S != 1) and fp32 (NCHW dlogits); pce_gatedcrf and pce_ms
at batch 64 (the benchmark's batch: 4096 CRF tiles, more than WSL_MAX_PARTIAL_BLOCKS, so the grid-stride path); UAMT (T = 8), mean
teacher (T = 0), entropy minimisation and DAN at 6 + 6; USTM at rot90 counts 0-3; Scribble2Label before and after thr_iter.

Each distinct launch is replayed once on fresh operands seeded from its key: logits with per-pixel scales 2^-4 .. 2^5, a saturated
band (probabilities exactly 0 and 1: log(p + 1e-6) at p = 0, sign(0), TV ties), a band where two classes tie exactly, and sample 0
without class 3 (a zero class std); labels 0-3 plus ignore 4 at a different rate per sample; images of flat blocks and edges in
[0, 1] with a dark top-left corner (the CRF's out-of-bounds term); u-label weights exactly at thr_conf; regulariser gradients of
mean-type size.  Values the step keeps in device memory (beta, the threshold, the ramp weight, thr_conf / w_u, the noise seed
offset) are set by the replay; S2L runs both with w_u = 0 and w_u = 0.5.  Consumers run on the producing kernel's fp32 outputs.

Beyond the recorded calls: every reduction runs twice back to back on one workspace and must give bit-identical results (the
ticket reset); every backward with an accumulate flag runs again with accumulate = 1 and must double; the 16-bit logit gradient is
also written next to the fp32 one and must be its round-to-nearest; a Gated CRF at 3 x 4 x 232 x 200 puts partial tiles on the
right and bottom edges; the functional pDice runs wsl_mask_count on ragged ignore masks; no-label batches give NaN losses with zero
gradients; and each planted fault of tests/test_loss_check_cpu.py, applied to a copy of a real kernel output, fails its bound."""
import gc
import math
import os
import re
import time
import zlib

import numpy as np
import pytest
import torch

import _loss_check as L
import wsl_oracle as O
from _gpu_util import LaunchRecorder

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if torch.cuda.is_available():
    from wsl4mis_b200 import _lib
    from wsl4mis_b200._lib import LIB, call
    from wsl4mis_b200.engine import DANStep, EntropyMinStep, MeanTeacherStep, S2LStep, TrainStep, UAMTStep, USTMStep, VARIANTS
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT


def loss_entry_points():
    src = open(os.path.join(ROOT, "wsl4mis_b200", "csrc", "losses.cu")).read()
    return set(re.findall(r"WSL_API int (wsl_\w+)\(", src))


# losses.cu entry points other files check: the validation path (bitwise in test_gpu_val.py / test_gpu_train.py) and the
# deep-supervision resize (test_gpu_netops_at_scale.py); wsl_mix_argmax without p2 is the validation argmax
LEFT_TO_OTHERS = {"wsl_zoom_nearest", "wsl_zoom_nearest_ragged", "wsl_overlap_counts", "wsl_nearest_resize_fwd", "wsl_nearest_resize_bwd"}
SEED_OFFSET = 0x2545F4914F6CDD1D
THR_CONF = float(np.float32(0.8))
_HARVEST, _REPLAYS = {}, {}
PEAK = {"mib": 0.0}


# ------------------------------------------------------------------------------------------------------------ harvest
def _batch(B, hw, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 1, hw, hw, generator=g).to(DEV), torch.randint(0, 4, (B, hw, hw), generator=g, dtype=torch.uint8).to(DEV)


def _scribbles(lab, seed):
    g = torch.Generator().manual_seed(seed)
    keep = (torch.rand(tuple(lab.shape), generator=g) < 0.1).to(DEV)
    return torch.where(keep, lab, torch.full_like(lab, 4))


STEP_VARIANTS = ("pce", "pce_gatedcrf", "pce_ms", "pce_tv", "dmpls", "pce_entropy", "pce_variance", "ce_dice")   # engine.VARIANTS


def _configs():
    cfg = {}
    for v in STEP_VARIANTS:
        for prec in ("bf16", "fp16", "fp32"):
            cfg[f"train-{v}-{prec}-n12"] = ("train", v, prec, 12)
    cfg["train-pce_gatedcrf-bf16-n64"] = ("train", "pce_gatedcrf", "bf16", 64)
    cfg["train-pce_ms-bf16-n64"] = ("train", "pce_ms", "bf16", 64)
    for m in ("uamt", "mt", "em", "dan"):
        cfg[f"{m}-6+6"] = (m, None, "bf16", 6)
    for k in range(4):
        cfg[f"ustm-rot{k}-n12"] = ("ustm", k, "bf16", 12)
    cfg["s2l-before-n12"] = ("s2l", 0, "bf16", 12)
    cfg["s2l-after-n12"] = ("s2l", 10, "bf16", 12)
    return cfg


CONFIGS = _configs()


def _step_and_call(config):
    kind, arg, prec, N = CONFIGS[config]
    torch.manual_seed(11)
    if kind == "train":
        step = TrainStep(UNet_CCT(1, 4).to(DEV).set_precision(prec), arg, graph=False)
        step.iter_num = 900
        img, lab = _batch(N, 256, 13)
        return lambda: step(img, _scribbles(lab, 14))
    if kind == "s2l":
        step = S2LStep(UNet(1, 4).to(DEV).set_precision(prec), thr_iter=5, graph=False)
        step.iter_num = arg
        img, lab = _batch(N, 256, 16)
        w = torch.softmax(torch.rand(N, 256, 256, 4, generator=torch.Generator().manual_seed(17)) * 4, -1).to(DEV)
        return lambda: step(img, _scribbles(lab, 18), w)
    if kind == "ustm":
        step = USTMStep(UNet(1, 4).to(DEV), UNet(1, 4).to(DEV))
        step.iter_num = 5000
        img, lab = _batch(N, 256, 23)
        return lambda: step(img, _scribbles(lab, 24), rot_times=arg)
    s = UNet(1, 4).to(DEV)
    if kind == "em":
        step = EntropyMinStep(s)
    elif kind == "dan":
        step = DANStep(s, FCDiscriminator(4).to(DEV), graph=False)
    else:
        step = (UAMTStep if kind == "uamt" else MeanTeacherStep)(s, UNet(1, 4).to(DEV))
    step.iter_num = 900
    img_l, lab_l = _batch(N, 256, 20)
    img_u, _ = _batch(N, 256, 21)
    return lambda: step(img_l, lab_l, img_u)


def _harvest(config):
    if config not in _HARVEST:
        entries = loss_entry_points()
        run = _step_and_call(config)
        rec, saved = LaunchRecorder(lambda name: name in entries), _lib.PROFILE
        _lib.PROFILE = rec
        try:
            run()
            torch.cuda.synchronize()
        finally:
            _lib.PROFILE = saved
        del run
        gc.collect()                                   # the step's model and executor buffers
        torch.cuda.empty_cache()
        _HARVEST[config] = rec.launches
    return _HARVEST[config]


# ------------------------------------------------------------------------------------------------------------ operands
def _logits(N, H, W, g, shift=0):
    """[N,4,H,W]: per-pixel scales 2^-4 .. 2^5, a saturated band, a band where classes 1 and 2 tie, no class 3 in sample 0"""
    scale = 2.0 ** (torch.rand(N, 1, H, W, device=DEV, generator=g) * 9 - 4)
    x = torch.randn(N, 4, H, W, device=DEV, generator=g) * scale
    r0 = (H // 8 + shift) % (H - H // 8)
    band = x[:, :, r0:r0 + H // 8]
    band.fill_(-200.0)
    for n in range(N):
        band[n, n % 4] = 200.0
    r1 = (H // 2 + shift) % (H - H // 16)
    t = x[:, :, r1:r1 + H // 16]
    t[:, 1] = t[:, 2] = t.max(1).values + 0.5
    x[0, 3] = -300.0
    return x.contiguous()


def _probs(x):
    """the producing kernel's fp32 softmax"""
    N, C, H, W = x.shape
    p = torch.empty_like(x)
    call("wsl_softmax_pce_fwd", x, None, p, N, C, H, W, 255, torch.zeros(2, device=DEV), _ws())
    return p


def _labels(N, H, W, g, ignore=4):
    """0-3 and, with ignore 4, the ignore label at a rate from 30 % to 97 % depending on the sample"""
    lab = torch.randint(0, 4, (N, H, W), device=DEV, generator=g, dtype=torch.uint8)
    if ignore != 4:
        return lab
    rate = torch.linspace(0.3, 0.97, N, device=DEV).view(N, 1, 1)
    return torch.where(torch.rand(N, H, W, device=DEV, generator=g) < rate, torch.full_like(lab, 4), lab)


def _image(N, H, W, g):
    lev = torch.rand(N, 1, max(1, H // 16), max(1, W // 16), device=DEV, generator=g)
    img = torch.nn.functional.interpolate(lev, size=(H, W), mode="nearest")
    ramp = torch.linspace(0, 0.2, W, device=DEV).view(1, 1, 1, W)
    img = (img * 0.8 + ramp).clamp(0, 1)
    img[:, :, : H // 5, : W // 5] = 0.0
    return img.contiguous()


def _gprobs(N, H, W, g):
    """a regulariser's probability gradient: mean-type size 2^-4 .. 2^4 / (N H W)"""
    return (torch.randn(N, 4, H, W, device=DEV, generator=g) * 2.0 ** (torch.rand(N, 1, H, W, device=DEV, generator=g) * 8 - 4)
            / (N * H * W)).contiguous()


def _ws():
    return torch.zeros(LIB.load().wsl_workspace_floats(), device=DEV)


def _nchw(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _rep(got, ref, bound, what, shape=None):
    return L.report(_nchw(got) if got.dim() == 4 else got.reshape(-1, 1), _nchw(ref) if ref.dim() == 4 else ref.reshape(-1, 1),
                    _nchw(bound) if bound.dim() == 4 else bound.reshape(-1, 1), shape, what=what)


def _same(a, b, what):
    ok = torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)
    return {"worst": 0.0 if ok else math.inf, "bad": 0 if ok else 1, "msg": None if ok else f"{what}: two back-to-back runs differ"}


def _acc(name, args, idx_acc, idx_out, ref, bound, what):
    """rerun a backward with accumulate = 1 on its own result: the doubled reference within twice the bound"""
    args = list(args)
    args[idx_acc] = 1
    call(name, *args)
    got = args[idx_out]
    return _rep(got, 2 * ref, 2 * bound + 2.0 ** -24 * 2 * ref.abs(), what + " (accumulate = 1)", _shape4(ref))


def _shape4(t):
    return (t.shape[0], t.shape[2], t.shape[3]) if t.dim() == 4 else None


# ------------------------------------------------------------------------------------------------------------ replays
def _r_softmax_pce(a, null, g):
    N, H, W, ig = a["N"], a["H"], a["W"], a["ignore_index"]
    x = _logits(N, H, W, g)
    lab = None if "label" in null else _labels(N, H, W, g, ig)
    reps, outs = [], []
    ws = _ws()
    for _ in range(2):
        p, st = torch.empty_like(x), torch.zeros(2, device=DEV)
        call("wsl_softmax_pce_fwd", x, lab, p, N, 4, H, W, ig, st, ws)
        outs.append((p, st))
    (p, st), (p2, st2) = outs
    ref = L.probs_ref(x)
    reps.append(_rep(p, ref, L.probs_bound(ref, x), "probs", (N, H, W)))
    if lab is not None:
        loss, cnt, mag = L.pce_ref(x, lab, ig)
        reps.append(L.scalar(st[0], loss, mag / cnt, "pCE"))
        reps.append(L.scalar(st[1], cnt, 0.0, "labelled count"))
    else:
        reps.append(L.scalar(st[1], 0.0, 0.0, "count without labels"))
    reps += [_same(p, p2, "probs"), _same(st.nan_to_num(7.0), st2.nan_to_num(7.0), "pCE stats")]
    return {}, reps


def _r_head_bwd(a, null, g):
    N, H, W, ig, dt = a["N"], a["H"], a["W"], a["ignore_index"], a["dtype16"]
    w_ce, gs = a["w_ce"], a["gprobs_scale"]
    x = _logits(N, H, W, g)
    lab = None if "label" in null else _labels(N, H, W, g, ig)
    p, st = torch.empty_like(x), torch.zeros(2, device=DEV)
    call("wsl_softmax_pce_fwd", x, lab, p, N, 4, H, W, ig, st, _ws())
    gp = None if "gprobs" in null else _gprobs(N, H, W, g)
    go = None if "grad_out" in null else torch.tensor([0.75], device=DEV)
    cnt = int(st[1].item())
    ref, mag = L.head_bwd_ref(p, lab, ig, w_ce * (1.0 if go is None else 0.75), cnt, gp, gs)
    d = torch.full_like(x, math.nan)
    d16 = torch.full((N, H, W, 16), math.nan, device=DEV, dtype=L.TORCH_T[dt if dt != 1 else 0])
    reps = []
    args = [p, lab, None if "ce_stats" in null else st, go, w_ce, gp, gs, N, 4, H, W, ig,
            None if "dlogits" in null else d, None if "dlogits_nhwc16" in null else d16, dt]
    call("wsl_head_bwd", *args)
    if "dlogits" not in null:
        reps.append(_rep(d, ref, L.grad_bound(ref, mag), "dlogits", (N, H, W)))
    if "dlogits_nhwc16" not in null:
        reps += L.check_nhwc16(d16, ref, mag, dt, "dlogits nhwc16")
        args[12], args[13] = d, d16                                                 # both outputs from one launch
        call("wsl_head_bwd", *args)
        reps.append(L.exact(d16[..., :4].reshape(-1, 4), L.round16(_nchw(d), dt), (N, H, W), what="nhwc16 = rn(fp32)"))
    return {"dtype": "fp32" if "dlogits_nhwc16" in null else {0: "bf16", 2: "fp16"}[dt]}, reps


def _crf_case(N, H, W, g, radius=5, sxy=6.0, srgb=0.1, weight=1.0):
    y = _probs(_logits(N, H, W, g))
    img = _image(N, H, W, g)
    ws = _ws()
    outs = []
    for _ in range(2):
        gp, out = torch.full_like(y, math.nan), torch.zeros(2, device=DEV)
        call("wsl_gatedcrf_fwd", y, img, gp, N, 4, H, W, radius, sxy, srgb, weight, out, ws)
        outs.append((gp, out))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss, ksum, ref, mag, lmag = L.crf_ref(y, img, radius, sxy, srgb, weight)
    PEAK["mib"] = max(PEAK["mib"], (torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    (gp, out), (gp2, out2) = outs
    reps = [_rep(gp, ref, L.CRF_REL * mag, "CRF gradient", (N, H, W)), L.scalar(out[0], loss, lmag, "CRF loss"),
            L.scalar(out[1], ksum, ksum, "sum k"), _same(out, out2, "CRF loss"), _same(gp, gp2, "CRF gradient")]
    return reps, (y, img, gp, ref, mag, ws)


def _r_gatedcrf(a, null, g):
    reps, _ = _crf_case(a["N"], a["H"], a["W"], g, a["radius"], a["sigma_xy"], a["sigma_rgb"], a["weight"])
    tiles = a["N"] * -(-a["W"] // 32) * -(-a["H"] // 32)
    return {"tiles": tiles}, reps


def _r_ms_fwd(a, null, g):
    N, H, W = a["N"], a["H"], a["W"]
    y, img = _probs(_logits(N, H, W, g)), _image(N, H, W, g)
    ws, outs = _ws(), []
    for _ in range(2):
        out, cent = torch.zeros(1, device=DEV), torch.zeros(N * 4, device=DEV)
        call("wsl_mumford_shah_fwd", img, y, N, 4, H, W, out, cent, ws)
        outs.append((out, cent))
    loss, mag, cents, _ = L.ms_ref(img, y, 1.0)
    (out, cent), (out2, cent2) = outs
    return {}, [L.scalar(out, loss, mag, "MS loss"), L.scalar(cent, cents.reshape(-1), 2 * cents.reshape(-1).abs(), "centroids"),
                _same(out, out2, "MS loss"), _same(cent, cent2, "centroids")]


def _r_ms_bwd(a, null, g):
    N, H, W, sc = a["N"], a["H"], a["W"], a["scale"]
    y, img = _probs(_logits(N, H, W, g)), _image(N, H, W, g)
    out, cent = torch.zeros(1, device=DEV), torch.zeros(N * 4, device=DEV)
    call("wsl_mumford_shah_fwd", img, y, N, 4, H, W, out, cent, _ws())
    _, _, cents, ref = L.ms_ref(img, y, sc)
    b = L.ms_bwd_bound(img, y, cent, cents, sc) + 2.0 ** -22 * ref.abs()
    gp0 = torch.randn_like(y) * 1e-3 * abs(sc) if a["accumulate"] else torch.full_like(y, math.nan)
    gp = gp0.clone()
    args = [img, y, cent, N, 4, H, W, sc, a["accumulate"], gp]
    call("wsl_mumford_shah_bwd", *args)
    base = gp0.double() if a["accumulate"] else 0.0
    reps = [_rep(gp, ref + base, b + 2.0 ** -24 * (ref + base).abs(), "MS gradient", (N, H, W))]
    if not a["accumulate"]:
        reps.append(_acc("wsl_mumford_shah_bwd", args, 8, 9, ref, b, "MS gradient"))
    return {}, reps


def _dice_case(a, null, g):
    N, H, W, mc = a["N"], a["H"], a["W"], a["mconst"]
    y = _probs(_logits(N, H, W, g))
    msum = None
    if "msum" not in null:
        tgt, mode = _labels(N, H, W, g), "pdice"
        msum = torch.empty(H, W, device=DEV)
        call("wsl_mask_count", tgt, N, H, W, 4, msum)
    elif mc == 1.0:
        tgt, mode = _labels(N, H, W, g), "dice"
    else:
        assert mc == float(N), f"pdice_fwd with M = {mc} on a batch of {N}: only M = N (no ignored pseudo label) is a step's"
        tgt, mode = _labels(N, H, W, g, ignore=255), "pdice"
    return y, tgt, mode, msum


def _r_pdice_fwd(a, null, g):
    N, H, W, mc = a["N"], a["H"], a["W"], a["mconst"]
    y, tgt, mode, msum = _dice_case(a, null, g)
    ws, outs = _ws(), []
    for _ in range(2):
        out = torch.zeros(13, device=DEV)
        call("wsl_pdice_fwd", y, tgt, msum, mc, N, 4, H, W, out, ws)
        outs.append(out)
    loss, s, _, M = L.dice_ref(y, tgt, mode, 1.0)
    reps = [L.scalar(outs[0][1:], s, s, "Dice sums I, Y, Z"), L.scalar(outs[0][0], loss, L.dice_loss_tol(s) / L.STAT_TOL, "Dice"),
            _same(outs[0], outs[1], "Dice sums")]
    if msum is not None:
        reps.append(L.exact(msum.view(-1, 1), M.float().view(-1, 1), what="mask_count"))
    return {"mode": mode}, reps


def _r_pdice_bwd(a, null, g):
    N, H, W, mc, sc = a["N"], a["H"], a["W"], a["mconst"], a["scale"]
    y, tgt, mode, msum = _dice_case(a, null, g)
    sums = torch.zeros(13, device=DEV)
    call("wsl_pdice_fwd", y, tgt, msum, mc, N, 4, H, W, sums, _ws())
    _, s, ref, M = L.dice_ref(y, tgt, mode, sc)
    b = L.dice_bwd_bound(y, tgt, M, s, sc) + 2.0 ** -22 * ref.abs()
    gp = torch.full_like(y, math.nan)
    args = [y, tgt, msum, mc, sums, N, 4, H, W, sc, 0, gp]
    assert a["accumulate"] == 0
    call("wsl_pdice_bwd", *args)
    return {"mode": mode}, [_rep(gp, ref, b, "Dice gradient", (N, H, W)), _acc("wsl_pdice_bwd", args, 10, 11, ref, b, "Dice gradient")]


def _r_tv(a, null, g):
    planes, H, W, gsc = a["planes"], a["H"], a["W"], a["grad_scale"]
    y = _probs(_logits(planes // 4, H, W, g)).view(planes, H, W)
    ws, outs = _ws(), []
    for _ in range(2):
        gp, out = torch.zeros_like(y), torch.zeros(1, device=DEV)
        call("wsl_tv_loss", y, planes, H, W, gsc, gp, out, ws)
        outs.append((gp, out))
    loss, mag, ref = L.tv_ref(y, gsc)
    gk = float(np.float32(np.float32(gsc) / np.float32(planes * H * W)))
    (gp, out), (_, out2) = outs
    ties = int((y[:, :, 1:] == y[:, :, :-1]).sum())
    return {"ties": ties}, [_rep(gp, ref, L.tv_bound(ref, gk), "TV gradient"), L.scalar(out, loss, mag / y.numel(), "TV"),
                            _same(out, out2, "TV loss")]


def _uamt_case(a, null, g):
    T, B, H, W = a["T"], a["B"], a["H"], a["W"]
    s, t = _logits(B, H, W, g), _logits(B, H, W, g, shift=7)
    mc = mask = thr_ptr = None
    thr = a.get("threshold", 0.0)
    if T:
        base = torch.randn(B, 4, H, W, device=DEV, generator=g) * 2.0 ** (torch.rand(B, 1, H, W, device=DEV, generator=g) * 4 - 1)
        mc = (base.repeat(T, 1, 1, 1) + 0.5 * torch.randn(T * B, 4, H, W, device=DEV, generator=g)).contiguous()
        unc, band = L.uncertainty_ref(mc, T, B)
        thr = float(np.float32(unc.median().item()))
        mask = torch.full((B, H, W), 7, dtype=torch.uint8, device=DEV)
        if "threshold_ptr" not in null:
            thr_ptr = torch.tensor([thr], device=DEV)
    return s, t, mc, mask, thr_ptr, thr


def _r_uamt_fwd(a, null, g):
    T, B, H, W = a["T"], a["B"], a["H"], a["W"]
    s, t, mc, mask, thr_ptr, thr = _uamt_case(a, null, g)
    ws, outs = _ws(), []
    for _ in range(2):
        out = torch.zeros(3, device=DEV)
        call("wsl_uamt_consistency_fwd", s, t, mc, T, B, 4, H, W, thr_ptr, thr, mask, out, ws)
        outs.append(out)
    reps, row = [], {}
    if T:
        unc, band = L.uncertainty_ref(mc, T, B)
        rep, frac = L.mask_check(mask, unc, band, thr)
        reps.append(rep)
        row["band"] = frac
        if frac > 0.01:
            reps.append({"worst": math.inf, "bad": 1, "msg": f"{frac:.2%} of the pixels lie in the threshold band"})
    loss, dsum, cnt, _, _ = L.consistency_ref(s, t, mask, 1.0)
    reps += [L.scalar(outs[0][0], dsum, dsum, "masked distance sum"), L.scalar(outs[0][1], cnt, 0.0, "count"),
             L.scalar(outs[0][2], loss, loss, "consistency"), _same(outs[0], outs[1], "consistency stats")]
    return row, reps


def _r_uamt_bwd(a, null, g):
    B, H, W = a["B"], a["H"], a["W"]
    T = 0 if "mask" in null else 8
    s, t, mc, mask, thr_ptr, thr = _uamt_case(dict(a, T=T), null, g)
    st = torch.zeros(3, device=DEV)
    call("wsl_uamt_consistency_fwd", s, t, mc, T, B, 4, H, W, thr_ptr, thr, mask, st, _ws())
    w = float(np.float32(0.37)) if "weight_ptr" not in null else a["weight"]
    wp = torch.tensor([w], device=DEV) if "weight_ptr" not in null else None
    _, _, _, ref, b = L.consistency_ref(s, t, mask, w)
    d = torch.full_like(s, math.nan)
    call("wsl_uamt_consistency_bwd", s, t, mask, st, wp, a["weight"], B, 4, H, W, d)
    return {}, [_rep(d, ref, b + L.FP32_MIN, "consistency gradient", (B, H, W))]


def _r_noise(a, null, g):
    n, reps_, sig, cl, seed = a["n"], a["reps"], a["sigma"], a["clamp"], a["seed"]
    x = torch.rand(n, device=DEV, generator=g)
    sp = None if "seed_ptr" in null else torch.tensor([SEED_OFFSET], dtype=torch.int64, device=DEV)
    eff = (seed + (SEED_OFFSET if sp is not None else 0)) & ((1 << 64) - 1)
    out = torch.full((n * reps_,), math.nan, device=DEV)
    call("wsl_add_clamped_noise", x, n, reps_, sig, cl, seed, sp, out)
    ref, b = L.noise_ref(x, reps_, sig, cl, eff)
    return {}, [_rep(out, ref, b, "noisy input")]


def _r_entropy_fwd(a, null, g):
    N, H, W = a["N"], a["H"], a["W"]
    y = _probs(_logits(N, H, W, g))
    ws, outs = _ws(), []
    for _ in range(2):
        out = torch.zeros(1, device=DEV)
        call("wsl_entropy_fwd", y, N, 4, H, W, out, ws)
        outs.append(out)
    loss, mag, _, _ = L.entropy_ref(y, 1.0)
    return {}, [L.scalar(outs[0], loss, mag, "entropy"), _same(outs[0], outs[1], "entropy")]


def _r_entropy_bwd(a, null, g):
    N, H, W, sc = a["N"], a["H"], a["W"], a["scale"]
    y = _probs(_logits(N, H, W, g))
    _, _, ref, b = L.entropy_ref(y, sc)
    gp = torch.full_like(y, math.nan)
    args = [y, N, 4, H, W, sc, 0, gp]
    assert a["accumulate"] == 0
    call("wsl_entropy_bwd", *args)
    return {}, [_rep(gp, ref, b, "entropy gradient", (N, H, W)), _acc("wsl_entropy_bwd", args, 6, 7, ref, b, "entropy gradient")]


def _variance_case(a, g):
    N, H, W = a["N"], a["H"], a["W"]
    y, img = _probs(_logits(N, H, W, g)), _image(N, H, W, g)
    return N, H, W, y, img


def _r_variance_fwd(a, null, g):
    N, H, W, y, img = _variance_case(a, g)
    ws, outs = _ws(), []
    for _ in range(2):
        out, st = torch.zeros(3, device=DEV), torch.zeros(N * 10, device=DEV)
        call("wsl_class_variance_fwd", img, y, N, 4, H, W, out, st, ws)
        outs.append((out, st))
    r = L.variance_ref(img, y, 1.0)
    dsd, dmean, dsdn = L.variance_tols(r)
    (out, st), (out2, st2) = outs
    sn = st[: N * 8].view(N, 4, 2)
    sp = st[N * 8:].view(N, 2)
    tol = lambda t: t / L.STAT_TOL
    reps = [L.scalar(out[1], r["inter"], tol(dsdn.mean()).item(), "inter"), L.scalar(out[2], r["intra"], tol(dsd.mean()).item(), "intra"),
            L.scalar(out[0], r["loss"], tol(dsdn.mean() + dsd.mean()).item(), "inter - intra"),
            L.scalar(sn[..., 0], r["mean"], tol(dmean), "class means"), L.scalar(sn[..., 1], r["sd"], tol(dsd), "class stds"),
            L.scalar(sp[:, 0], r["mbar"], tol(dmean.mean(1)), "mean of the class means"), L.scalar(sp[:, 1], r["sdn"], tol(dsdn), "std of the class means"),
            _same(out, out2, "variance"), _same(st, st2, "variance statistics")]
    return {"zero_std": int(r["zero"].sum())}, reps


def _r_variance_bwd(a, null, g):
    N, H, W, y, img = _variance_case(a, g)
    sc = a["scale"]
    out, st = torch.zeros(3, device=DEV), torch.zeros(N * 10, device=DEV)
    call("wsl_class_variance_fwd", img, y, N, 4, H, W, out, st, _ws())
    r = L.variance_ref(img, y, sc)
    dsd, dmean, dsdn = L.variance_tols(r)
    ref = r["grad"]
    b = L.variance_bwd_bound(img, y, r, sc, dsd, dmean, dsdn) + 2.0 ** -22 * ref.abs() + L.FP32_MIN
    gp = torch.full_like(y, math.nan)
    args = [img, y, st, N, 4, H, W, sc, 0, gp]
    assert a["accumulate"] == 0
    call("wsl_class_variance_bwd", *args)
    reps = [_rep(gp, ref, b, "variance gradient", (N, H, W)), _acc("wsl_class_variance_bwd", args, 8, 9, ref, b, "variance gradient")]
    if not bool(r["zero"].any()):
        reps.append({"worst": math.inf, "bad": 1, "msg": "no zero class std was replayed"})
    return {"zero_std": int(r["zero"].sum())}, reps


def _r_rot90(a, null, g):
    planes, S, k, acc = a["planes"], a["S"], a["k"], a["accumulate"]
    src = torch.randn(planes, S, S, device=DEV, generator=g)
    d0 = torch.randn(planes, S, S, device=DEV, generator=g) if acc else torch.full_like(src, math.nan)
    dst = d0.clone()
    call("wsl_rot90", src, planes, S, k, acc, dst)
    rot = torch.rot90(src, k, [1, 2])
    if acc:
        ref = d0.double() + rot.double()
        return {}, [_rep(dst, ref, 2.0 ** -24 * ref.abs(), "rot90 + dst")]
    return {}, [L.exact(dst.reshape(-1, 1), rot.reshape(-1, 1), what="rot90")]


def _r_ema(a, null, g):
    n, alpha = a["n"], a["alpha"]
    e, p = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    ref, b = L.ema_ref(e, p, alpha)
    call("wsl_ema_update", e, p, n, alpha)
    return {}, [_rep(e, ref, b, "EMA")]


def _r_mix_argmax(a, null, g):
    N, H, W = a["N"], a["H"], a["W"]
    x1, x2 = _logits(N, H, W, g), _logits(N, H, W, g)
    p1, p2 = _probs(x1), _probs(x2)
    if "beta_ptr" in null:
        beta, bp = a["beta"], None
    else:
        beta = float(np.float32(torch.rand(1, generator=torch.Generator().manual_seed(int(g.initial_seed()) & 0xFFFF)).item()))
        bp = torch.tensor([beta, 1.0 - beta], dtype=torch.float32, device=DEV)
    out = torch.full((N, H, W), 9, dtype=torch.uint8, device=DEV)
    call("wsl_mix_argmax", p1, p2, a["beta"], a["one_minus_beta"], bp, N, 4, H, W, out)
    ref = O.mix_pseudo_label(p1, p2, beta).to(torch.uint8)                      # fp32, two products and one add, as the script
    mixed = beta * p1 + (1.0 - beta) * p2
    top = mixed.topk(2, 1).values
    ties = int((top[:, 0] == top[:, 1]).sum())
    return {"ties": ties}, [L.exact(out.view(-1, 1), ref.view(-1, 1), (N, H, W), what="mixed pseudo label")]


def _s2l_case(a, g, w_u):
    N, H, W = a["N"], a["H"], a["W"]
    x = _logits(N, H, W, g)
    scr = _labels(N, H, W, g)
    weight = torch.rand(N, H, W, 4, device=DEV, generator=g)
    weight[:, : H // 16] = THR_CONF                                              # exactly at thr_conf: no u-label
    ctrl = torch.tensor([THR_CONF, w_u], device=DEV)
    return N, H, W, x, scr, weight.contiguous(), ctrl


def _r_s2l_fwd(a, null, g):
    reps = []
    for w_u in (0.0, 0.5):
        N, H, W, x, scr, weight, ctrl = _s2l_case(a, g, w_u)
        ws, outs = _ws(), []
        for _ in range(2):
            p, ul, out = torch.empty_like(x), torch.full((N, H, W), 9, dtype=torch.uint8, device=DEV), torch.zeros(5, device=DEV)
            call("wsl_s2l_fwd", x, scr, weight, ctrl, N, 4, H, W, p, ul, out, ws)
            outs.append((p, ul, out))
        (p, ul, out), (_, ul2, out2) = outs
        r = L.s2l_ref(x, scr, weight, THR_CONF, w_u)
        pre = f"w_u {w_u}: "
        ref = L.probs_ref(x)
        reps += [_rep(p, ref, L.probs_bound(ref, x), pre + "probs", (N, H, W)),
                 L.exact(ul.view(-1, 1), r["ulab"].view(-1, 1), (N, H, W), what=pre + "u-labels"),
                 L.scalar(out[0], r["ce"], r["mag"] / r["n"], pre + "pCE"), L.scalar(out[1], r["n"], 0.0, pre + "labelled count"),
                 L.scalar(out[2], r["ce_u"], r["mag_u"] / r["n_u"], pre + "CE_u"), L.scalar(out[3], r["n_u"], 0.0, pre + "u count"),
                 L.scalar(out[4], r["loss"], r["mag"] / r["n"] + w_u * r["mag_u"] / r["n_u"], pre + "loss"),
                 _same(out, out2, pre + "S2L stats"), _same(ul, ul2, pre + "u-labels")]
    return {}, reps


def _r_s2l_bwd(a, null, g):
    S, dt = a["scale"], a["dtype16"]
    reps = []
    for w_u in (0.0, 0.5):
        N, H, W, x, scr, weight, ctrl = _s2l_case(a, g, w_u)
        p, ul, st = torch.empty_like(x), torch.empty((N, H, W), dtype=torch.uint8, device=DEV), torch.zeros(5, device=DEV)
        call("wsl_s2l_fwd", x, scr, weight, ctrl, N, 4, H, W, p, ul, st, _ws())
        ref, mag = L.s2l_bwd_ref(p, scr, ul, S, w_u, int(st[1].item()), int(st[3].item()))
        d = torch.full_like(x, math.nan)
        d16 = torch.full((N, H, W, 16), math.nan, device=DEV, dtype=L.TORCH_T[dt if dt != 1 else 0])
        args = [p, scr, ul, st, ctrl, S, N, 4, H, W, None if "dlogits" in null else d, None if "dlogits_nhwc16" in null else d16, dt]
        call("wsl_s2l_head_bwd", *args)
        pre = f"w_u {w_u}: "
        if "dlogits" not in null:
            reps.append(_rep(d, ref, L.grad_bound(ref, mag), pre + "dlogits", (N, H, W)))
        if "dlogits_nhwc16" not in null:
            reps += L.check_nhwc16(d16, ref, mag, dt, pre + "dlogits nhwc16")
            args[10], args[11] = d, d16
            call("wsl_s2l_head_bwd", *args)
            reps.append(L.exact(d16[..., :4].reshape(-1, 4), L.round16(_nchw(d), dt), (N, H, W), what=pre + "nhwc16 = rn(fp32)"))
    return {}, reps


REPLAY = {
    "wsl_softmax_pce_fwd": _r_softmax_pce, "wsl_head_bwd": _r_head_bwd, "wsl_gatedcrf_fwd": _r_gatedcrf,
    "wsl_mumford_shah_fwd": _r_ms_fwd, "wsl_mumford_shah_bwd": _r_ms_bwd, "wsl_pdice_fwd": _r_pdice_fwd,
    "wsl_pdice_bwd": _r_pdice_bwd, "wsl_tv_loss": _r_tv, "wsl_uamt_consistency_fwd": _r_uamt_fwd,
    "wsl_uamt_consistency_bwd": _r_uamt_bwd, "wsl_add_clamped_noise": _r_noise, "wsl_entropy_fwd": _r_entropy_fwd,
    "wsl_entropy_bwd": _r_entropy_bwd, "wsl_class_variance_fwd": _r_variance_fwd, "wsl_class_variance_bwd": _r_variance_bwd,
    "wsl_rot90": _r_rot90, "wsl_ema_update": _r_ema, "wsl_mix_argmax": _r_mix_argmax, "wsl_s2l_fwd": _r_s2l_fwd,
    "wsl_s2l_head_bwd": _r_s2l_bwd,
}
# checked by the extra tests below rather than replayed from a step (no training step launches it)
CHECKED_BY_EXTRA_TESTS = {"wsl_mask_count"}


def _left_to_others(key):
    name, _, null = key
    return name in LEFT_TO_OTHERS or (name == "wsl_mix_argmax" and "p2" in null)


def _shape(a):
    if "planes" in a:
        return f"{a['planes']}x{a.get('S', a.get('H'))}x{a.get('S', a.get('W'))}"
    if "n" in a:
        return f"n {a['n']}"
    N = a.get("N", a.get("B"))
    return f"{N}x4x{a['H']}x{a['W']}"


def _replay(key):
    if key not in _REPLAYS:
        name, scal, null = key
        a = dict(scal)
        g = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))
        t0 = time.perf_counter()
        row, reps = REPLAY[name](a, null, g)
        torch.cuda.synchronize()
        row = dict(row, entry=name, shape=_shape(a), null=null, worst=max([r["worst"] for r in reps] + [0.0]),
                   secs=time.perf_counter() - t0, args={k: v for k, v in a.items() if k not in ("N", "C", "H", "W", "B", "planes", "S", "n")})
        torch.cuda.empty_cache()
        _REPLAYS[key] = (row, [r["msg"] for r in reps if r["bad"]])
    return _REPLAYS[key]


def _run(config):
    rows, fails = [], []
    for key in _harvest(config):
        if _left_to_others(key):
            continue
        if key[0] not in REPLAY:
            fails.append(f"{key[0]}: no check")
            continue
        row, f = _replay(key)
        rows.append(row)
        fails += [f"{row['entry']} {row['shape']} {row['args']}: {m}" for m in f]
    return rows, fails


def _print(config, rows):
    print(f"\n[{config}] {len(rows)} distinct loss launches")
    for r in rows:
        extra = "".join(f" {k} {r[k]:.3g}" if isinstance(r[k], float) else f" {k} {r[k]}" for k in ("mode", "ties", "band", "zero_std", "tiles", "dtype") if k in r)
        print(f"  {r['entry']:<26} {r['shape']:<16} error/bound {r['worst']:.3g}{extra}  {r['args']}" + (f" NULL {list(r['null'])}" if r["null"] else ""))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_loss_launch_of_a_training_step_against_fp64(config):
    rows, fails = _run(config)
    _print(config, rows)
    assert rows, "no loss launch was recorded"
    assert not fails, "\n".join(fails[:40])


# ------------------------------------------------------------------------------------------------------------ extra checks
def test_gatedcrf_with_partial_tiles_on_the_right_and_bottom_edges():
    g = torch.Generator(device=DEV).manual_seed(232)
    reps, _ = _crf_case(3, 232, 200, g)
    bad = [r["msg"] for r in reps if r["bad"]]
    print(f"\ngated CRF 3x4x232x200: error/bound {max(r['worst'] for r in reps):.3g}")
    assert not bad, "\n".join(bad)


def test_functional_pdice_with_ragged_ignore_masks():
    """wsl_mask_count's per-location batch sums, and pDLoss forward / backward weighted by them (functional.pdice)"""
    a = {"N": 12, "H": 256, "W": 256, "mconst": 1.0, "scale": 1.0, "accumulate": 0}
    g = torch.Generator(device=DEV).manual_seed(12)
    row, reps = _r_pdice_fwd(a, (), g)
    _, reps2 = _r_pdice_bwd(a, (), g)
    bad = [r["msg"] for r in reps + reps2 if r["bad"]]
    print(f"\nfunctional pDice 12x4x256x256: error/bound {max(r['worst'] for r in reps + reps2):.3g}")
    assert not bad, "\n".join(bad)


def test_no_qualifying_pixel_gives_nan_losses_and_zero_gradients():
    N, H, W = 4, 64, 64
    g = torch.Generator(device=DEV).manual_seed(4)
    x = _logits(N, H, W, g)
    lab = torch.full((N, H, W), 4, dtype=torch.uint8, device=DEV)
    p, st = torch.empty_like(x), torch.zeros(2, device=DEV)
    call("wsl_softmax_pce_fwd", x, lab, p, N, 4, H, W, 4, st, _ws())
    assert math.isnan(st[0].item()) and st[1].item() == 0
    d = torch.full_like(x, math.nan)
    call("wsl_head_bwd", p, lab, st, None, 1.0, None, 0.0, N, 4, H, W, 4, d, None, 1)
    assert torch.equal(d, torch.zeros_like(d))
    scr = _labels(N, H, W, g)
    weight = torch.full((N, H, W, 4), THR_CONF, device=DEV)                  # nothing > thr_conf
    ctrl = torch.tensor([THR_CONF, 0.5], device=DEV)
    ul, s5 = torch.empty((N, H, W), dtype=torch.uint8, device=DEV), torch.zeros(5, device=DEV)
    call("wsl_s2l_fwd", x, scr, weight, ctrl, N, 4, H, W, p, ul, s5, _ws())
    assert s5[3].item() == 0 and math.isnan(s5[2].item()) and math.isnan(s5[4].item()) and not math.isnan(s5[0].item())
    call("wsl_s2l_head_bwd", p, scr, ul, s5, ctrl, 1.0, N, 4, H, W, d, None, 0)
    ref, mag = L.s2l_bwd_ref(p, scr, ul, 1.0, 0.5, int(s5[1].item()), 0)
    rep = _rep(d, ref, L.grad_bound(ref, mag), "S2L gradient without u-labels", (N, H, W))
    assert rep["bad"] == 0, rep["msg"]
    assert torch.equal(d.permute(0, 2, 3, 1)[scr == 4], torch.zeros(int((scr == 4).sum()), 4, device=DEV))


def test_planted_faults_on_real_kernel_outputs_fail_the_bounds():
    """each fault of tests/test_loss_check_cpu.py, applied to a copy of what the kernel wrote, is over its bound"""
    g = torch.Generator(device=DEV).manual_seed(99)
    # Gated CRF: one tap dropped / a halo row from the wrong tile (two samples of a 64-sample launch's operands)
    N, H, W = 2, 256, 256
    reps, (y, img, gp, ref, mag, _) = _crf_case(N, H, W, g)
    assert not [r for r in reps if r["bad"]]
    gscale = -2.0 / (N * H * W)
    s = L.crf_s(y, img)
    for fault in ({"drop": (5, 5)}, {"seam": (32, 32)}):
        bad = (gp.double() + gscale * (L.crf_s(y, img, **fault) - s)).float()
        assert _rep(bad, ref, L.CRF_REL * mag, "CRF")["bad"] > 0, fault
    # a lost block partial: pCE at 12 x 256 x 256 from the workspace's per-block partials {nll sum, count}
    N = 12
    x, lab = _logits(N, H, W, g), _labels(N, H, W, g)
    p, st, ws = torch.empty_like(x), torch.zeros(2, device=DEV), _ws()
    call("wsl_softmax_pce_fwd", x, lab, p, N, 4, H, W, 4, st, ws)
    loss, cnt, m = L.pce_ref(x, lab, 4)
    grid = min(-(-(N * H * W // 4) // 256), 8 * torch.cuda.get_device_properties(0).multi_processor_count)
    parts = ws[64: 64 + 2 * grid].view(grid, 2).double()
    assert L.scalar(parts[:, 0].sum() / parts[:, 1].sum(), loss, m / cnt, "pCE")["bad"] == 0
    assert L.scalar(parts[1:, 0].sum() / cnt, loss, m / cnt, "pCE")["bad"] == 1
    # TV: the last extremum instead of the first
    y = p[1:].reshape(-1, H, W)
    gpt, out = torch.zeros_like(y), torch.zeros(1, device=DEV)
    call("wsl_tv_loss", y, y.shape[0], H, W, 1e-2, gpt, out, _ws())
    _, _, ref = L.tv_ref(y, 1e-2)
    gk = 1e-2 / y.numel()
    assert _rep(gpt, ref, L.tv_bound(ref, gk), "TV")["bad"] == 0
    bad = gpt.double() - L.tv_route(y, gk) + L.tv_route(y, gk, last=True)
    assert _rep(bad, ref, L.tv_bound(ref, gk), "TV")["bad"] > 0
    # UAMT: a sample-major Monte-Carlo layout
    a = {"T": 8, "B": 6, "H": H, "W": W}
    s_, t_, mc, mask, thr_ptr, thr = _uamt_case(a, (), g)
    call("wsl_uamt_consistency_fwd", s_, t_, mc, 8, 6, 4, H, W, thr_ptr, thr, mask, torch.zeros(3, device=DEV), _ws())
    unc, band = L.uncertainty_ref(mc, 8, 6)
    assert L.mask_check(mask, unc, band, thr)[0]["bad"] == 0
    assert L.mask_check((L.uncertainty_fp32(mc, 8, 6, "sample_major") < thr).to(torch.uint8), unc, band, thr)[0]["bad"] > 0
    # bf16 stores truncated: the fp32 gradient of one head_bwd launch, truncated
    gpr = _gprobs(N, H, W, g)
    d = torch.empty_like(x)
    call("wsl_head_bwd", p, lab, st, None, 1.0, gpr, 0.1, N, 4, H, W, 4, d, None, 0)
    ref, mag = L.head_bwd_ref(p, lab, 4, 1.0, int(st[1].item()), gpr, 0.1)
    d16 = torch.zeros(N, H, W, 16, dtype=torch.bfloat16, device=DEV)
    d16[..., :4] = L.round16(d.permute(0, 2, 3, 1), 0)
    assert sum(r["bad"] for r in L.check_nhwc16(d16, ref, mag, 0, "bf16")) == 0
    d16[..., :4] = L.round16(d.permute(0, 2, 3, 1), 0, truncate=True)
    assert sum(r["bad"] for r in L.check_nhwc16(d16, ref, mag, 0, "bf16")) > 0
    # S2L: the first qualifying class wins
    _, _, _, x, scr, weight, ctrl = _s2l_case({"N": N, "H": H, "W": W}, g, 0.5)
    ul, s5 = torch.empty((N, H, W), dtype=torch.uint8, device=DEV), torch.zeros(5, device=DEV)
    call("wsl_s2l_fwd", x, scr, weight, ctrl, N, 4, H, W, torch.empty_like(x), ul, s5, _ws())
    r = L.s2l_ref(x, scr, weight, THR_CONF, 0.5)
    assert L.exact(ul.view(-1, 1), r["ulab"].view(-1, 1))["bad"] == 0
    assert L.exact(L.u_labels_first_wins(weight, scr, THR_CONF).view(-1, 1), r["ulab"].view(-1, 1))["bad"] > 0


def test_coverage_of_the_step_shapes():
    """every losses.cu entry point is checked here or named as left to another file, every harvested launch was replayed, and the
    replays reached the edges the docstring names"""
    entries = loss_entry_points()
    unchecked = entries - set(REPLAY) - LEFT_TO_OTHERS - CHECKED_BY_EXTRA_TESTS
    assert not unchecked, f"losses.cu entry points without a check: {sorted(unchecked)}"
    assert STEP_VARIANTS == VARIANTS
    rows, fails, launched = [], [], set()
    for c in CONFIGS:
        r, f = _run(c)
        rows += r
        fails += f
        launched |= {k[0] for k in _harvest(c)}
    assert not fails, "\n".join(fails[:20])
    replayed = {(r["entry"], r["shape"], tuple(sorted(r["args"].items())), r["null"]) for r in rows}
    keys = {k for c in CONFIGS for k in _harvest(c) if not _left_to_others(k)}
    assert len(keys) == len(_REPLAYS.keys() & keys), "a harvested launch was not replayed"
    missing = launched - set(REPLAY) - LEFT_TO_OTHERS
    assert not missing, f"launched by a step without a check: {sorted(missing)}"
    worst = {}
    for r in rows:
        worst[r["entry"]] = max(worst.get(r["entry"], 0.0), r["worst"])
    print(f"\n{len(keys)} distinct loss launches replayed ({len(replayed)} rows); fp64 reference peak {PEAK['mib']:.0f} MiB")
    for e in sorted(worst):
        print(f"  {e:<28} worst error / bound {worst[e]:.3g}")
    assert {r["dtype"] for r in rows if r["entry"] == "wsl_head_bwd"} >= {"bf16", "fp16", "fp32"}
    assert {r["args"]["k"] for r in rows if r["entry"] == "wsl_rot90"} == {0, 1, 2, 3}
    assert any(r["entry"] == "wsl_gatedcrf_fwd" and r["tiles"] > 2048 for r in rows), "no grid-stride CRF launch"
    assert any(r["entry"] == "wsl_uamt_consistency_fwd" and "band" in r for r in rows)
    assert sum(r.get("ties", 0) for r in rows if r["entry"] == "wsl_mix_argmax") > 0
    assert sum(r.get("ties", 0) for r in rows if r["entry"] == "wsl_tv_loss") > 0
