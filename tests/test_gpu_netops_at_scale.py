"""Every non-convolution launch of a training step (BatchNorm statistics / finalize / activation / pooling / backward, upsample,
channel dropout, feature noise, deep-supervision resize, LeakyReLU, layout conversion, weight packing, the first layer's CUDA-core
convolution), replayed at the step's own shapes in every storage type and checked per element against fp64
(tests/_netop_check.py states the bounds and the counter-RNG restatement).

The launches are harvested as tests/test_gpu_conv_at_scale.py harvests the convolutions: one eager forward (+ backward) per
configuration runs with a LaunchRecorder in place of wsl4mis_b200._lib.PROFILE, which keeps each distinct (entry point, scalar
arguments, NULL pointer arguments) of every entry point that file does not check.  Each is replayed once on fresh operands seeded
from the key: BatchNorm inputs sigma_c * randn + mu_c rounded to the storage type (sigma_c in 2^-4 .. 2^4, mu_c / sigma_c in
[-8, 8]), three channels on three levels only (so 2 x 2 pool windows tie), upstream gradients with per-channel scales 2^-4 .. 2^4,
gamma in [0.5, 1.5], beta in +-0.2, and a device seed offset wherever the step passed one.  Consumers are checked at the kernel's
own fp32 save / ss, so a statistics error is reported at the statistics kernel.

Beyond the recorded calls, every BatchNorm backward is replayed with accumulate = 1 on top of the first result (dgamma, dbeta and
dw must double), wsl_bn_bwd once more with g0 = NULL (MODE 4), and the synchronised-BatchNorm kernels as R = 2 and R = 5 ranks
(ddp.shard_range split of the batch; raw sums added in fp32 in rank order as the all-reduce does) against fp64 BatchNorm over the
whole batch.

Bounds specific to this file (the others are in _netop_check):
  * conv_first and the single-channel conv_direct (PNet2D's first layer): 9 fp32 FMAs + bias, so |got - ref| <= u_T |ref| + 2^-19 S (10 roundings of at
    most S = conv(|x|, |w|) + |b|);
    its BatchNorm rows and wgrad_first / bn_bwd_first / wgrad_direct's dw as the convolution scale test checks them
    (STAT_TOL, rel-L2 1e-4).
  * upsample forward: six fp32 roundings of a convex combination (< 2^-21 M, M = the largest of the source neighbourhood) and
    lam = ratio * Y - base formed in fp32 (ratio rounded, the product rounded: off by <= 2^-23 h), which moves the output by
    <= 2^-22 h M per axis: |got - ref| <= u_T |ref| + (2^-21 + 2^-22 (h + w)) M.
  * upsample backward: <= 16 fp32 FMAs (2^-20) with weights off by <= 2^-23 (h + w) + 2^-22, relative to the unweighted 4 x 4 window
    sum |du|: |got - ref| <= u_T |ref| + 2^-20 (1 + h + w) sum_window |du|.
  * nearest_resize backward: sum rule (a source pixel sums <= 256 values: 256 * 2^-24 < 2^-14 of sum |terms| worst case; the
    step's 4 .. 64 stay below STAT_TOL).
  * uniform_fill: lo + f32(hi - lo) * u with the product and the sum rounded (or fused): <= 2^-24 (|f32(hi - lo) u| + |ref|).
  * bn_eval_prepare: rsqrtf is within 2 ulp, rv + eps and the product round once more: scale within 3 * 2^-23 relative; shift
    beta - rm * scale at the kernel's own scale within 2^-23 (|beta| + |rm scale|).
  * running statistics: momentum update of the fp64 mean / unbiased variance, within momentum x the mean / invstd bounds
    (1e-5 rms, 2e-4 var) + 2^-22 of the terms; num_batches_tracked + 1 (+ N per-sample).
  * bn_bwd_coef: fp64 arithmetic rounded once to fp32: 2^-23 of the magnitude of the terms."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _conv_check as CC
import _netop_check as K
from _gpu_util import LaunchRecorder, pack_conv_weights
from test_gpu_conv_at_scale import HARVESTED as CONV_HARVESTED

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200 import _lib, ddp
    from wsl4mis_b200._lib import LIB, call
    from wsl4mis_b200.networks.pnet import PNet2D
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT, UNet_CCT_3H, UNet_DS

# id -> (model, N, precision, mode); mode: train | sync | folded | per_sample | eval | ds
CONFIGS = {
    "unet_cct-n12-bf16": ("unet_cct", 12, "bf16", "train"),
    "unet_cct-n64-bf16": ("unet_cct", 64, "bf16", "train"),
    "unet_cct-n12-fp16": ("unet_cct", 12, "fp16", "train"),
    "unet_cct-n12-fp16x3": ("unet_cct", 12, "fp16x3", "train"),
    "unet_cct-n12-bf16-sync": ("unet_cct", 12, "bf16", "sync"),
    "unet_cct-n12-fp16x3-sync": ("unet_cct", 12, "fp16x3", "sync"),
    "unet_cct-n12-bf16-folded": ("unet_cct", 12, "bf16", "folded"),
    "unet-n64-bf16-per-sample": ("unet", 64, "bf16", "per_sample"),
    "unet-n12-bf16-eval": ("unet", 12, "bf16", "eval"),
    "unet_ds-n12-bf16": ("unet_ds", 12, "bf16", "train"),
    "unet_cct_3h-n12-bf16": ("unet_cct_3h", 12, "bf16", "train"),
    "pnet2d-n12-bf16": ("pnet2d", 12, "bf16", "train"),
    "pnet2d-n12-fp16": ("pnet2d", 12, "fp16", "train"),
}
DTN = {0: "bf16", 1: "fp32", 2: "fp16"}
SEED_OFFSET = 0x2545F4914F6CDD1D       # device seed offset passed wherever the step passed a seed_ptr
STAT_BOUND = K.STAT_TOL
_HARVEST, _REPLAYS, _TABLES = {}, {}, {}


def _keep(name):
    return name not in CONV_HARVESTED and name not in ("wsl_abi_version", "wsl_workspace_floats", "wsl_tc_available", "wsl_last_error")


def _model(kind):
    if kind == "unet_cct":
        return UNet_CCT(1, 4)
    if kind == "unet":
        return UNet(1, 4)
    if kind == "unet_ds":
        return UNet_DS(1, 4)
    if kind == "unet_cct_3h":
        return UNet_CCT_3H(1, 4)
    return PNet2D(1, 4, 64, [1, 2, 4, 8, 16])


def _harvest(config):
    if config in _HARVEST:
        return _HARVEST[config]
    kind, N, precision, mode = CONFIGS[config]
    torch.manual_seed(0)
    m = _model(kind).to(DEV).set_precision(precision)
    if mode == "sync":
        m.executor.sync_bn = (1, None)          # one rank: ddp.allreduce_flat is a no-op, the synchronised kernels still run
    if mode == "folded":
        m.executor.fold_finalize = True
    x = torch.rand(N, 1, 256, 256, device=DEV)
    rec, saved = LaunchRecorder(_keep), _lib.PROFILE
    _lib.PROFILE = rec
    try:
        if mode == "eval":
            m.eval()
            with torch.no_grad():
                m(x)
        elif mode == "per_sample":
            m.train()
            with torch.no_grad():
                m.executor.forward(x, True, False, None, None, bn_per_sample=True)
        else:
            m.train()
            out = m(x)
            outs = out if isinstance(out, (tuple, list)) else (out,)
            loss = sum((o.float() * torch.randn_like(o.float())).mean() for o in outs)
            loss.backward()
        torch.cuda.synchronize()
    finally:
        _lib.PROFILE = saved
    for key in rec.launches:
        if key[0] == "wsl_pack_conv_weights_batched":
            _TABLES[key] = m.executor._pack_table.cpu()
    del m
    torch.cuda.empty_cache()
    _HARVEST[config] = (rec.launches, N)
    return _HARVEST[config]


# ------------------------------------------------------------------------------------------------------------ launch geometry
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_for(items):
    """net_ops.cu / losses.cu grid_for: one CTA per 256 items, at most 8 per SM"""
    return max(1, min(-(-items // 256), 8 * _sms()))


def bn_grid(P, C, per_sm=3):
    """net_ops.cu bn_grid: >= 96 KB streamed per CTA, at most per_sm CTAs per SM"""
    return max(1, min(-(-(P * C * 2) // (96 * 1024)), _sms() * per_sm))


def _walk(total, stride, unrolled):
    """iterations of the busiest thread of a grid-stride loop over `total` items with `stride` threads, and whether some thread
    ends on the single-item tail of a two-item unrolled loop (unrolled) or the last wave is ragged (plain loops)"""
    lo, rem = divmod(total, stride)
    counts = {lo, lo + 1} if rem else {lo}
    tail = any(c % 2 == 1 and c >= 1 for c in counts) if unrolled else rem != 0
    return lo + (1 if rem else 0), tail


# ------------------------------------------------------------------------------------------------------------ operands
def _scales(C, g):
    return 2.0 ** (torch.rand(C, device=DEV, generator=g) * 8 - 4)


def _bn_input(P, C, dt, g):
    """[P, C] BatchNorm input: sigma_c * randn + mu_c, three channels on three levels only, rounded to the storage type"""
    sig = _scales(C, g)
    mu = sig * (torch.rand(C, device=DEV, generator=g) * 16 - 8)
    z = torch.randn(P, C, device=DEV, generator=g)
    for c in (1, C // 2 + 1, C - 3):
        z[:, c] = torch.randint(-1, 2, (P,), device=DEV, generator=g).float()
    return (z * sig + mu).to(K.TORCH_T[dt])


def _grad(shape, C, dt, g):
    return (torch.randn(*shape, device=DEV, generator=g) * _scales(C, g)).to(K.TORCH_T[dt])


def _affine(C, g):
    return 0.5 + torch.rand(C, device=DEV, generator=g), 0.4 * torch.rand(C, device=DEV, generator=g) - 0.2


def _save_ss(y2d, gamma, beta, eps=1e-5):
    """fp32 {mean, invstd} and {scale, shift} from the fp64 statistics of [P, C] (or [N, HW, C] per image)"""
    y = y2d.double()
    mean = y.mean(-2)
    var = (y * y).mean(-2) - mean * mean
    inv = (1.0 / (var + eps).sqrt()).float()
    sc = gamma * inv
    return torch.cat([mean.float(), inv], -1).contiguous(), torch.cat([sc, beta - mean.float() * sc], -1).contiguous()


def _ws():
    return torch.zeros(LIB.load().wsl_workspace_floats(), device=DEV)


def _seed(a, null):
    """effective seed of a replay and the device offset to pass"""
    sp = None
    if "seed_ptr" not in null:
        sp = torch.tensor([SEED_OFFSET], dtype=torch.int64, device=DEV)
    return (a.get("seed", 0) + (SEED_OFFSET if sp is not None else 0)) & K.M64, sp


def _keep_bits(a, null, P, C, g):
    """(mask tensor or None, bool [P, C] keep decisions on the device)"""
    p = a["drop_p"]
    if "mask" not in null:
        mask = (torch.rand(P, C, device=DEV, generator=g) >= 0.3).to(torch.uint8)
        return mask, mask.bool() if p > 0 else torch.ones(P, C, dtype=torch.bool, device=DEV)
    seed, _ = _seed(a, null)
    return None, torch.from_numpy(K.keep_mask(seed, P, C, p)).to(DEV)


def _merge(reps, fails, row, prefix=""):
    for r in reps:
        row["worst"] = max(row.get("worst", 0.0), r["worst"])
        if r["bad"]:
            fails.append(prefix + r["msg"])


# ------------------------------------------------------------------------------------------------------------ statistics
def _check_running(rm, rv, rm0, rv0, mean, var, n, m):
    m = float(np.float32(m))
    var_u = var * n / (n - 1)
    ref_m = (1 - m) * rm0.double() + m * mean
    ref_v = (1 - m) * rv0.double() + m * var_u
    rms = (var + mean * mean).sqrt()
    tm = m * 1e-5 * rms + K.ACT_REL * ((1 - m) * rm0.double().abs() + m * mean.abs())
    tv = m * 2e-4 * var_u + K.ACT_REL * ((1 - m) * rv0.double().abs() + m * var_u)
    reps = []
    for what, got, ref, tol in (("running_mean", rm, ref_m, tm), ("running_var", rv, ref_v, tv)):
        reps.append(K.report(got.view(1, -1), ref.view(1, -1), tol.view(1, -1), what=what))
    return reps


def _check_ss(ss, save, gamma, beta, C):
    sc_ref = gamma * save[..., C:]
    reps = [K.exact(ss[..., :C].contiguous(), sc_ref.contiguous(), what="scale = gamma * invstd")]
    sh_ref = beta.double() - save[..., :C].double() * ss[..., :C].double()
    tol = 2.0 ** -23 * (beta.double().abs() + (save[..., :C].double() * ss[..., :C].double()).abs())
    reps.append(K.report(ss[..., C:].reshape(1, -1), sh_ref.reshape(1, -1), tol.reshape(1, -1), what="shift"))
    return reps


def _stats_case(P, C, dt, g, momentum, eps, null):
    y = _bn_input(P, C, dt, g)
    gamma, beta = _affine(C, g)
    run = "running_mean" not in null
    rm0 = torch.randn(C, device=DEV, generator=g)
    rv0 = 0.5 + torch.rand(C, device=DEV, generator=g)
    nbt0 = torch.tensor([5], dtype=torch.int64, device=DEV)
    return y, gamma, beta, run, rm0, rv0, nbt0


def _finish_stats(row, fails, P, C, y, save, ss, gamma, beta, run, rm, rv, rm0, rv0, nbt, nbt0, momentum, eps, inc=1):
    s, a_, sq = K.stats_ref(y)
    rep, mean, var = K.check_mean_invstd(save[:C], save[C:], s, sq, P, eps)
    reps = [rep] + _check_ss(ss, save, gamma, beta, C)
    if run:
        reps += _check_running(rm, rv, rm0, rv0, mean, var, P, momentum)
        if nbt.item() != nbt0.item() + inc:
            fails.append(f"num_batches_tracked {nbt0.item()} -> {nbt.item()}, expected +{inc}")
    _merge(reps, fails, row)
    row["mean_sd"] = (mean.abs() / var.sqrt()).max().item()


def _replay_bn_stats(a, null, g, N_cfg):
    P, C, dt, mom, eps = a["P"], a["C"], a["dtype"], a["momentum"], a["eps"]
    grid = bn_grid(P, C)
    rows = 256 // (C // 8)
    it, tail = _walk(P, grid * rows, False)
    row = {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": "bn_stats", "worst": 0.0}
    fails = []
    y, gamma, beta, run, rm0, rv0, nbt0 = _stats_case(P, C, dt, g, mom, eps, null)
    if "raw_sums" in null:
        save, ss = torch.full((2 * C,), math.nan, device=DEV), torch.full((2 * C,), math.nan, device=DEV)
        rm, rv, nbt = rm0.clone(), rv0.clone(), nbt0.clone()
        call("wsl_bn_stats", y, dt, P, C, gamma, beta, rm if run else None, rv if run else None, nbt if run else None, mom, eps,
             save, ss, _ws(), None)
        torch.cuda.synchronize()
        _finish_stats(row, fails, P, C, y, save, ss, gamma, beta, run, rm, rv, rm0, rv0, nbt, nbt0, mom, eps)
        return row, fails
    # synchronised BatchNorm: R ranks, raw sums added in fp32 in rank order, finalised against the global pixel count
    HW = P // N_cfg
    for R in (2, 5):
        raws, ws = [], _ws()
        for r in range(R):
            lo, hi = ddp.shard_range(N_cfg, r, R)
            raw = torch.full((2 * C,), math.nan, device=DEV)
            call("wsl_bn_stats", y[lo * HW:hi * HW], dt, (hi - lo) * HW, C, gamma, beta, None, None, None, mom, eps, None, None, ws, raw)
            raws.append(raw)
        torch.cuda.synchronize()
        for r, raw in enumerate(raws):
            lo, hi = ddp.shard_range(N_cfg, r, R)
            s, a_, sq = K.stats_ref(y[lo * HW:hi * HW])
            _merge([K.sums(raw[:C], s, a_, what=f"R={R} rank {r} raw sum"), K.sums(raw[C:], sq, sq, what=f"R={R} rank {r} raw sum of squares")],
                   fails, row)
        tot = raws[0].clone()
        for raw in raws[1:]:
            tot = tot + raw
        save, ss = torch.full((2 * C,), math.nan, device=DEV), torch.full((2 * C,), math.nan, device=DEV)
        rm, rv, nbt = rm0.clone(), rv0.clone(), nbt0.clone()
        call("wsl_bn_finalize", tot, 1, P, C, gamma, beta, rm, rv, nbt, mom, eps, save, ss)
        torch.cuda.synchronize()
        _finish_stats(row, fails, P, C, y, save, ss, gamma, beta, True, rm, rv, rm0, rv0, nbt, nbt0, mom, eps)
    row["family"] = "bn_stats(raw_sums)"
    return row, fails


def _rows_of(y, nrows):
    """fp32 partial rows [nrows][2][C] of contiguous pixel chunks (the layout of the convolution epilogues' rows)"""
    P = y.shape[0]
    edges = [P * i // nrows for i in range(nrows + 1)]
    yd = y.double()
    return torch.stack([torch.stack([yd[a:b].sum(0), (yd[a:b] ** 2).sum(0)]) for a, b in zip(edges[:-1], edges[1:])]).float().contiguous()


def _replay_bn_finalize(a, null, g, N_cfg):
    nrows, P, C, mom, eps = a["nrows"], a["P"], a["C"], a["momentum"], a["eps"]
    row = {"dtype": "fp32", "grid": (C + 15) // 16, "iters": -(-nrows // 16), "tail": nrows % 16 != 0, "family": "bn_finalize",
           "worst": 0.0}
    fails = []
    y, gamma, beta, run, rm0, rv0, nbt0 = _stats_case(P, C, 1, g, mom, eps, null)
    parts = _rows_of(y, nrows)
    save, ss = torch.full((2 * C,), math.nan, device=DEV), torch.full((2 * C,), math.nan, device=DEV)
    rm, rv, nbt = rm0.clone(), rv0.clone(), nbt0.clone()
    call("wsl_bn_finalize", parts, nrows, P, C, gamma, beta, rm if run else None, rv if run else None, nbt if run else None, mom, eps, save, ss)
    torch.cuda.synchronize()
    _finish_stats(row, fails, P, C, y.float(), save, ss, gamma, beta, run, rm, rv, rm0, rv0, nbt, nbt0, mom, eps)
    return row, fails


def _replay_bn_stats_ps(a, null, g, N_cfg):
    N, HW, C, dt, mom, eps = a["N"], a["HW"], a["C"], a["dtype"], a["momentum"], a["eps"]
    nblk = max(1, min(32, -(-(HW * C) // 65536)))
    it, tail = _walk(HW, nblk * (256 // (C // 8)), False)
    row = {"dtype": DTN[dt], "grid": nblk * N, "iters": it, "tail": tail, "family": "bn_stats_ps", "worst": 0.0}
    fails = []
    y, gamma, beta, run, rm0, rv0, nbt0 = _stats_case(N * HW, C, dt, g, mom, eps, null)
    save, ss = torch.full((N, 2 * C), math.nan, device=DEV), torch.full((N, 2 * C), math.nan, device=DEV)
    rm, rv, nbt = rm0.clone(), rv0.clone(), nbt0.clone()
    call("wsl_bn_stats_ps", y, dt, N, HW, C, gamma, beta, rm if run else None, rv if run else None, nbt if run else None, mom, eps,
         save, ss, _ws())
    torch.cuda.synchronize()
    yd = y.double().view(N, HW, C)
    s, sq = yd.sum(1), (yd * yd).sum(1)
    reps = []
    for n in range(N):
        rep, _, _ = K.check_mean_invstd(save[n, :C], save[n, C:], s[n], sq[n], HW, eps)
        if rep["bad"]:
            rep["msg"] = f"image {n}: " + rep["msg"]
        reps.append(rep)
    reps += _check_ss(ss, save, gamma, beta, C)
    if run:
        m = float(np.float32(mom))
        ref_m, ref_v = rm0.double(), rv0.double()
        for n in range(N):
            mean = s[n] / HW
            var = sq[n] / HW - mean * mean
            ref_m = (1 - m) * ref_m + m * mean
            ref_v = (1 - m) * ref_v + m * var * HW / (HW - 1)
        rms = (sq / HW).sqrt().max(0).values
        reps.append(K.report(rm.view(1, -1), ref_m.view(1, -1), (1e-5 * rms + 2.0 ** -20 * ref_m.abs()).view(1, -1), what="running_mean"))
        reps.append(K.report(rv.view(1, -1), ref_v.view(1, -1), (2e-4 * ref_v.abs() + 2.0 ** -20 * ref_v.abs()).view(1, -1), what="running_var"))
        if nbt.item() != nbt0.item() + N:
            fails.append(f"num_batches_tracked {nbt0.item()} -> {nbt.item()}, expected +{N}")
    _merge(reps, fails, row)
    return row, fails


def _replay_bn_eval_prepare(a, null, g, N_cfg):
    C, eps = a["C"], a["eps"]
    gamma, beta = _affine(C, g)
    rm = torch.randn(C, device=DEV, generator=g) * 4
    rv = 0.01 + 10 * torch.rand(C, device=DEV, generator=g)
    ss = torch.full((2 * C,), math.nan, device=DEV)
    call("wsl_bn_eval_prepare", gamma, beta, rm, rv, eps, C, ss)
    torch.cuda.synchronize()
    sc_ref = gamma.double() / (rv.double() + float(np.float32(eps))).sqrt()
    sh_ref = beta.double() - rm.double() * ss[:C].double()
    reps = [K.report(ss[:C].view(1, -1), sc_ref.view(1, -1), (3 * 2.0 ** -23 * sc_ref.abs()).view(1, -1), what="eval scale"),
            K.report(ss[C:].view(1, -1), sh_ref.view(1, -1), (2.0 ** -23 * (beta.double().abs() + (rm.double() * ss[:C].double()).abs())).view(1, -1),
                     what="eval shift")]
    row, fails = {"dtype": "fp32", "grid": (C + 127) // 128, "iters": 1, "tail": False, "family": "bn_eval_prepare", "worst": 0.0}, []
    _merge(reps, fails, row)
    return row, fails


# ------------------------------------------------------------------------------------------------------------ activation
def _replay_bn_act(name, a, null, g, N_cfg):
    N, H, W, C, dt = a["N"], a["H"], a["W"], a["C"], a["dtype"]
    P, p, slope = N * H * W, a["drop_p"], a["slope"]
    T = K.TORCH_T[dt]
    pooled = "pooled" not in null
    cg = C // 8
    items = P * cg // (4 if pooled else 1)
    grid = grid_for((items + 1) // 2)
    rows = 256 // cg
    it, tail = _walk(P // 4 if pooled else P, grid * rows, not pooled)
    fam = {"wsl_bn_act_fwd": "bn_act_fwd", "wsl_bn_act_fwd_ps": "bn_act_fwd_ps", "wsl_bn_finalize_act_fwd": "bn_finalize_act_fwd"}[name]
    row = {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": fam + ("+pool" if pooled else ""), "worst": 0.0,
           "drop_p": p}
    fails = []
    y = _bn_input(P, C, dt, g)
    gamma, beta = _affine(C, g)
    mask, keep = _keep_bits(a, null, P, C, g)
    seed, sp = _seed(a, null)
    act = torch.full((P, C), math.nan, device=DEV, dtype=T)
    pl = torch.full((P // 4, C), math.nan, device=DEV, dtype=T) if pooled else None
    idx = torch.full((P // 4, C), 255, device=DEV, dtype=torch.uint8) if pooled else None
    if name == "wsl_bn_act_fwd_ps":
        save, ss = _save_ss(y.view(N, H * W, C), gamma, beta)
        call(name, y, dt, ss, N, H, W, C, slope, p, mask, a["seed"], sp, act, pl, idx)
        sc = ss[:, :C].repeat_interleave(H * W, 0)
        sh = ss[:, C:].repeat_interleave(H * W, 0)
    elif name == "wsl_bn_finalize_act_fwd":
        nrows, mom, eps = a["nrows"], a["momentum"], a["eps"]
        parts = _rows_of(y, nrows)
        run = "running_mean" not in null
        rm0, rv0 = torch.randn(C, device=DEV, generator=g), 0.5 + torch.rand(C, device=DEV, generator=g)
        nbt0 = torch.tensor([5], dtype=torch.int64, device=DEV)
        rm, rv, nbt = rm0.clone(), rv0.clone(), nbt0.clone()
        save, ss = torch.full((2 * C,), math.nan, device=DEV), torch.full((2 * C,), math.nan, device=DEV)
        call(name, y, dt, parts, nrows, gamma, beta, rm if run else None, rv if run else None, nbt if run else None, mom, eps, save, ss,
             N, H, W, C, slope, p, mask, a["seed"], sp, act, pl, idx)
        torch.cuda.synchronize()
        _finish_stats(row, fails, P, C, y, save, ss, gamma, beta, run, rm, rv, rm0, rv0, nbt, nbt0, mom, eps)
        sc, sh = ss[:C], ss[C:]
    else:
        save, ss = _save_ss(y, gamma, beta)
        call(name, y, dt, ss, N, H, W, C, slope, p, mask, a["seed"], sp, act, pl, idx)
        sc, sh = ss[:C], ss[C:]
    torch.cuda.synchronize()
    ref = K.act_ref(y, sc, sh, slope, keep, p)
    lay = K.Layout("pool", C, grid, H * W, W) if pooled else K.Layout("rows", C, grid)
    reps = [K.report(act, ref, K.act_bound(ref, dt), (N, H, W), lay, what="activation")]
    row["dropped"] = float((~keep).float().mean().item()) if p > 0 else 0.0
    if pooled:
        pref, iref, ties = K.pool_ref(act.view(N, H, W, C))
        reps.append(K.exact(pl, pref.view(-1, C), (N, H // 2, W // 2), what="pooled"))
        reps.append(K.exact(idx, iref.view(-1, C), (N, H // 2, W // 2), what="pool_idx"))
        row["ties"] = ties
    _merge(reps, fails, row)
    return row, fails


# ------------------------------------------------------------------------------------------------------------ backward
def _bwd_operands(a, null, g, P, N, H, W, C, dt):
    y = _bn_input(P, C, dt, g)
    gamma, beta = _affine(C, g)
    save, ss = _save_ss(y, gamma, beta)
    ops = {"y": y, "save": save, "ss": ss, "gamma": gamma}
    dA = torch.zeros(P, C, dtype=torch.float64, device=DEV)
    dA_abs = torch.zeros_like(dA)
    for nm in ("g0", "g1"):
        ops[nm] = None if nm in null else _grad((P, C), C, dt, g)
    ops["cs1"] = None if "cs1" in null else 2 * torch.rand(N, C, device=DEV, generator=g)
    ops["gpool"] = None if "gpool" in null else _grad((N, H // 2, W // 2, C), C, dt, g)
    ops["pool_idx"] = None if "pool_idx" in null else torch.randint(0, 4, (N, H // 2, W // 2, C), device=DEV, generator=g, dtype=torch.uint8)
    parts = {}
    if ops["g0"] is not None:
        parts["g0"] = ops["g0"].double()
    if ops["g1"] is not None:
        g1 = ops["g1"].double()
        if ops["cs1"] is not None:
            g1 = (g1.view(N, H * W, C) * ops["cs1"].double().view(N, 1, C)).view(P, C)
        parts["g1"] = g1
    if ops["gpool"] is not None:
        parts["gp"] = K.route_pool(ops["gpool"], ops["pool_idx"], H, W).view(P, C)
    ops["parts"] = parts
    return ops


def _dA(parts, without=()):
    dA = 0
    mag = 0
    for k, v in parts.items():
        if k not in without:
            dA = dA + v
            mag = mag + v.abs()
    if isinstance(dA, int):
        return None, None
    return dA, mag


def _bwd_ref(ops, keep, a, P, dt, without=()):
    dA, mag = _dA(ops["parts"], without)
    C = ops["y"].shape[1]
    if dA is None:
        dA = mag = torch.zeros(P, C, dtype=torch.float64, device=DEV)
    sv, ss = ops["save"], ops["ss"]
    return K.bn_bwd_ref(ops["y"], ss[:C], ss[C:], sv[:C], sv[C:], dA, mag, keep, a["drop_p"], a["slope"], P)


def _check_bwd(r, dgamma, dbeta, dy, ops, P, dt, shape, lay, scale=1.0, what=""):
    C = ops["y"].shape[1]
    reps = [K.sums(dgamma, scale * r["dgamma"], scale * r["dgamma_mag"], what=what + "dgamma"),
            K.sums(dbeta, scale * r["dbeta"], scale * r["dbeta_mag"], what=what + "dbeta")]
    if dy is not None:
        ref, bound = K.dy_ref(r, ops["ss"][:C], ops["save"][:C], ops["save"][C:], P, dt)
        reps.append(K.report(dy, ref, bound, shape, lay, what=what + "dY"))
    return reps


def _replay_bn_bwd(a, null, g, N_cfg):
    N, H, W, C, dt = a["N"], a["H"], a["W"], a["C"], a["dtype"]
    P = N * H * W
    mode = 4 if "g0" in null else (("g1" not in null) | (("gpool" not in null) << 1))
    grid = bn_grid(P, C, 3 if mode in (0, 4) else 2)
    it, tail = _walk(P, grid * (256 // (C // 8)), True)
    row = {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": "bn_bwd", "mode": mode, "worst": 0.0,
           "drop_p": a["drop_p"]}
    fails = []
    ops = _bwd_operands(a, null, g, P, N, H, W, C, dt)
    mask, keep = _keep_bits(a, null, P, C, g)
    seed, sp = _seed(a, null)
    lay = K.Layout("rows", C, grid)

    def run(g0, dgamma, dbeta, acc):
        dy = torch.full((P, C), math.nan, device=DEV, dtype=K.TORCH_T[dt])
        coef = torch.full((2 * C,), math.nan, device=DEV)
        call("wsl_bn_bwd", ops["y"], dt, ops["ss"], ops["save"], g0, ops["g1"], ops["cs1"], ops["gpool"], ops["pool_idx"], mask,
             a["seed"], sp, a["drop_p"], a["slope"], N, H, W, C, dgamma, dbeta, coef, dy, _ws(), acc)
        torch.cuda.synchronize()
        return dy

    r = _bwd_ref(ops, keep, a, P, dt)
    dgamma, dbeta = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dy = run(ops["g0"], dgamma, dbeta, a["accumulate"])
    reps = _check_bwd(r, dgamma, dbeta, dy, ops, P, dt, (N, H, W), lay)
    del dy
    run(ops["g0"], dgamma, dbeta, 1)                           # accumulate: a second backward adds on top
    reps += _check_bwd(r, dgamma, dbeta, None, ops, P, dt, None, None, 2.0, "accumulate = 1: ")
    if mode != 4:                                              # g0 = NULL selects MODE 4
        r4 = _bwd_ref(ops, keep, a, P, dt, without=("g0",))
        d4g, d4b = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        dy = run(None, d4g, d4b, 0)
        reps += _check_bwd(r4, d4g, d4b, dy, ops, P, dt, (N, H, W), lay, what="MODE 4 (g0 = NULL): ")
        row["mode4_replayed"] = True
    _merge(reps, fails, row)
    return row, fails


def _replay_bn_bwd_phase(a, null, g, N_cfg):
    """synchronised BatchNorm backward as R ranks: phase 1 per shard, raw sums added in fp32 in rank order, bn_bwd_coef with the
    global pixel count, phase 2 per shard; against fp64 BatchNorm backward over the whole batch"""
    N, H, W, C, dt = a["N"], a["H"], a["W"], a["C"], a["dtype"]
    assert N == N_cfg
    HW, P = H * W, N * H * W
    mode = 4 if "g0" in null else (("g1" not in null) | (("gpool" not in null) << 1))
    row = {"dtype": DTN[dt], "family": "bn_bwd_phase", "mode": mode, "worst": 0.0, "drop_p": a["drop_p"]}
    fails = []
    ops = _bwd_operands(a, null, g, P, N, H, W, C, dt)
    seed, sp = _seed(a, null)
    p = a["drop_p"]
    for R in (2, 5):
        shards = [ddp.shard_range(N, r, R) for r in range(R)]
        masks, keeps = [], []
        for lo, hi in shards:                                 # each rank draws its dropout over its own shard
            m_, k_ = _keep_bits(a, null, (hi - lo) * HW, C, g)
            masks.append(m_)
            keeps.append(k_)
        keep = torch.cat(keeps, 0)
        r_all = _bwd_ref(ops, keep, a, P, dt)

        def sl(t, lo, hi, per_pixel=True):
            if t is None:
                return None
            return t[lo * HW:hi * HW] if per_pixel else t[lo:hi]

        ws = _ws()
        dgs, dbs, raws, dys = [], [], [], []
        for (lo, hi), m_ in zip(shards, masks):
            Nr = hi - lo
            dg, db, raw = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.full((2 * C,), math.nan, device=DEV)
            coef = torch.full((2 * C,), math.nan, device=DEV)
            call("wsl_bn_bwd_phase", sl(ops["y"], lo, hi), dt, ops["ss"], ops["save"], sl(ops["g0"], lo, hi), sl(ops["g1"], lo, hi),
                 sl(ops["cs1"], lo, hi, False), sl(ops["gpool"], lo, hi, False), sl(ops["pool_idx"], lo, hi, False), m_, a["seed"], sp, p,
                 a["slope"], Nr, H, W, C, dg, db, coef, None, ws, 0, 1, raw)
            dgs.append(dg)
            dbs.append(db)
            raws.append(raw)
        tot = raws[0].clone()
        for raw in raws[1:]:
            tot = tot + raw
        coef = torch.full((2 * C,), math.nan, device=DEV)
        call("wsl_bn_bwd_coef", tot, P, ops["ss"], ops["save"], C, coef)
        for (lo, hi), m_ in zip(shards, masks):
            Nr = hi - lo
            dy = torch.full((Nr * HW, C), math.nan, device=DEV, dtype=K.TORCH_T[dt])
            call("wsl_bn_bwd_phase", sl(ops["y"], lo, hi), dt, ops["ss"], ops["save"], sl(ops["g0"], lo, hi), sl(ops["g1"], lo, hi),
                 sl(ops["cs1"], lo, hi, False), sl(ops["gpool"], lo, hi, False), sl(ops["pool_idx"], lo, hi, False), m_, a["seed"], sp, p,
                 a["slope"], Nr, H, W, C, None, None, coef, dy, ws, 0, 2, None)
            dys.append(dy)
        torch.cuda.synchronize()
        dg_sum = torch.stack(dgs).double().sum(0)
        db_sum = torch.stack(dbs).double().sum(0)
        reps = _check_bwd(r_all, dg_sum, db_sum, torch.cat(dys, 0), ops, P, dt, (N, H, W), None, what=f"R={R}: ")
        reps.append(K.sums(tot[:C], r_all["dbeta"], r_all["dbeta_mag"], what=f"R={R}: all-reduced sum dz"))
        reps.append(K.sums(tot[C:], r_all["dgamma"], r_all["dgamma_mag"], what=f"R={R}: all-reduced sum dz xhat"))
        # accumulate = 1: phase 1 again on top of each rank's own dgamma / dbeta
        for (lo, hi), m_, dg, db in zip(shards, masks, dgs, dbs):
            Nr = hi - lo
            call("wsl_bn_bwd_phase", sl(ops["y"], lo, hi), dt, ops["ss"], ops["save"], sl(ops["g0"], lo, hi), sl(ops["g1"], lo, hi),
                 sl(ops["cs1"], lo, hi, False), sl(ops["gpool"], lo, hi, False), sl(ops["pool_idx"], lo, hi, False), m_, a["seed"], sp, p,
                 a["slope"], Nr, H, W, C, dg, db, coef, None, ws, 1, 1, torch.empty(2 * C, device=DEV))
        torch.cuda.synchronize()
        reps += _check_bwd(r_all, torch.stack(dgs).double().sum(0), torch.stack(dbs).double().sum(0), None, ops, P, dt, None, None, 2.0,
                           f"R={R}, accumulate = 1: ")
        _merge(reps, fails, row)
        del dys
    lo, hi = ddp.shard_range(N, 0, 5)
    Pr = (hi - lo) * HW
    row["grid"] = bn_grid(Pr, C, 3 if mode in (0, 4) else 2)
    row["iters"], row["tail"] = _walk(Pr, row["grid"] * (256 // (C // 8)), True)
    return row, fails


def _replay_bn_bwd_coef(a, null, g, N_cfg):
    P, C = a["P_global"], a["C"]
    raw = torch.randn(2 * C, device=DEV, generator=g) * P * 1e-3
    gamma, beta = _affine(C, g)
    y = _bn_input(4096, C, 0, g)
    save, ss = _save_ss(y, gamma, beta)
    coef = torch.full((2 * C,), math.nan, device=DEV)
    call("wsl_bn_bwd_coef", raw, P, ss, save, C, coef)
    torch.cuda.synchronize()
    c1, c2 = raw[:C].double() / P, raw[C:].double() / P
    sc, mean, inv = ss[:C].double(), save[:C].double(), save[C:].double()
    B, D = -sc * c2 * inv, -sc * c1 + sc * c2 * mean * inv
    reps = [K.report(coef[:C].view(1, -1), B.view(1, -1), (2.0 ** -23 * B.abs()).view(1, -1), what="coef B"),
            K.report(coef[C:].view(1, -1), D.view(1, -1), (2.0 ** -23 * ((sc * c1).abs() + (sc * c2 * mean * inv).abs())).view(1, -1),
                     what="coef D")]
    row, fails = {"dtype": "fp32", "grid": (C + 127) // 128, "iters": 1, "tail": False, "family": "bn_bwd_coef", "worst": 0.0}, []
    _merge(reps, fails, row)
    return row, fails


# ------------------------------------------------------------------------------------------------------------ first layer
def _image(N, H, W, g):
    return torch.rand(N, H, W, device=DEV, generator=g)


def _replay_conv_first(a, null, g, N_cfg):
    N, H, W, dt = a["N"], a["H"], a["W"], a["dtype"]
    b = max(1, min(-(-(N * H * ((W + 1) // 2) * 2) // 256), _sms() * 4))
    it, tail = _walk(N * H * ((W + 1) // 2), b * 128, False)
    row = {"dtype": DTN[dt], "grid": b, "iters": it, "tail": tail, "family": "conv_first", "worst": 0.0}
    fails = []
    x = _image(N, H, W, g)
    w = torch.randn(16, 1, 3, 3, device=DEV, generator=g) / 3
    bias = torch.randn(16, device=DEV, generator=g)
    stats = "stat_partials" not in null
    y = torch.full((N, H, W, 16), math.nan, device=DEV, dtype=K.TORCH_T[dt])
    parts = torch.full((_sms() * 4 * 32,), math.nan, device=DEV) if stats else None
    nr = ctypes.c_int(-1)
    call("wsl_conv_first", x, w, bias, y, dt, N, H, W, 16, parts, ctypes.addressof(nr) if stats else None)
    torch.cuda.synchronize()
    ref, S = CC.reference(x[:, None].double(), w.double(), bias.double())
    rep = CC.check_output(y.permute(0, 3, 1, 2).double(), ref, S, K.U[dt], 2.0 ** -19)
    row["worst"] = rep["worst"]
    if rep["bad"]:
        fails.append(CC.describe(rep))
    if stats:
        assert nr.value == b, (nr.value, b)
        st = parts[: b * 32].view(b, 2, 16).double().sum(0)
        s, a_, sq = K.stats_ref(y.view(-1, 16))
        _merge([K.sums(st[0], s, a_, what="BatchNorm row sums"), K.sums(st[1], sq, sq, what="BatchNorm row sums of squares")], fails, row)
    return row, fails


def _replay_conv_direct(a, null, g, N_cfg):
    """the CUDA-core convolution of a single-channel fp32 image (PNet2D's first layer); one CTA per 16 x 16 pixels x 16 channels"""
    C0, C1, sf, om, N, H, W = a["C0"], a["C1"], a["src_f32"], a["out_mode"], a["N"], a["H"], a["W"]
    CinP, CoutP, Cs, ks = a["CinP"], a["CoutP"], a["CoutStore"], a["ksize"]
    odt = {0: 0, 1: 1, 2: 1, 3: 2}[om]
    row = {"dtype": DTN[odt], "grid": N * -(-H // 16) * -(-W // 16) * (CoutP // 16), "iters": 1, "tail": False, "family": "conv_direct",
           "worst": 0.0}
    if not (sf == 1 and C0 == 1 and C1 == 0):
        return row, ["replayed for the single-channel image layer only"]
    x = _image(N, H, W, g)
    w = torch.randn(Cs, 1, ks, ks, device=DEV, generator=g) / ks
    pk = pack_conv_weights(w, [1])
    assert pk["CinP"] == CinP and pk["CoutP"] == CoutP
    bias = b64 = None
    if "bias" not in null:
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = torch.randn(Cs, device=DEV, generator=g)
        b64 = bias[:Cs].double()
    shape = (N, Cs, H, W) if om == 1 else (N, H, W, Cs)
    out = torch.full(shape, math.nan, device=DEV, dtype=K.TORCH_T[odt])
    call("wsl_conv_direct", x, 1, None, 0, 1, pk["wf"], bias, out, om, N, H, W, CinP, CoutP, Cs, ks)
    torch.cuda.synchronize()
    ref, S = CC.reference(x[:, None].double(), w.double(), b64)
    got = out.double() if om == 1 else out.permute(0, 3, 1, 2).double()
    rep = CC.check_output(got, ref, S, K.U[odt], 2.0 ** -19, CC.Tiling(H, W, 16, 16, 16))
    row["worst"] = rep["worst"]
    return row, ([] if rep["bad"] == 0 else [CC.describe(rep)])


def _replay_wgrad_direct(a, null, g, N_cfg):
    """weight (+ bias) gradient of the same single-channel image convolution; dw and dbias accumulate"""
    C0, C1, sf, N, H, W = a["C0"], a["C1"], a["src_f32"], a["N"], a["H"], a["W"]
    CoutP, Cr, ks, ddt = a["CoutP"], a["CoutReal"], a["ksize"], a["dy_f32"]
    row = {"dtype": DTN[ddt], "grid": 0, "iters": 0, "tail": False, "family": "wgrad_direct", "worst": 0.0}
    if not (sf == 1 and C0 == 1 and C1 == 0):
        return row, ["replayed for the single-channel image layer only"]
    fails = []
    x = _image(N, H, W, g)
    dy = torch.zeros(N, H, W, CoutP, device=DEV, dtype=K.TORCH_T[ddt])
    dy[..., :Cr] = _grad((N, H, W, Cr), Cr, ddt, g)
    ref = CC.wgrad_reference(x[:, None].double(), dy[..., :Cr].permute(0, 3, 1, 2).double(), ks)
    dbias_ref = dy[..., :Cr].double().sum((0, 1, 2))
    dbias_mag = dy[..., :Cr].double().abs().sum((0, 1, 2))
    dw = torch.zeros(Cr, 1, ks, ks, device=DEV)
    db = None if "dbias" in null else torch.zeros(Cr, device=DEV)
    for k in (1, 2):                                          # the second call adds on top
        call("wsl_wgrad_direct", x, 1, None, 0, 1, dy, ddt, CoutP, dw, db, N, H, W, Cr, ks)
        torch.cuda.synchronize()
        r = CC.check_wgrad(dw, k * ref, 16, 1)
        row["worst"] = max(row["worst"], r["worst"])
        if r["bad"]:
            fails.append(f"dw (call {k}) over the bound in (co block, -, rel-L2) {r['bad'][:4]}")
        if db is not None:
            _merge([K.sums(db, k * dbias_ref, k * dbias_mag, what=f"dbias (call {k})")], fails, row)
    return row, fails


def _replay_wgrad_first(a, null, g, N_cfg):
    N, H, W, dt = a["N"], a["H"], a["W"], a["dtype"]
    b = max(1, min(-(-(N * H * W) // 4096), _sms()))
    it, tail = _walk(N * H * W, b * 256, False)
    row = {"dtype": DTN[dt], "grid": 2 * b, "iters": it, "tail": tail, "family": "wgrad_first", "worst": 0.0}
    fails = []
    x = _image(N, H, W, g)
    dy = _grad((N, H, W, 16), 16, dt, g)
    ref = CC.wgrad_reference(x[:, None].double(), dy.permute(0, 3, 1, 2).double(), 3)
    dw = torch.zeros(16, 1, 3, 3, device=DEV)
    for k in (1, 2):                                          # the second call adds on top
        call("wsl_wgrad_first", x, dy, dt, dw, N, H, W, 16)
        torch.cuda.synchronize()
        r = CC.check_wgrad(dw, k * ref, 8, 1)
        row["worst"] = max(row["worst"], r["worst"])
        if r["bad"]:
            fails.append(f"dw (call {k}) over the bound in (channel half, -, rel-L2) {r['bad']}")
    return row, fails


def _replay_bn_bwd_first(a, null, g, N_cfg):
    N, H, W, dt = a["N"], a["H"], a["W"], a["dtype"]
    C, P = 16, N * H * W
    grid = bn_grid(P, C, 3)
    it, tail = _walk(P, grid * 128, True)
    row = {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": "bn_bwd_first", "worst": 0.0, "drop_p": a["drop_p"]}
    fails = []
    ops = _bwd_operands(a, tuple(null) + ("g1", "cs1", "gpool", "pool_idx"), g, P, N, H, W, C, dt)
    mask, keep = _keep_bits(a, null, P, C, g)
    seed, sp = _seed(a, null)
    x = _image(N, H, W, g)
    r = _bwd_ref(ops, keep, a, P, dt)
    dyref, _ = K.dy_ref(r, ops["ss"][:C], ops["save"][:C], ops["save"][C:], P, dt)
    dwref = CC.wgrad_reference(x[:, None].double(), dyref.view(N, H, W, C).permute(0, 3, 1, 2), 3)
    del dyref
    dgamma, dbeta, dw = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(16, 1, 3, 3, device=DEV)
    ws = _ws()
    for k, acc in ((1, a["accumulate"]), (2, 1)):
        coef = torch.full((2 * C,), math.nan, device=DEV)
        call("wsl_bn_bwd_first", ops["y"], dt, ops["ss"], ops["save"], ops["g0"], mask, a["seed"], sp, a["drop_p"], a["slope"], N, H, W,
             dgamma, dbeta, coef, x, dw, ws, acc)
        torch.cuda.synchronize()
        reps = _check_bwd(r, dgamma, dbeta, None, ops, P, dt, None, None, float(k), f"call {k}: ")
        _merge(reps, fails, row)
        rw = CC.check_wgrad(dw, k * dwref, 8, 1)
        row["worst"] = max(row["worst"], rw["worst"])
        if rw["bad"]:
            fails.append(f"call {k}: dw over the bound in (channel half, -, rel-L2) {rw['bad']}")
    return row, fails


# ------------------------------------------------------------------------------------------------------------ resampling
def _replay_upsample(name, a, null, g, N_cfg):
    N, h, w, C, dt = a["N"], a["h"], a["w"], a["C"], a["dtype"]
    T = K.TORCH_T[dt]
    cg = C // 8
    grid = grid_for(N * h * w * cg)
    it, tail = _walk(N * h * w * cg, grid * 256, False)
    fwd = name == "wsl_upsample2x_fwd"
    row = {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": "upsample_fwd" if fwd else "upsample_bwd", "worst": 0.0}
    fails = []
    lay = K.Layout("vec", C, grid)
    if fwd:
        t = _grad((N, h, w, C), C, dt, g)
        u = torch.full((N, 2 * h, 2 * w, C), math.nan, device=DEV, dtype=T)
        call(name, t, dt, N, h, w, C, u)
        torch.cuda.synchronize()
        t64 = t.permute(0, 3, 1, 2).double()
        ref = F.interpolate(t64, scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
        M = F.interpolate(F.max_pool2d(t64.abs(), 3, 1, 1), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
        bound = K.U[dt] * ref.abs() + (2.0 ** -21 + 2.0 ** -22 * (h + w)) * M
        rep = K.report(u.view(-1, C), ref.reshape(-1, C), bound.reshape(-1, C), (N, 2 * h, 2 * w), what="upsample")
    else:
        du = _grad((N, 2 * h, 2 * w, C), C, dt, g)
        dt_ = torch.full((N, h, w, C), math.nan, device=DEV, dtype=T)
        call(name, du, dt, N, h, w, C, dt_)
        torch.cuda.synchronize()
        t64 = torch.zeros(N, C, h, w, dtype=torch.float64, device=DEV, requires_grad=True)
        F.interpolate(t64, scale_factor=2, mode="bilinear", align_corners=True).backward(du.permute(0, 3, 1, 2).double())
        ref = t64.grad.permute(0, 2, 3, 1)
        win = F.avg_pool2d(du.permute(0, 3, 1, 2).double().abs(), 4, 2, 1, count_include_pad=True) * 16
        bound = K.U[dt] * ref.abs() + 2.0 ** -20 * (1 + h + w) * win.permute(0, 2, 3, 1)
        rep = K.report(dt_.view(-1, C), ref.reshape(-1, C), bound.reshape(-1, C), (N, h, w), lay, what="upsample backward")
    _merge([rep], fails, row)
    return row, fails


def _nearest_idx(dst, scale, n):
    s = np.floor(np.arange(dst, dtype=np.float32) * np.float32(scale)).astype(np.int64)
    return torch.from_numpy(np.minimum(s, n - 1)).to(DEV)


def _replay_nearest(name, a, null, g, N_cfg):
    planes, h, w, H, W = a["planes"], a["h"], a["w"], a["H"], a["W"]
    fwd = name == "wsl_nearest_resize_fwd"
    total = planes * (H * W if fwd else h * w)
    grid = grid_for(total)
    it, tail = _walk(total, grid * 256, False)
    row = {"dtype": "fp32", "grid": grid, "iters": it, "tail": tail, "family": "nearest_fwd" if fwd else "nearest_bwd", "worst": 0.0}
    fails = []
    iy = _nearest_idx(H, np.float32(h) / np.float32(H), h)
    ix = _nearest_idx(W, np.float32(w) / np.float32(W), w)
    if fwd:
        src = torch.randn(planes, h, w, device=DEV, generator=g)
        dst = torch.full((planes, H, W), math.nan, device=DEV)
        call(name, src, planes, h, w, H, W, dst)
        torch.cuda.synchronize()
        ref = src[:, iy][:, :, ix]
        rep = K.exact(dst.view(-1, 1), ref.reshape(-1, 1), what="nearest resize")
    else:
        gd = torch.randn(planes, H, W, device=DEV, generator=g)
        gs = torch.full((planes, h, w), math.nan, device=DEV)
        call(name, gd, planes, h, w, H, W, gs)
        torch.cuda.synchronize()
        lin = (iy.view(H, 1) * w + ix.view(1, W)).reshape(-1)
        ref = torch.zeros(planes, h * w, dtype=torch.float64, device=DEV).index_add_(1, lin, gd.view(planes, -1).double())
        mag = torch.zeros_like(ref).index_add_(1, lin, gd.view(planes, -1).double().abs())
        rep = K.sums(gs.view(-1), ref.view(-1), mag.view(-1), what="nearest resize backward")
    _merge([rep], fails, row)
    return row, fails


# ------------------------------------------------------------------------------------------------------------ elementwise
def _elementwise_row(family, dt, items):
    grid = grid_for(items)
    it, tail = _walk(items, grid * 256, False)
    return {"dtype": DTN[dt], "grid": grid, "iters": it, "tail": tail, "family": family, "worst": 0.0}


def _f32(v):
    return torch.tensor(float(np.float32(v)), dtype=torch.float32, device=DEV)


def _replay_lrelu(name, a, null, g, N_cfg):
    dt, n, slope = a["dtype"], a["n"], a["slope"]
    T = K.TORCH_T[dt]
    fwd = name == "wsl_lrelu_fwd"
    row, fails = _elementwise_row("lrelu_fwd" if fwd else "lrelu_bwd", dt, n // 8), []
    y = (torch.randn(n, device=DEV, generator=g) * 2.0 ** (torch.rand(n, device=DEV, generator=g) * 8 - 4)).to(T)
    out = torch.full((n,), math.nan, device=DEV, dtype=T)
    yf = y.float()
    if fwd:
        call(name, y, dt, slope, n, out)
        ref = torch.where(yf > 0, yf, yf * _f32(slope)).to(T)
    else:
        gr = _grad((n,), 1, dt, g)
        call(name, y, dt, gr, slope, n, out)
        ref = torch.where(yf > 0, gr.float(), gr.float() * _f32(slope)).to(T)
    torch.cuda.synchronize()
    _merge([K.exact(out.view(-1, 8), ref.view(-1, 8), what=name[4:])], fails, row)
    return row, fails


def _replay_chan_mask_gen(a, null, g, N_cfg):
    n, p = a["n"], a["p"]
    seed, sp = _seed(a, null)
    cs = torch.full((n,), math.nan, device=DEV)
    call("wsl_chan_mask_gen", a["seed"], sp, n, p, cs)
    torch.cuda.synchronize()
    u = K.uniform(seed, n)
    ref = torch.from_numpy(np.where(u >= np.float32(p), np.float32(1.0) / (np.float32(1.0) - np.float32(p)), np.float32(0)).astype(np.float32))
    row, fails = {"dtype": "fp32", "grid": -(-n // 256), "iters": 1, "tail": False, "family": "chan_mask_gen", "worst": 0.0}, []
    _merge([K.exact(cs.view(1, -1), ref.to(DEV).view(1, -1), what="chan_mask_gen")], fails, row)
    return row, fails


def _replay_chan_scale(a, null, g, N_cfg):
    N, H, W, C, dt = a["N"], a["H"], a["W"], a["C"], a["dtype"]
    T = K.TORCH_T[dt]
    row, fails = _elementwise_row("chan_scale", dt, N * H * W * (C // 8)), []
    x = _grad((N, H, W, C), C, dt, g)
    cs = 2 * torch.rand(N, C, device=DEV, generator=g)
    d = torch.full((N, H, W, C), math.nan, device=DEV, dtype=T)
    call("wsl_chan_scale", x, dt, cs, N, H, W, C, d)
    torch.cuda.synchronize()
    ref = (x.float() * cs.view(N, 1, 1, C)).to(T)
    _merge([K.exact(d.view(-1, C), ref.view(-1, C), (N, H, W), K.Layout("vec", C, row["grid"]), what="chan_scale")], fails, row)
    return row, fails


def _replay_uniform_fill(a, null, g, N_cfg):
    n, lo, hi = a["n"], a["lo"], a["hi"]
    seed, sp = _seed(a, null)
    row, fails = _elementwise_row("uniform_fill", 1, n), []
    out = torch.full((n,), math.nan, device=DEV)
    call("wsl_uniform_fill", a["seed"], sp, n, lo, hi, out)
    torch.cuda.synchronize()
    u = torch.from_numpy(K.uniform(seed, n)).to(DEV).double()
    span = float(np.float32(hi) - np.float32(lo))
    ref = float(np.float32(lo)) + span * u
    bound = 2.0 ** -24 * ((span * u).abs() + ref.abs())
    _merge([K.report(out.view(1, -1), ref.view(1, -1), bound.view(1, -1), what="uniform_fill")], fails, row)
    return row, fails


def _replay_feat_noise(name, a, null, g, N_cfg):
    dt, N, hwc = a["dtype"], a["N"], a["hwc"]
    T = K.TORCH_T[dt]
    fwd = name == "wsl_feat_noise_fwd"
    row, fails = _elementwise_row("feat_noise_fwd" if fwd else "feat_noise_bwd", dt, N * hwc // 8), []
    f = _grad((N, hwc // 8, 8), 8, dt, g).view(N, hwc)
    z = 0.6 * torch.rand(hwc, device=DEV, generator=g) - 0.3
    base = (f.double() * z.double() + f.double()).float()              # fmaf(v, z, v): exact in fp64, rounded once to fp32
    reps = []
    for with_acc in ((False,) if fwd else (False, True)):
        out = torch.full((N, hwc), math.nan, device=DEV, dtype=T)
        if fwd:
            call(name, f, dt, z, N, hwc, out)
            ref = base.to(T)
        elif with_acc:
            acc = _grad((N, hwc // 8, 8), 8, dt, g).view(N, hwc)
            ref = (base + acc.float()).to(T)
            call(name, f, dt, z, N, hwc, acc, None)
            out = acc
        else:
            call(name, f, dt, z, N, hwc, None, out)
            ref = base.to(T)
        torch.cuda.synchronize()
        reps.append(K.exact(out.view(-1, 8), ref.view(-1, 8), what=name[4:] + (" (acc)" if with_acc else "")))
    _merge(reps, fails, row)
    return row, fails


def _replay_nchw_to_nhwc(a, null, g, N_cfg):
    N, Cr, H, W, CP, dt, S = a["N"], a["Creal"], a["H"], a["W"], a["CP"], a["dtype"], a["scale"]
    T = K.TORCH_T[dt]
    row, fails = _elementwise_row("nchw_f32_to_nhwc", dt, N * H * W), []
    src = torch.randn(N, Cr, H, W, device=DEV, generator=g) * _scales(Cr, g).view(1, Cr, 1, 1) / S
    dst = torch.full((N, H, W, CP), math.nan, device=DEV, dtype=T)
    call("wsl_nchw_f32_to_nhwc", src, N, Cr, H, W, CP, dst, dt, S)
    torch.cuda.synchronize()
    ref = torch.zeros(N, H, W, CP, device=DEV, dtype=T)
    ref[..., :Cr] = (src * _f32(S)).permute(0, 2, 3, 1).to(T)
    _merge([K.exact(dst.view(-1, CP), ref.view(-1, CP), (N, H, W), what="nchw_f32_to_nhwc")], fails, row)
    return row, fails


def _replay_channel_sum(a, null, g, N_cfg):
    dt, P, C, Cr = a["dtype"], a["P"], a["C"], a["Creal"]
    rows = 256 // (C // 8)
    b = max(1, min(-(-P // (rows * 16)), 2 * _sms()))
    it, tail = _walk(P, b * rows, False)
    row = {"dtype": DTN[dt], "grid": b, "iters": it, "tail": tail, "family": "channel_sum", "worst": 0.0}
    fails = []
    x = _grad((P, C), C, dt, g)
    outs = []
    for _ in range(2):
        out = torch.zeros(Cr, device=DEV)
        call("wsl_channel_sum", x, dt, P, C, Cr, out, None if "ws" in null else _ws())
        outs.append(out)
    torch.cuda.synchronize()
    xd = x[:, :Cr].double()
    _merge([K.sums(o, xd.sum(0), xd.abs().sum(0), what="channel_sum") for o in outs], fails, row)
    if "ws" not in null:
        row["bit_identical"] = torch.equal(outs[0], outs[1])
        if not row["bit_identical"]:
            fails.append("deterministic channel_sum: two runs differ")
    return row, fails


def _replay_pack_batched(key, a, null, g, N_cfg):
    table = _TABLES[key]
    n, dt = a["n_entries"], a["dtype16"]
    assert table.shape[0] == n
    row, fails = _elementwise_row("pack_conv_weights_batched", dt, a["total_items"]), []
    rows, refs, w = [], [], None
    first = 0
    for e in range(n):
        Cout, Cin, T, CoutP, CinP, beg, cnt = (int(v) for v in table[e, 5:12])
        if beg == 0:
            w = torch.randn(Cout, Cin, int(round(math.sqrt(T))), int(round(math.sqrt(T))), device=DEV, generator=g)
        sp = (cnt + 15) // 16 * 16
        has = [int(table[e, k]) != 0 for k in (1, 2, 3, 4)]
        bufs = [torch.full((T * CinP * CoutP,), math.nan, device=DEV) if has[0] else None,
                torch.full((T * CoutP * sp,), math.nan, device=DEV) if has[1] else None,
                torch.full((T * CoutP * CinP,), -1, device=DEV, dtype=torch.int16) if has[2] else None,
                torch.full((T * CoutP * sp,), -1, device=DEV, dtype=torch.int16) if has[3] else None]
        twins = [None if b is None else b.clone() for b in bufs]
        ks = int(round(math.sqrt(T)))
        call("wsl_pack_conv_weights", w, Cout, Cin, ks, CoutP, CinP, beg, cnt, *twins, dt)
        rows.append([w.data_ptr()] + [0 if b is None else b.data_ptr() for b in bufs] + [Cout, Cin, T, CoutP, CinP, beg, cnt, first])
        first += T * CoutP * CinP
        refs.append((bufs, twins, w))
    assert first == a["total_items"]
    tab = torch.tensor(rows, dtype=torch.int64).to(DEV)
    call("wsl_pack_conv_weights_batched", tab, n, first, dt)
    torch.cuda.synchronize()
    for e, (bufs, twins, _) in enumerate(refs):
        for nm, b, t in zip(("wf", "wd", "bf", "bd"), bufs, twins):
            if b is not None and not torch.equal(b.view(torch.int32) if b.dtype == torch.float32 else b,
                                                 t.view(torch.int32) if t.dtype == torch.float32 else t):
                fails.append(f"entry {e}: {nm} differs from wsl_pack_conv_weights")
    return row, fails


# ------------------------------------------------------------------------------------------------------------ driver
def _canonical(key):
    """the two phases of a synchronised BatchNorm backward are replayed together"""
    name, scal, null = key
    if name == "wsl_bn_bwd_phase":
        return (name, tuple((k, 1 if k == "phase" else (0 if k == "accumulate" else v)) for k, v in scal),
                tuple(n for n in null if n not in ("raw_sums", "dgamma", "dbeta", "dy")))
    return key


REPLAY = {
    "wsl_bn_stats": _replay_bn_stats,
    "wsl_bn_finalize": _replay_bn_finalize,
    "wsl_bn_stats_ps": _replay_bn_stats_ps,
    "wsl_bn_eval_prepare": _replay_bn_eval_prepare,
    "wsl_bn_act_fwd": lambda *r: _replay_bn_act("wsl_bn_act_fwd", *r),
    "wsl_bn_act_fwd_ps": lambda *r: _replay_bn_act("wsl_bn_act_fwd_ps", *r),
    "wsl_bn_finalize_act_fwd": lambda *r: _replay_bn_act("wsl_bn_finalize_act_fwd", *r),
    "wsl_bn_bwd": _replay_bn_bwd,
    "wsl_bn_bwd_phase": _replay_bn_bwd_phase,
    "wsl_bn_bwd_coef": _replay_bn_bwd_coef,
    "wsl_bn_bwd_first": _replay_bn_bwd_first,
    "wsl_conv_first": _replay_conv_first,
    "wsl_conv_direct": _replay_conv_direct,
    "wsl_wgrad_direct": _replay_wgrad_direct,
    "wsl_wgrad_first": _replay_wgrad_first,
    "wsl_upsample2x_fwd": lambda *r: _replay_upsample("wsl_upsample2x_fwd", *r),
    "wsl_upsample2x_bwd": lambda *r: _replay_upsample("wsl_upsample2x_bwd", *r),
    "wsl_nearest_resize_fwd": lambda *r: _replay_nearest("wsl_nearest_resize_fwd", *r),
    "wsl_nearest_resize_bwd": lambda *r: _replay_nearest("wsl_nearest_resize_bwd", *r),
    "wsl_lrelu_fwd": lambda *r: _replay_lrelu("wsl_lrelu_fwd", *r),
    "wsl_lrelu_bwd": lambda *r: _replay_lrelu("wsl_lrelu_bwd", *r),
    "wsl_chan_mask_gen": _replay_chan_mask_gen,
    "wsl_chan_scale": _replay_chan_scale,
    "wsl_uniform_fill": _replay_uniform_fill,
    "wsl_feat_noise_fwd": lambda *r: _replay_feat_noise("wsl_feat_noise_fwd", *r),
    "wsl_feat_noise_bwd": lambda *r: _replay_feat_noise("wsl_feat_noise_bwd", *r),
    "wsl_nchw_f32_to_nhwc": _replay_nchw_to_nhwc,
    "wsl_channel_sum": _replay_channel_sum,
}


def _shape(a):
    if "H" in a and "N" in a and "C" in a:
        return f"{a['N']}x{a['H']}x{a['W']}x{a['C']}"
    if "h" in a and "C" in a:
        return f"{a['N']}x{a['h']}x{a['w']}x{a['C']} (low res)"
    if "planes" in a:
        return f"{a['planes']}x{a['h']}x{a['w']} <-> {a['H']}x{a['W']}"
    if "H" in a:
        return f"{a['N']}x{a['H']}x{a['W']}" + (f" C {a['Creal']}->{a['CP']}" if "CP" in a else "")
    if "HW" in a:
        return f"{a['N']}x{a['HW']}x{a['C']}"
    if "P" in a:
        return f"P {a['P']} C {a.get('C', '')}"
    if "P_global" in a:
        return f"P {a['P_global']} C {a['C']}"
    return " ".join(f"{k} {a[k]}" for k in ("n", "n_entries", "C") if k in a)


def _replay(key, N_cfg):
    ck = _canonical(key)
    if ck in _REPLAYS:
        return _REPLAYS[ck]
    name, scal, null = key
    a = dict(scal)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(ck).encode()))
    if name == "wsl_pack_conv_weights_batched":
        row, fails = _replay_pack_batched(key, a, null, g, N_cfg)
    else:
        row, fails = REPLAY[name](a, null, g, N_cfg)
    row.update(entry=name, shape=_shape(a), null=null)
    torch.cuda.empty_cache()
    _REPLAYS[ck] = (row, fails)
    return row, fails


def _run(config):
    launches, N = _harvest(config)
    rows, fails = [], []
    unknown = sorted({k[0] for k in launches} - set(REPLAY) - {"wsl_pack_conv_weights_batched"} - NOT_REPLAYED)
    if unknown:
        fails.append(f"no replay for {unknown}")
    for key in launches:
        if key[0] in NOT_REPLAYED:
            continue
        row, f = _replay(key, N)
        rows.append(row)
        fails += [f"{row['entry']} {row['shape']} ({row['dtype']}): {m}" for m in f]
    return rows, fails


# entry points a training step reaches that other suites check: wsl_pack_split_weights stages the fp16x3 weights the convolution
# scale test replays through its own packing; wsl_sgd_step and the loss kernels are out of this file's scope
NOT_REPLAYED = {"wsl_pack_split_weights", "wsl_sgd_step", "wsl_pack_conv_weights"}


def _print(config, rows):
    print(f"\n[{config}] {len(rows)} distinct launches")
    for r in rows:
        extra = ""
        if "mode" in r:
            extra += f" MODE {r['mode']}"
        if r.get("drop_p"):
            extra += f" p {r['drop_p']:.2f}"
        if "ties" in r:
            extra += f" ties {r['ties']}"
        if "bit_identical" in r:
            extra += f" bit-identical {r['bit_identical']}"
        print(f"  {r['entry']:<28} {r['dtype']:<5} {r['shape']:<30} grid {r.get('grid', 0):>5} iters/thread {r.get('iters', 0):>4}"
              f"{' tail' if r.get('tail') else '     '}  error/bound {r['worst']:.3g}{extra}")
    fam = {}
    for r in rows:
        k = (r["family"], r["dtype"])
        fam[k] = max(fam.get(k, 0.0), r["worst"])
    print(f"[{config}] worst error / bound per family: " + ", ".join(f"{k} {d} {v:.3g}" for (k, d), v in sorted(fam.items())))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_netop_launch_of_a_training_step_against_fp64(config):
    rows, fails = _run(config)
    _print(config, rows)
    assert rows, "no launch was recorded"
    assert not fails, "\n".join(fails[:40])


@pytest.mark.parametrize("dt", [0, 1, 2])
def test_nhwc_to_nchw_f32_at_scale(dt):
    """wsl_nhwc_to_nchw_f32 has no caller in the package (feature export of the C ABI): bit-exact widening transpose"""
    N, H, W, C = 12, 256, 256, 16
    g = torch.Generator(device=DEV).manual_seed(dt)
    src = _grad((N, H, W, C), C, dt, g)
    dst = torch.full((N, C, H, W), math.nan, device=DEV)
    call("wsl_nhwc_to_nchw_f32", src, dt, N, C, H, W, dst)
    torch.cuda.synchronize()
    assert torch.equal(dst, src.float().permute(0, 3, 1, 2)), K.exact(dst.permute(0, 2, 3, 1).reshape(-1, C),
                                                                      src.float().view(-1, C), (N, H, W))["msg"]


def test_coverage_of_the_step_shapes():
    """the claims of this file's docstring, from the launches the step made on this device"""
    rows = [r for c in CONFIGS for r in _run(c)[0]]
    sms = _sms()
    fams = {}
    for r in rows:
        fams.setdefault(r["family"].replace("+pool", ""), []).append(r)
    print(f"\n{sms} SMs")
    for f in sorted(fams):
        rs = fams[f]
        print(f"  {f:<26} up to {max(r.get('iters', 0) for r in rs)} iterations per thread, "
              f"{sum(1 for r in rs if r.get('iters', 0) >= 2 and r.get('tail'))} of {len(rs)} launches with >= 2 and a tail")
    # two-pixel unrolled loops must end on their single-pixel tail somewhere; the plain grid-stride loops must walk >= 2 iterations
    # (bn_grid sizes uncapped BatchNorm grids to exactly 24 pixels per thread, so only the capped N = 64 launches reach the tail)
    for f in ("bn_act_fwd", "bn_act_fwd_ps", "bn_finalize_act_fwd", "bn_bwd", "bn_bwd_first"):
        assert any(r.get("iters", 0) >= 2 and r.get("tail") for r in fams.get(f, [])), f"no {f} launch walks >= 2 iterations into its tail"
    for f in ("bn_stats", "bn_stats_ps", "bn_bwd_phase", "upsample_fwd", "upsample_bwd", "chan_scale", "lrelu_fwd", "lrelu_bwd",
              "feat_noise_fwd", "feat_noise_bwd", "channel_sum", "conv_first", "wgrad_first", "nearest_fwd", "nearest_bwd",
              "nchw_f32_to_nhwc"):
        assert any(r.get("iters", 0) >= 2 for r in fams.get(f, [])), f"no {f} launch gives a thread >= 2 iterations"
    bwd = fams["bn_bwd"] + fams["bn_bwd_phase"]
    assert {r["mode"] for r in bwd} >= {0, 1, 2, 3}, sorted({r["mode"] for r in bwd})
    assert any(r.get("mode4_replayed") for r in fams["bn_bwd"])
    assert sum(r.get("ties", 0) for r in rows) > 0, "no tied pool window was replayed"
    fp16 = {r["family"].replace("+pool", "") for r in rows if r["dtype"] == "fp16"}
    assert fp16 >= {"bn_act_fwd", "bn_bwd", "bn_bwd_first", "upsample_fwd", "upsample_bwd"}, sorted(fp16)
    reached = {r["entry"] for r in rows}
    want = {"wsl_bn_stats", "wsl_bn_act_fwd", "wsl_bn_bwd", "wsl_upsample2x_fwd", "wsl_upsample2x_bwd", "wsl_chan_scale",
            "wsl_chan_mask_gen", "wsl_bn_bwd_first", "wsl_bn_bwd_phase", "wsl_bn_bwd_coef", "wsl_bn_finalize", "wsl_bn_stats_ps",
            "wsl_bn_act_fwd_ps", "wsl_conv_first", "wsl_wgrad_first", "wsl_nearest_resize_fwd", "wsl_nearest_resize_bwd",
            "wsl_lrelu_fwd", "wsl_lrelu_bwd", "wsl_uniform_fill", "wsl_feat_noise_fwd", "wsl_feat_noise_bwd",
            "wsl_pack_conv_weights_batched", "wsl_bn_eval_prepare", "wsl_bn_finalize_act_fwd", "wsl_nchw_f32_to_nhwc", "wsl_channel_sum"}
    assert reached >= want, sorted(want - reached)
    assert any(r["entry"] == "wsl_bn_stats" and "raw_sums" not in r["null"] for r in rows)
