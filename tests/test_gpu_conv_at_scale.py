"""Every convolution launch of a training step and of the evaluation forwards (tensor-core and CUDA-core kernels), replayed at the
steps' own batch sizes and checked per element against fp64 (tests/_conv_check.py states the bounds).

The launches are not hand-written: one eager forward + backward of the model runs with a recorder in place of
wsl4mis_b200._lib.PROFILE, which keeps each distinct (entry point, scalar arguments, NULL pointer arguments) of the
convolution, weight-gradient and fp16 hi/lo staging entry points.  Each is replayed once on fresh seeded operands of the same
shapes: 16-bit-rounded inputs whose channels carry scales from 2^-4 .. 2^4 (a misplaced channel block shows up as a large error),
16-bit-rounded weights, and biases three standard deviations from zero.  At these shapes a persistent CTA walks several pixel
tiles or row items, so the mbarrier phase carried across tiles, the per-tile accumulator reset, the BatchNorm partial sums over a
CTA's tiles and the split-K chunk loops all run; the coverage test asserts that from the device's SM count.

The configurations are the recipes' batches (6, 12, 16, 24 and bench.py's 64) in training (forward + backward), the evaluation
forwards of the resident validation pass (64 slices), of the test step (16) and of the adversarial step's maps (6), the fp32 mode
(which runs every layer on the CUDA-core wsl_conv_direct / wsl_wgrad_direct) and the discriminator of the adversarial step.  A
distinct launch is replayed once however many configurations make it.  The census test runs one eager iteration of every recipe in
wsl4mis_b200.train.RECIPES, one validation pass and one test-step volume, and requires every convolution launch they make to be
among the replayed ones.

Per launch: outputs within |got - ref| <= u |ref| + slack S; fused BatchNorm rows equal the fp64 sums of the stored outputs and
wsl_bn_finalize turns them into fp64-accurate mean / invstd; weight gradients within rel-L2 1e-4 per output tile, bit-identical
on the deterministic split-K path, within the same bound on the atomics path, and accumulating (a second call adds on top).
The direct convolution's replay takes any recorded form: one or two sources of any storage type (the single-channel fp32 image
included), ksize 1 or 3, every out_mode, a forward with bias or a data gradient through the 'wd' pack; its weight gradient is
checked with dbias against the fp64 sums of dY."""
import ctypes
import gc
import math
import time
import zlib

import pytest
import torch

import _conv_check as CC
from _gpu_util import LaunchRecorder, pack_conv_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200 import _lib
    from wsl4mis_b200._lib import call
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    from wsl4mis_b200.networks.pnet import PNet2D
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT

CONV = ("wsl_conv_tc", "wsl_conv_tc_dil", "wsl_conv_tc2", "wsl_conv_tc_split")
WGRAD = ("wsl_wgrad_tc", "wsl_wgrad_tc3", "wsl_wgrad_tc_dil", "wsl_wgrad_tc_split")
DIRECT = ("wsl_conv_direct", "wsl_wgrad_direct")
HARVESTED = CONV + WGRAD + DIRECT + ("wsl_split_f32",)
T16 = {0: torch.bfloat16, 2: torch.float16}
DTYPE = {0: torch.bfloat16, 1: torch.float32, 2: torch.float16}              # dtype codes of the C ABI
DTN = {0: "bf16", 1: "fp32", 2: "fp16"}
OUT_T = {0: torch.bfloat16, 1: torch.float32, 2: torch.float32, 3: torch.float16}   # out_mode -> stored type
REF_BYTES = 2 << 30          # fp64 reference working set per image chunk
STAT_TOL = CC.STAT_TOL       # BatchNorm rows vs fp64 sums, relative to sum |y| and sum y^2
DBIAS_MARGIN = 10            # a direct weight gradient's smallest split share of dbias, in units of its bound

# (model, N, precision, mode): mode 'train' = forward + backward, 'eval' = eval-mode forward under no_grad.  N = 12 is the scripts'
# training batch, 6 / 16 / 24 the other recipes' (and each semi-supervised stream's), 64 bench.py's and the validation chunk, 16 the
# test step's chunk, 6 the adversarial step's no-grad maps of the unlabelled batch; the discriminator runs at that step's B = 6 and
# 2B = 12.
CONFIGS = {
    "unet_cct-n12-bf16": ("unet_cct", 12, "bf16", "train"),
    "unet_cct-n64-bf16": ("unet_cct", 64, "bf16", "train"),
    "unet_cct-n12-fp16": ("unet_cct", 12, "fp16", "train"),
    "unet_cct-n12-fp16x3": ("unet_cct", 12, "fp16x3", "train"),
    "pnet2d-n12-bf16": ("pnet2d", 12, "bf16", "train"),
    "pnet2d-n12-fp16": ("pnet2d", 12, "fp16", "train"),
    "unet_cct-n12-fp32": ("unet_cct", 12, "fp32", "train"),
    "unet_cct-n64-fp32": ("unet_cct", 64, "fp32", "train"),
    "unet-n64-bf16-eval": ("unet", 64, "bf16", "eval"),
    "unet-n16-bf16-eval": ("unet", 16, "bf16", "eval"),
    "unet-n6-bf16-eval": ("unet", 6, "bf16", "eval"),
    "unet_cct-n6-bf16": ("unet_cct", 6, "bf16", "train"),
    "unet_cct-n16-bf16": ("unet_cct", 16, "bf16", "train"),
    "unet_cct-n24-bf16": ("unet_cct", 24, "bf16", "train"),
    "disc-n6-bf16": ("disc", 6, "bf16", "train"),
    "disc-n12-bf16": ("disc", 12, "bf16", "train"),
}
_RESULTS, _REPLAYS, _KEYS = {}, {}, {}


def _model(kind):
    if kind == "unet_cct":
        return UNet_CCT(1, 4)
    if kind == "unet":
        return UNet(1, 4)
    if kind == "disc":
        return FCDiscriminator(4)
    return PNet2D(1, 4, 64, [1, 2, 4, 8, 16])


def _record(run):
    """the distinct convolution launches of run()"""
    rec, saved = LaunchRecorder(lambda name: name in HARVESTED), _lib.PROFILE
    _lib.PROFILE = rec
    try:
        run()
        torch.cuda.synchronize()
    finally:
        _lib.PROFILE = saved
    gc.collect()
    torch.cuda.empty_cache()
    return rec.launches


def _harvest(model, N, precision, mode):
    torch.manual_seed(0)
    m = _model(model).to(DEV).set_precision(precision)
    x = torch.rand(N, 1, 256, 256, device=DEV)

    def run():
        if mode == "eval":
            m.eval()
            with torch.no_grad():
                m(x)
            return
        m.train()
        if model == "disc":           # the adversarial step back-propagates into the segmentation maps
            mp = torch.softmax(torch.randn(N, 4, 256, 256, device=DEV), 1).requires_grad_(True)
            out = m(mp, x)
        else:
            out = m(x)
        outs = out if isinstance(out, (tuple, list)) else (out,)
        sum((o.float() * torch.randn_like(o.float())).mean() for o in outs).backward()
    launches = _record(run)
    del m
    return launches


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n_tile(CoutP):
    """N tile of the per-tap kernels (conv_tc, conv_tc_dil, conv_tc_split)"""
    nt = min(128, CoutP)
    while nt > 16 and CoutP % nt:
        nt //= 2
    return nt


def _conv_tc2_plan(C0, C1, N, H, W, CoutP, ks):
    """the host dispatch of wsl_conv_tc2: row kernel or halo kernel, its tile and N tile"""
    if ks == 3 and CoutP in (16, 32) and W % 128 == 0 and H % 16 == 0 and C0 + C1 <= 64:
        RS = 32 if H % 32 == 0 and N * (W // 128) * (H // 32) >= 4 * _sms() else 16
        return {"kernel": "conv_row", "th": RS, "tw": 128, "nt": CoutP, "order": "xy", "items": N * (W // 128) * (H // RS), "RS": RS}
    kblk = 64
    while kblk > 16 and (C0 % kblk or (C1 and C1 % kblk)):
        kblk //= 2
    mt = {64: 1, 32: 2, 16: 4}[kblk]
    while mt > 1 and H % (16 * mt):
        mt //= 2
    nt = min(128, CoutP)
    while nt > 16 and (CoutP % nt or ks * ks * (C0 + C1) * nt * 2 > 148 * 1024 or mt * nt > 128):
        nt //= 2
    return {"kernel": "conv_tc2", "th": 16 * mt, "tw": 8, "nt": nt, "order": "yx", "items": N * (W // 8) * (H // (16 * mt)), "MT": mt}


def _scales(C, g):
    return 2.0 ** (torch.rand(C, device=DEV, generator=g) * 8 - 4)


def _bias(scale, w64, g):
    """fp32 bias three standard deviations of the output from zero, per channel with a random sign"""
    sigma = ((scale.double().view(1, -1, 1, 1) * w64) ** 2).sum((1, 2, 3)).sqrt()
    sign = torch.where(torch.rand(w64.shape[0], device=DEV, generator=g) < 0.5, -1.0, 1.0).double()
    return (3 * sigma * sign).float()


def _chunk(N, per_image_bytes):
    return max(1, min(N, REF_BYTES // max(1, per_image_bytes)))


def _stage(x2d):
    """fp32 [P][C] -> fp16 hi | lo planes and {2^k, 2^-k, scratch}"""
    P, C = x2d.shape
    st = torch.empty((P, 2 * C), device=DEV, dtype=torch.float16)
    k = torch.zeros(3, device=DEV)
    call("wsl_split_f32", x2d, C, None, 0, P, st, k)
    return st, k


def _check_conv_output(x, w64, b64, dil, out, mode, u, slack, tiling, stats):
    """x: NHWC operand (any dtype, exact in fp64); out: NHWC (mode 0, 2) or NCHW (mode 1).  Returns the merged report and, when
    stats, the fp64 per-channel {sum, sum |y|, sum y^2} of the stored outputs."""
    N, H, W, Cin = x.shape
    Cs = w64.shape[0]
    cn = _chunk(N, H * W * (2 * Cin + 8 * Cs) * 8)
    reps, sums = [], torch.zeros(3, Cs, dtype=torch.float64, device=DEV)
    for n0 in range(0, N, cn):
        ref, S = CC.reference(x[n0:n0 + cn].permute(0, 3, 1, 2).double(), w64, b64, dil)
        o = out[n0:n0 + cn]
        got = (o if mode == 1 else o.permute(0, 3, 1, 2)).double()
        reps.append(CC.check_output(got, ref, S, u, slack, tiling, n0))
        if stats:
            sums += torch.stack([got.sum((0, 2, 3)), got.abs().sum((0, 2, 3)), (got * got).sum((0, 2, 3))])
        del ref, S, got
    return CC.merge(reps), sums


def _replay_conv(name, a, null, g):
    C0, C1, N, H, W = a["C0"], a["C1"], a["N"], a["H"], a["W"]
    CoutP, Cs, ks, dt, mode = a["CoutP"], a["CoutStore"], a["ksize"], a["dtype"], a["out_mode"]
    dil, Cin = a.get("dilation", 1), C0 + C1
    scale = _scales(Cin, g)
    x = (torch.randn(N, H, W, Cin, device=DEV, generator=g) * scale).to(T16[dt])
    w = torch.randn(Cs, Cin, ks, ks, device=DEV, generator=g) / math.sqrt(Cin * ks * ks)
    w64 = w.to(T16[dt]).double()
    bias = b64 = None
    if "bias" not in null:
        b = _bias(scale, w64, g)
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = b
        b64 = b.double()
    pk = pack_conv_weights(w, [Cin], dt)
    assert pk["CoutP"] == CoutP
    s0 = x[..., :C0].contiguous()
    s1 = x[..., C0:].contiguous() if C1 else None
    out = torch.full((N, Cs, H, W) if mode == 1 else (N, H, W, Cs), float("nan"), device=DEV,
                     dtype=T16[dt] if mode == 0 else torch.float32)
    stats = name == "wsl_conv_tc2" and "stat_partials" not in null and mode == 0
    row = {"dtype": {0: "bf16", 2: "fp16"}[dt]}
    if name == "wsl_conv_tc2":
        rows = ctypes.c_int(-1)
        parts = torch.full((592 * 2 * CoutP,), float("nan"), device=DEV) if stats else None
        call(name, s0, C0, s1, C1, pk["bf"], bias, out, mode, N, H, W, CoutP, Cs, ks, dt, parts, ctypes.addressof(rows))
        plan = _conv_tc2_plan(C0, C1, N, H, W, CoutP, ks)
        grid = rows.value
        assert 1 <= grid <= plan["items"], (plan, grid)
        tiling = CC.Tiling(H, W, plan["th"], plan["tw"], plan["nt"], grid, plan["order"])
        row.update(kernel=plan["kernel"], grid=grid, items=plan["items"], RS=plan.get("RS"), MT=plan.get("MT"), NT=plan["nt"])
    else:
        extra = (dil,) if name == "wsl_conv_tc_dil" else ()
        call(name, s0, C0, s1, C1, pk["bf"], bias, out, mode, N, H, W, CoutP, Cs, ks, dt, *extra)
        tiling = CC.Tiling(H, W, 8, 16, _n_tile(CoutP))
        items = N * (H // 8) * (W // 16)
        row.update(kernel=name[4:], grid=items, items=items, NT=tiling.nt)
    torch.cuda.synchronize()
    u = CC.UNIT_ROUNDOFF[T16[dt]] if mode == 0 else 0.0
    rep, sums = _check_conv_output(x, w64, b64, dil, out, mode, u, CC.SLACK_16, tiling, stats)
    fails = [] if rep["bad"] == 0 else [CC.describe(rep)]
    if stats:
        nr, P = rows.value, N * H * W
        st = parts[: nr * 2 * CoutP].view(nr, 2, CoutP).double().sum(0)[:, :Cs]
        e_sum = ((st[0] - sums[0]).abs() / sums[1]).max().item()
        e_sq = ((st[1] - sums[2]).abs() / sums[2]).max().item()
        row["stat_err"] = max(e_sum, e_sq)
        if not row["stat_err"] <= STAT_TOL:
            fails.append(f"BatchNorm rows: sum off by {e_sum:.2e} of sum|y|, sum of squares by {e_sq:.2e}")
        save, ss = torch.zeros(2 * CoutP, device=DEV), torch.zeros(2 * CoutP, device=DEV)
        call("wsl_bn_finalize", parts, nr, P, CoutP, torch.ones(CoutP, device=DEV), torch.zeros(CoutP, device=DEV), None, None, None,
             0.1, 1e-5, save, ss)
        torch.cuda.synchronize()
        mean = sums[0] / P
        var = sums[2] / P - mean * mean
        rms = (sums[2] / P).sqrt()
        e_mean = ((save[:Cs].double() - mean).abs() / rms).max().item()
        e_inv = ((save[CoutP:CoutP + Cs].double() * (var + 1e-5).sqrt() - 1).abs()).max().item()
        row["mean_sigmas"] = (mean.abs() / var.sqrt()).min().item()
        if not (e_mean <= 1e-5 and e_inv <= 1e-4):
            fails.append(f"wsl_bn_finalize: mean off by {e_mean:.2e} of rms, invstd by {e_inv:.2e} relative")
    row["worst"] = rep["worst"]
    return row, fails


def _replay_conv_split(a, null, g):
    Cin, N, H, W = a["Cin"], a["N"], a["H"], a["W"]
    CoutP, Cs, ks, dil, mode = a["CoutP"], a["CoutStore"], a["ksize"], a["dilation"], a["out_mode"]
    T = ks * ks
    scale = _scales(Cin, g)
    x = torch.randn(N, H, W, Cin, device=DEV, generator=g) * scale
    st, k = _stage(x.view(-1, Cin))
    w = torch.randn(Cs, Cin, ks, ks, device=DEV, generator=g) / math.sqrt(Cin * T)
    f3 = torch.zeros(T * CoutP * 3 * Cin, device=DEV, dtype=torch.float16)
    d3 = torch.zeros(T * Cin * 3 * CoutP, device=DEV, dtype=torch.float16)
    call("wsl_pack_split_weights", w, Cs, Cin, ks, CoutP, Cin, 0, Cin, f3, d3)
    w64 = w.double()
    bias = b64 = None
    if "bias" not in null:
        b = _bias(scale, w64, g)
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = b
        b64 = b.double()
    out = torch.full((N, Cs, H, W) if mode == 1 else (N, H, W, Cs), float("nan"), device=DEV)
    call("wsl_conv_tc_split", st, Cin, k[1:], f3, bias, out, mode, N, H, W, CoutP, Cs, ks, dil)
    torch.cuda.synchronize()
    tiling = CC.Tiling(H, W, 8, 16, _n_tile(CoutP))
    rep, _ = _check_conv_output(x, w64, b64, dil, out, mode, 0.0, CC.split_slack(Cin * T), tiling, False)
    items = N * (H // 8) * (W // 16)
    row = {"dtype": "fp16x3", "kernel": "conv_tc_split", "grid": items, "items": items, "NT": tiling.nt, "worst": rep["worst"]}
    return row, ([] if rep["bad"] == 0 else [CC.describe(rep)])


def _replay_split_f32(a, null, g):
    C0, C1, P = a["C0"], a["C1"], a["P"]
    C = C0 + C1
    x = torch.randn(P, C, device=DEV, generator=g) * _scales(C, g)
    x0 = x[:, :C0].contiguous()
    x1 = x[:, C0:].contiguous() if C1 else None
    st = torch.full((P, 2 * C), float("nan"), device=DEV, dtype=torch.float16)
    k = torch.zeros(3, device=DEV)
    call("wsl_split_f32", x0, C0, x1, C1, P, st, k)
    torch.cuda.synchronize()
    up, down = k[0].item(), k[1].item()
    amax = x.abs().max().item()
    fails = []
    if not (2 ** 13 <= amax * up < 2 ** 14 and up * down == 1.0):
        fails.append(f"scale 2^k = {up} for max|v| = {amax}")
    worst = 0.0
    for p0 in range(0, P, 1 << 20):
        xs = x[p0:p0 + (1 << 20)].double()
        s = st[p0:p0 + (1 << 20)].double()
        rec = (s[:, :C] + s[:, C:]) * down
        bound = 2.0 ** -21 * xs.abs() + 2.0 ** -24 * down        # 22 significant bits; fp16 subnormal floor of the lo plane
        err = (rec - xs).abs()
        ok = err <= bound
        worst = max(worst, (err / bound).max().item() if bool(ok.all()) else math.inf)
    if worst > 1.0:
        fails.append(f"hi + lo planes reproduce v to {worst:.3g} x the 2^-21 bound")
    return {"dtype": "fp32", "kernel": "split_f32", "grid": 0, "items": 0, "worst": worst}, fails


def _replay_conv_direct(a, null, g):
    """CUDA-core convolution, one CTA per 16 x 16 pixels x 16 output channels.  With a bias it is a forward: w [CoutStore, C0 + C1]
    through the 'wf' pack, the sources split at C0.  Without one it is a data gradient as the executors call it: the operand is dY
    with C0 = the layer's padded Cout channels, the layer's weight [C0, CoutStore] goes through its 'wd' pack (taps flipped, roles
    swapped) and CoutStore is the source slice width."""
    C0, C1, sd, om, N, H, W = a["C0"], a["C1"], a["src_f32"], a["out_mode"], a["N"], a["H"], a["W"]
    CinP, CoutP, Cs, ks = a["CinP"], a["CoutP"], a["CoutStore"], a["ksize"]
    Cin, dgrad = C0 + C1, "bias" in null
    scale = _scales(Cin, g)
    x = (torch.randn(N, H, W, Cin, device=DEV, generator=g) * scale).to(DTYPE[sd])
    bias = b64 = None
    if dgrad:
        wl = torch.randn(C0, Cs, ks, ks, device=DEV, generator=g) / math.sqrt(C0 * ks * ks)     # the layer's weight [Cout, slice]
        pk = pack_conv_weights(wl, [Cs])
        assert C1 == 0 and pk["CoutP"] == CinP and len(pk["wd"][0]) == ks * ks * CinP * CoutP
        wpk, w64 = pk["wd"][0], wl.double().flip(2, 3).transpose(0, 1)
    else:
        w = torch.randn(Cs, Cin, ks, ks, device=DEV, generator=g) / math.sqrt(Cin * ks * ks)
        pk = pack_conv_weights(w, [C0, C1] if C1 else [C0])
        assert pk["CinP"] == CinP and pk["CoutP"] == CoutP
        wpk, w64 = pk["wf"], w.double()
        b = _bias(scale, w64, g)
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = b
        b64 = b.double()
    s0 = x[..., :C0].contiguous()
    s1 = x[..., C0:].contiguous() if C1 else None
    out = torch.full((N, Cs, H, W) if om == 1 else (N, H, W, Cs), float("nan"), device=DEV, dtype=OUT_T[om])
    call("wsl_conv_direct", s0, C0, s1, C1, sd, wpk, bias, out, om, N, H, W, CinP, CoutP, Cs, ks)
    torch.cuda.synchronize()
    tiling = CC.Tiling(H, W, 16, 16, 16) if H % 16 == 0 and W % 16 == 0 else None
    K = ks * ks * Cin
    rep, _ = _check_conv_output(x, w64, b64, 1, out, om, CC.direct_u(OUT_T[om]), CC.direct_slack(K), tiling, False)
    items = N * -(-H // 16) * -(-W // 16)
    row = {"dtype": DTN[sd], "kernel": "conv_direct", "grid": items, "items": items, "NT": 16, "worst": rep["worst"],
           "out_mode": om, "sources": 2 if C1 else 1, "form": "dgrad" if dgrad else "fwd", "K": K}
    return row, ([] if rep["bad"] == 0 else [CC.describe(rep)])


def _direct_splits(CoutP, Cin, ntiles):
    """the host dispatch of wsl_wgrad_direct: split count of the pixel tiles"""
    ob = (CoutP // 16) * -(-Cin // 16)
    return max(1, min(-(-_sms() * 6 // ob), ntiles))


def _replay_wgrad_direct(a, null, g):
    """CUDA-core weight gradient: CTA (16 co, 16 ci, split) sums its split's 8 x 16 pixel tiles; dw and dbias accumulate atomically"""
    C0, C1, sd, dd = a["C0"], a["C1"], a["src_f32"], a["dy_f32"]
    CoutP, N, H, W, Cr, ks = a["CoutP"], a["N"], a["H"], a["W"], a["CoutReal"], a["ksize"]
    Cin, P = C0 + C1, a["N"] * a["H"] * a["W"]
    x = (torch.randn(N, H, W, Cin, device=DEV, generator=g) * _scales(Cin, g)).to(DTYPE[sd])
    # dY per channel: scale 2^-4 .. 2^4 and a mean two standard deviations from zero, so that the signed sum dbias moves by a
    # split's share when a split is lost (zero-mean dY would leave that share near the noise of the sum)
    mean = torch.where(torch.rand(Cr, device=DEV, generator=g) < 0.5, -2.0, 2.0)
    dy = torch.zeros(N, H, W, CoutP, device=DEV, dtype=DTYPE[dd])
    dy[..., :Cr] = ((torch.randn(N, H, W, Cr, device=DEV, generator=g) + mean) * _scales(Cr, g)).to(DTYPE[dd])
    s0 = x[..., :C0].contiguous()
    s1 = x[..., C0:].contiguous() if C1 else None
    ref = _wgrad_reference(x, dy, Cr, ks, 1)
    db_ref = dy[..., :Cr].double().sum((0, 1, 2))
    db_mag = dy[..., :Cr].double().abs().sum((0, 1, 2))
    ntiles = N * -(-W // 16) * -(-H // 8)
    row = {"dtype": DTN[dd], "kernel": "wgrad_direct", "grid": _direct_splits(CoutP, Cin, ntiles), "items": ntiles,
           "src": DTN[sd], "sources": 2 if C1 else 1, "dbias": "dbias" not in null}
    fails = []
    margin = CC.chunks_missing_margin(P)              # one 8 x 16 pixel tile left out of P pixels
    row["margin"] = margin / CC.WGRAD_TOL
    if margin < 50 * CC.WGRAD_TOL:
        fails.append(f"one 8 x 16 tile of {P} pixels moves dw by {margin:.1e}, under 50x the {CC.WGRAD_TOL} bound")
    if row["dbias"]:
        # dbias is one atomic per (split, channel) from the ci block 0 CTAs: the smallest split's share of the signed sum (the last
        # split when the tiles divide raggedly) must stand well above the STAT_TOL bound, or a lost or doubled split could pass
        S = row["grid"]
        tile = ((torch.arange(N, device=DEV).view(N, 1, 1) * -(-H // 8) + torch.arange(H, device=DEV).view(1, H, 1) // 8) * -(-W // 16)
                + torch.arange(W, device=DEV).view(1, 1, W) // 16)
        share = dy[tile % S == S - 1][:, :Cr].double().sum(0).abs()
        row["db_margin"] = (share / (STAT_TOL * db_mag)).min().item()
        if row["db_margin"] < DBIAS_MARGIN:
            fails.append(f"one split's share of dbias is {row['db_margin']:.3g}x the {STAT_TOL} bound, under {DBIAS_MARGIN}x")
    dw = torch.zeros(Cr, Cin, ks, ks, device=DEV)
    db = torch.zeros(Cr, device=DEV) if row["dbias"] else None
    worst = 0.0
    for k in (1, 2):                                  # the second call adds on top: dw and dbias double
        call("wsl_wgrad_direct", s0, C0, s1, C1, sd, dy, dd, CoutP, dw, db, N, H, W, Cr, ks)
        torch.cuda.synchronize()
        r = CC.check_wgrad(dw, k * ref, 16, 16)
        worst = max(worst, r["worst"])
        if r["bad"]:
            fails.append(f"dw (call {k}) over the bound in (co block, ci block, rel-L2) {r['bad'][:4]}")
        if db is not None:
            r = CC.check_sums(db, k * db_ref, k * db_mag)
            worst = max(worst, r["worst"])
            if r["bad"]:
                fails.append(f"dbias (call {k}) over {STAT_TOL} of sum |dY| at channels {r['bad'][:8]}")
    row["worst"] = worst
    return row, fails


def _wgrad_reference(x, dy, Cr, ks, dil):
    N, H, W, Cin = x.shape
    cn = _chunk(N, H * W * (Cin + dy.shape[3]) * 8 * 2)
    ref = 0
    for n0 in range(0, N, cn):
        ref = ref + CC.wgrad_reference(x[n0:n0 + cn].permute(0, 3, 1, 2).double(), dy[n0:n0 + cn, :, :, :Cr].permute(0, 3, 1, 2).double(),
                                       ks, dil)
    return ref


def _replay_wgrad(name, a, null, g):
    split = name == "wsl_wgrad_tc_split"
    Cin = a["Cin"] if split else a["C0"] + a["C1"]
    CoutP, N, H, W, Cr, ks = a["CoutP"], a["N"], a["H"], a["W"], a["CoutReal"], a["ksize"]
    dil, P = a.get("dilation", 1), a["N"] * a["H"] * a["W"]
    scale = _scales(Cin, g)
    x = torch.randn(N, H, W, Cin, device=DEV, generator=g) * scale
    dy = torch.zeros(N, H, W, CoutP, device=DEV)
    dy[..., :Cr] = torch.randn(N, H, W, Cr, device=DEV, generator=g)
    row = {"kernel": name[4:]}
    if split:
        sx, kx = _stage(x.view(-1, Cin))
        sg, kg = _stage(dy.view(-1, CoutP))
        ws = None

        def run(dw, _ws):
            call(name, sx, Cin, kx[1:], sg, CoutP, kg[1:], dw, N, H, W, Cr, ks, dil)
        row["dtype"] = "fp16x3"
    else:
        dt = a["dtype"]
        x, dy = x.to(T16[dt]), dy.to(T16[dt])
        C0, C1 = a["C0"], a["C1"]
        s0 = x[..., :C0].contiguous()
        s1 = x[..., C0:].contiguous() if C1 else None
        has_ws = "partial_floats" in a
        ws = torch.empty(a["partial_floats"], device=DEV) if has_ws and "partial_ws" not in null else None

        def run(dw, _ws):
            extra = (dil,) if name == "wsl_wgrad_tc_dil" else ()
            tail = (_ws, _ws.numel() if _ws is not None else 0) if has_ws else ()
            call(name, s0, C0, s1, C1, dy, CoutP, dw, N, H, W, Cr, ks, dt, *extra, *tail)
        row["dtype"] = {0: "bf16", 2: "fp16"}[dt]
    ref = _wgrad_reference(x, dy, Cr, ks, dil)
    blk = (min(64, Cr), 16)
    fails = []
    margin = CC.chunks_missing_margin(P)
    row["margin"] = margin / CC.WGRAD_TOL
    if margin < 50 * CC.WGRAD_TOL:
        fails.append(f"one 128-pixel chunk of {P} moves dw by {margin:.1e}, under 50x the {CC.WGRAD_TOL} bound")
    dw = torch.zeros(Cr, Cin, ks, ks, device=DEV)
    run(dw, ws)
    torch.cuda.synchronize()
    r = CC.check_wgrad(dw, ref, *blk)
    worst = r["worst"]
    if r["bad"]:
        fails.append(f"dw over the bound in (co block, ci block, rel-L2) {r['bad'][:4]}")
    run(dw, ws)                                     # accumulation: a second call adds on top
    torch.cuda.synchronize()
    r = CC.check_wgrad(dw, 2 * ref, *blk)
    worst = max(worst, r["worst"])
    if r["bad"]:
        fails.append(f"second call does not add on top: {r['bad'][:4]}")
    if ws is not None:
        d1, d2, d3 = (torch.zeros_like(dw) for _ in range(3))
        run(d1, ws)
        run(d2, ws)
        run(d3, None)                               # the atomics path
        torch.cuda.synchronize()
        row["bit_identical"] = torch.equal(d1, d2)
        if not row["bit_identical"]:
            fails.append("deterministic split-K: two replays differ")
        r = CC.check_wgrad(d3, ref, *blk)
        worst = max(worst, r["worst"])
        if r["bad"]:
            fails.append(f"atomics path over the bound: {r['bad'][:4]}")
    row.update(grid=0, items=P // CC.CHUNK_PX, worst=worst)
    return row, fails


def _replay(key):
    name, scal, null = key
    a = dict(scal)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))
    if name == "wsl_conv_direct":
        row, fails = _replay_conv_direct(a, null, g)
    elif name == "wsl_wgrad_direct":
        row, fails = _replay_wgrad_direct(a, null, g)
    elif name == "wsl_conv_tc_split":
        row, fails = _replay_conv_split(a, null, g)
    elif name in CONV:
        row, fails = _replay_conv(name, a, null, g)
    elif name == "wsl_split_f32":
        row, fails = _replay_split_f32(a, null, g)
    else:
        row, fails = _replay_wgrad(name, a, null, g)
    if "N" in a:
        cin = a.get("Cin", a.get("C0", 0) + a.get("C1", 0))
        cout = a.get("CoutStore", a.get("CoutReal"))
        row["shape"] = f"{a['N']}x{a['H']}x{a['W']} {cin}->{cout} k{a['ksize']}" + (f" d{a['dilation']}" if a.get("dilation", 1) > 1 else "")
    else:
        row["shape"] = f"P {a['P']} C {a['C0']}+{a['C1']}"
    row["entry"] = name
    if row.get("grid"):
        row["per_cta"] = -(-row["items"] // row["grid"])
        row["ragged"] = row["items"] % row["grid"] != 0
    torch.cuda.empty_cache()
    return row, fails


def _run(config):
    """-> (rows, failures) of the configuration's launches; a launch another configuration made is not replayed again"""
    if config not in _RESULTS:
        launches = _KEYS[config] = _harvest(*CONFIGS[config])
        rows, fails = [], []
        for key in launches:
            if key not in _REPLAYS:
                row, f = _replay(key)
                _REPLAYS[key] = (row, [f"{row['entry']} {row['shape']} ({row['kernel']}, {row['dtype']}): {m}" for m in f])
            rows.append(_REPLAYS[key][0])
            fails += _REPLAYS[key][1]
        _RESULTS[config] = (rows, fails)
    return _RESULTS[config]


def _family(r):
    k = r["kernel"]
    if k in ("conv_tc2", "conv_row") and "stat_err" not in r:
        k += " no-stats"
    return k, r["dtype"]


def _print(config, rows):
    print(f"\n[{config}] {len(rows)} distinct launches")
    for r in rows:
        print(f"  {r['entry']:<19} {r['kernel']:<14} {r['dtype']:<6} {r['shape']:<28} grid {r['grid']:>5} items {r['items']:>7} "
              f"per CTA {r.get('per_cta', '-'):>4}{' ragged' if r.get('ragged') else '       '}"
              + (f" RS {r['RS']}" if r.get("RS") else "") + (f" MT {r['MT']} NT {r['NT']}" if r.get("MT") else "")
              + f"  error/bound {r['worst']:.3g}"
              + (f"  BN rows {r['stat_err']:.1e} (mean {r['mean_sigmas']:.1f} sd)" if "stat_err" in r else "")
              + (f"  bit-identical {r['bit_identical']}" if "bit_identical" in r else "")
              + (f"  out_mode {r['out_mode']} {r['form']} K {r['K']}" if "out_mode" in r else "")
              + (f"  src {r['src']} dbias {r['dbias']}" if "dbias" in r else "")
              + (f" (split share {r['db_margin']:.3g}x bound)" if "db_margin" in r else ""))
    fam = {}
    for r in rows:
        k = _family(r)
        fam[k] = max(fam.get(k, 0.0), r["worst"])
    print(f"[{config}] worst error / bound per kernel family: " + ", ".join(f"{k} {d} {v:.3g}" for (k, d), v in sorted(fam.items())))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_convolution_launch_of_a_training_step_against_fp64(config):
    t0 = time.perf_counter()
    rows, fails = _run(config)
    _print(config, rows)
    print(f"[{config}] {time.perf_counter() - t0:.1f} s (harvest and the replays no earlier configuration made)")
    assert rows, "no convolution launch was recorded"
    assert not fails, "\n".join(fails)


def test_coverage_of_the_multi_tile_paths():
    """the claims of this file's docstring, from the launches the dispatcher made on this device"""
    rows = _run("unet_cct-n12-bf16")[0] + _run("unet_cct-n64-bf16")[0]
    sms = _sms()
    tc2 = [r for r in rows if r["kernel"] == "conv_tc2"]
    row = [r for r in rows if r["kernel"] == "conv_row"]
    print(f"\n{sms} SMs: conv_tc2 up to {max(r['per_cta'] for r in tc2)} tiles per CTA, conv_row up to {max(r['per_cta'] for r in row)} "
          f"items per CTA, RS {sorted({r['RS'] for r in row})}")
    assert any(r["per_cta"] >= 2 for r in tc2), "no conv_tc2 launch gives a CTA two tiles"
    assert any(r["per_cta"] >= 2 for r in row), "no conv_row launch gives a CTA two row items"
    assert any(r["ragged"] for r in tc2 + row), "no persistent launch has a ragged last wave"
    assert any(r["RS"] == 32 for r in row) and any(r["RS"] == 16 for r in row)
    assert any("stat_err" in r and r["per_cta"] >= 2 for r in tc2 + row), "no multi-tile launch carries BatchNorm rows"
    assert any(r.get("bit_identical") and r["kernel"] == "wgrad_tc3" for r in rows)
    assert {r["kernel"] for r in _run("pnet2d-n12-bf16")[0]} >= {"conv_tc_dil", "wgrad_tc_dil", "conv_tc2", "wgrad_tc"}
    assert {r["kernel"] for r in _run("unet_cct-n12-fp16x3")[0]} >= {"conv_tc_split", "wgrad_tc_split", "split_f32"}
    # the evaluation forwards: conv_tc2 and the row kernel without BatchNorm rows, at the validation chunk
    ev = _run("unet-n64-bf16-eval")[0]
    for k in ("conv_tc2", "conv_row"):
        assert any(r["kernel"] == k and "stat_err" not in r and r["shape"].startswith("64x") for r in ev), f"no NULL-statistics {k} at N = 64"
    # the CUDA-core kernels in every form the fp32 mode and the image layer use
    everything = [r for c in CONFIGS for r in _run(c)[0]]
    cd = [r for r in everything if r["kernel"] == "conv_direct"]
    wd = [r for r in everything if r["kernel"] == "wgrad_direct"]
    print(f"conv_direct: out_mode {sorted({r['out_mode'] for r in cd})}, forms {sorted({r['form'] for r in cd})}, K up to "
          f"{max(r['K'] for r in cd)}; wgrad_direct: up to {max(r['per_cta'] for r in wd)} tiles per split, "
          f"{sum(r['ragged'] for r in wd)} of {len(wd)} launches with a ragged split")
    assert {0, 1, 2, 3} <= {r["out_mode"] for r in cd}, sorted({r["out_mode"] for r in cd})
    assert any(r["sources"] == 2 for r in cd) and any(r["form"] == "dgrad" for r in cd)
    assert any(r["dtype"] == "fp32" and r["src"] == "fp32" for r in wd), "no wgrad_direct with dy_f32 = 1"
    assert {"bf16", "fp16", "fp32"} <= {r["dtype"] for r in wd}, sorted({r["dtype"] for r in wd})
    assert any(r["dbias"] for r in wd) and any(r["sources"] == 2 for r in wd)
    print(f"wgrad_direct dbias: smallest split share {min(r['db_margin'] for r in wd if r['dbias']):.3g}x the bound")
    assert any(r["ragged"] for r in wd), "no wgrad_direct launch splits its tiles raggedly (ntiles % splits != 0)"


# ------------------------------------------------------------------------------------------------------------ census
def _census_inputs(script, recipe, args, B, g):
    img = torch.rand(B, 1, 256, 256, generator=g).to(DEV)
    lab = torch.randint(0, 4, (B, 256, 256), generator=g, dtype=torch.uint8)
    scr = torch.where(torch.rand(B, 256, 256, generator=g) < 0.1, lab, torch.full_like(lab, 4))
    lab, scr = lab.to(DEV), scr.to(DEV)
    if recipe.kind == "s2l":
        return img, scr, torch.softmax(torch.rand(B, 256, 256, 4, generator=g) * 4, -1).to(DEV)
    if recipe.kind == "semi" and script != "train_partially_fully_supervised.py":
        return img, lab, torch.rand(B, 1, 256, 256, generator=g).to(DEV)
    return img, scr if args.sup_type == "scribble" else lab


def _census():
    """{launch key: [where it was made]} over one eager bf16 iteration of every recipe at its own batch, one resident validation pass
    and one test-step volume"""
    import numpy as np
    from wsl4mis_b200 import test_2D, train, val_2D
    from wsl4mis_b200.networks.net_factory import net_factory
    seen = {}

    def note(launches, where):
        for key in launches:
            seen.setdefault(key, []).append(where)
    for script, recipe in train.RECIPES.items():
        args = train.parser_for(script).parse_args([])
        B = train.rank_batch(script, args.batch_size, 1)
        torch.manual_seed(0)
        model = net_factory(net_type=args.model, in_chns=1, class_num=args.num_classes).set_precision("bf16")
        step = recipe.step(args, model, 1)
        step.graph_enabled = False
        inputs = _census_inputs(script, recipe, args, B, torch.Generator().manual_seed(len(script)))
        note(_record(lambda: step(*inputs)), f"{script} at batch {B}")
        del model, step, inputs
    net = UNet(1, 4).to(DEV).set_precision("bf16")
    rs = np.random.RandomState(5)
    shapes = [(30, 200, 180), (25, 256, 256), (20, 212, 240)]
    vs = val_2D.ValidationSet.from_arrays([rs.rand(*s).astype(np.float32) for s in shapes],
                                          [rs.randint(0, 4, s).astype(np.uint8) for s in shapes])
    note(_record(lambda: vs.predict(net)), f"validation pass (chunk {vs.chunk})")
    vol = rs.rand(20, 230, 210).astype(np.float32)
    note(_record(lambda: test_2D.predict_volume(vol, net)), f"test step (chunk {test_2D.CHUNK})")
    del net, vs
    return seen


def test_census_every_convolution_launch_of_the_recipes_is_replayed():
    """the harvest above is complete: every convolution launch the recipes' steps, the validation pass and the test step make is
    one of the replayed launches"""
    seen = _census()
    replayed = set()
    for c in CONFIGS:
        _run(c)
        replayed |= set(_KEYS[c])
    missing = {k: w for k, w in seen.items() if k not in replayed}
    print(f"\ncensus: {len(seen)} distinct convolution launches, {len(seen) - len(missing)} replayed")
    assert not missing, "launches no configuration replays:\n" + "\n".join(
        f"  {k[0]} {dict(k[1])} NULL {list(k[2])}  <- {', '.join(sorted(set(w)))}" for k, w in sorted(missing.items(), key=repr))


def test_conv_tc2_rejects_fp32_nhwc_output():
    """both conv_tc2 epilogues store 16-bit NHWC or fp32 NCHW; out_mode 2 (fp32 NHWC) is an error, not an NCHW write"""
    x = torch.randn(1, 16, 128, 16, device=DEV).to(torch.bfloat16)
    pk = pack_conv_weights(torch.randn(16, 16, 3, 3, device=DEV), [16])
    out = torch.zeros(1, 16, 128, 16, device=DEV)
    with pytest.raises(RuntimeError, match="out_mode"):
        call("wsl_conv_tc2", x, 16, None, 0, pk["bf"], None, out, 2, 1, 16, 128, 16, 16, 3, 0, None, None)
    torch.cuda.synchronize()
    assert not out.any()


@pytest.mark.parametrize("out_mode", [0, 3, 4])
def test_conv_direct_rejects_a_partial_16_bit_channel_group(out_mode):
    """the 16-bit epilogue stores whole 8-channel groups, so CoutStore % 8 != 0 in out_mode 0 / 3 (and any out_mode beyond 3) is an
    error that leaves the output untouched, not a silently unwritten tail"""
    x = torch.randn(1, 16, 16, 16, device=DEV).to(torch.bfloat16)
    w = torch.randn(12, 16, 3, 3, device=DEV) / 12
    pk = pack_conv_weights(w, [16])
    out = torch.zeros(1, 16, 16, 12, device=DEV, dtype=torch.float16 if out_mode == 3 else torch.bfloat16)
    with pytest.raises(RuntimeError, match="CoutStore"):
        call("wsl_conv_direct", x, 16, None, 0, 0, pk["wf"], None, out, out_mode, 1, 16, 16, 16, 16, 12, 3)
    torch.cuda.synchronize()
    assert not out.any()
    # the same 12 channels stored as fp32 NHWC are written whole
    out = torch.full((1, 16, 16, 12), float("nan"), device=DEV)
    call("wsl_conv_direct", x, 16, None, 0, 0, pk["wf"], None, out, 2, 1, 16, 16, 16, 16, 12, 3)
    torch.cuda.synchronize()
    ref, S = CC.reference(x.permute(0, 3, 1, 2).double(), w.double(), None)
    rep = CC.check_output(out.permute(0, 3, 1, 2).double(), ref, S, CC.direct_u(torch.float32), CC.direct_slack(144))
    assert rep["bad"] == 0, CC.describe(rep)
