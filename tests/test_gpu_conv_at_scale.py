"""Every tensor-core convolution launch of a training step, replayed at the step's own batch sizes and checked per element
against fp64 (tests/_conv_check.py states the bounds).

The launches are not hand-written: one eager forward + backward of the model runs with a recorder in place of
wsl4mis_b200._lib.PROFILE, which keeps each distinct (entry point, scalar arguments, NULL pointer arguments) of the
convolution, weight-gradient and fp16 hi/lo staging entry points.  Each is replayed once on fresh seeded operands of the same
shapes: 16-bit-rounded inputs whose channels carry scales from 2^-4 .. 2^4 (a misplaced channel block shows up as a large error),
16-bit-rounded weights, and biases three standard deviations from zero.  At these shapes a persistent CTA walks several pixel
tiles or row items, so the mbarrier phase carried across tiles, the per-tile accumulator reset, the BatchNorm partial sums over a
CTA's tiles and the split-K chunk loops all run; the coverage test asserts that from the device's SM count.

Per launch: outputs within |got - ref| <= u |ref| + slack S; fused BatchNorm rows equal the fp64 sums of the stored outputs and
wsl_bn_finalize turns them into fp64-accurate mean / invstd; weight gradients within rel-L2 1e-4 per output tile, bit-identical
on the deterministic split-K path, within the same bound on the atomics path, and accumulating (a second call adds on top)."""
import ctypes
import math
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
    from wsl4mis_b200.networks.pnet import PNet2D
    from wsl4mis_b200.networks.unet import UNet_CCT

CONV = ("wsl_conv_tc", "wsl_conv_tc_dil", "wsl_conv_tc2", "wsl_conv_tc_split")
WGRAD = ("wsl_wgrad_tc", "wsl_wgrad_tc2", "wsl_wgrad_tc3", "wsl_wgrad_tc_dil", "wsl_wgrad_tc_split")
HARVESTED = CONV + WGRAD + ("wsl_split_f32",)
T16 = {0: torch.bfloat16, 2: torch.float16}
REF_BYTES = 2 << 30          # fp64 reference working set per image chunk
STAT_TOL = 1e-5              # BatchNorm rows vs fp64 sums, relative to sum |y| and sum y^2

# (model, N, precision): N = 12 is the scripts' training batch, N = 64 bench.py's
CONFIGS = {
    "unet_cct-n12-bf16": ("unet_cct", 12, "bf16"),
    "unet_cct-n64-bf16": ("unet_cct", 64, "bf16"),
    "unet_cct-n12-fp16": ("unet_cct", 12, "fp16"),
    "unet_cct-n12-fp16x3": ("unet_cct", 12, "fp16x3"),
    "pnet2d-n12-bf16": ("pnet2d", 12, "bf16"),
}
_RESULTS = {}


def _harvest(model, N, precision):
    torch.manual_seed(0)
    m = UNet_CCT(1, 4) if model == "unet_cct" else PNet2D(1, 4, 64, [1, 2, 4, 8, 16])
    m = m.to(DEV).set_precision(precision)
    m.train()
    x = torch.rand(N, 1, 256, 256, device=DEV)
    rec, saved = LaunchRecorder(lambda name: name in HARVESTED), _lib.PROFILE
    _lib.PROFILE = rec
    try:
        out = m(x)
        outs = out if isinstance(out, (tuple, list)) else (out,)
        loss = sum((o.float() * torch.randn_like(o.float())).mean() for o in outs)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        _lib.PROFILE = saved
    del m, out, outs, loss
    torch.cuda.empty_cache()
    return rec.launches


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n_tile(CoutP):
    """N tile of the per-tap kernels (conv_tc, conv_tc_dil, conv_tc_split)"""
    nt = min(128, CoutP)
    while nt > 16 and CoutP % nt:
        nt //= 2
    return nt


def _conv_tc2_plan(C0, C1, N, H, W, CoutP, ks):
    """the host dispatch of wsl_conv_tc2 (default settings): row kernel or halo kernel, its tile and N tile"""
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
    if name == "wsl_conv_tc_split":
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
    if config not in _RESULTS:
        launches = _harvest(*CONFIGS[config])
        rows, fails = [], []
        for key in launches:
            row, f = _replay(key)
            rows.append(row)
            fails += [f"{row['entry']} {row['shape']} ({row['kernel']}, {row['dtype']}): {m}" for m in f]
        _RESULTS[config] = (rows, fails)
    return _RESULTS[config]


def _print(config, rows):
    print(f"\n[{config}] {len(rows)} distinct launches")
    for r in rows:
        print(f"  {r['entry']:<19} {r['kernel']:<14} {r['dtype']:<6} {r['shape']:<28} grid {r['grid']:>5} items {r['items']:>7} "
              f"per CTA {r.get('per_cta', '-'):>4}{' ragged' if r.get('ragged') else '       '}"
              + (f" RS {r['RS']}" if r.get("RS") else "") + (f" MT {r['MT']} NT {r['NT']}" if r.get("MT") else "")
              + f"  error/bound {r['worst']:.3g}"
              + (f"  BN rows {r['stat_err']:.1e} (mean {r['mean_sigmas']:.1f} sd)" if "stat_err" in r else "")
              + (f"  bit-identical {r['bit_identical']}" if "bit_identical" in r else ""))
    fam = {}
    for r in rows:
        k = (r["kernel"], r["dtype"])
        fam[k] = max(fam.get(k, 0.0), r["worst"])
    print(f"[{config}] worst error / bound per kernel family: " + ", ".join(f"{k} {d} {v:.3g}" for (k, d), v in sorted(fam.items())))


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_convolution_launch_of_a_training_step_against_fp64(config):
    rows, fails = _run(config)
    _print(config, rows)
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


def test_conv_tc2_rejects_fp32_nhwc_output():
    """both conv_tc2 epilogues store 16-bit NHWC or fp32 NCHW; out_mode 2 (fp32 NHWC) is an error, not an NCHW write"""
    x = torch.randn(1, 16, 128, 16, device=DEV).to(torch.bfloat16)
    pk = pack_conv_weights(torch.randn(16, 16, 3, 3, device=DEV), [16])
    out = torch.zeros(1, 16, 128, 16, device=DEV)
    with pytest.raises(RuntimeError, match="out_mode"):
        call("wsl_conv_tc2", x, 16, None, 0, pk["bf"], None, out, 2, 1, 16, 128, 16, 16, 3, 0, None, None)
    torch.cuda.synchronize()
    assert not out.any()
