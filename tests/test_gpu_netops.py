"""Unit parity of the network operator kernels (C ABI) against plain PyTorch fp32 references of the same
op evaluated on the same bf16-rounded inputs.  bf16 outputs: tolerance = 1 bf16 ulp of the result scale
(2^-8 relative) unless stated; fp32 outputs: 1e-5 relative."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _gpu_util import bf16_round, nchw, nhwc, pack_conv_weights, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200._lib import call, workspace

BF = torch.bfloat16
T16 = {0: torch.bfloat16, 2: torch.float16}          # C-ABI dtype code -> torch dtype of the 16-bit storage / operand type
ULP = {0: 2 ** -8, 2: 2 ** -11}


def r16(x, dt):
    return x.to(T16[dt]).float()


CONV_CASES = [
    # (N, H, W, C0, C1, Cout, ks)
    (2, 16, 16, 16, 0, 16, 3), (2, 32, 32, 16, 0, 32, 3), (1, 16, 32, 32, 0, 32, 3), (2, 16, 16, 64, 0, 64, 3),
    (1, 16, 16, 128, 0, 128, 3), (1, 8, 16, 256, 0, 256, 3), (1, 16, 16, 128, 128, 128, 3), (2, 16, 16, 16, 16, 16, 3),
    (1, 32, 32, 32, 32, 32, 3), (1, 8, 16, 256, 0, 128, 1), (2, 16, 16, 32, 0, 16, 1), (1, 32, 32, 16, 0, 4, 3),
    (3, 8, 16, 64, 64, 64, 3),
    # shapes that exercise the multi-sub-tile (MT = 2, 4) persistent v2 kernel and several tiles per CTA
    (2, 64, 32, 16, 0, 16, 3), (1, 64, 64, 16, 16, 16, 3), (2, 32, 16, 32, 0, 64, 3), (1, 32, 32, 32, 32, 32, 3),
    (2, 32, 32, 64, 0, 128, 3), (1, 16, 16, 256, 0, 256, 3), (1, 32, 32, 128, 128, 128, 3), (1, 64, 64, 16, 0, 4, 3),
    (2, 16, 16, 256, 0, 128, 1), (2, 64, 64, 32, 0, 16, 1),
    # rows of >= 128 pixels with 16 / 32 (4) output channels: the row kernel (filter rows in the MMA's N dimension)
    (2, 32, 128, 16, 0, 16, 3), (1, 64, 256, 16, 16, 16, 3), (3, 16, 128, 32, 0, 32, 3), (1, 32, 128, 32, 32, 32, 3),
    (2, 48, 256, 16, 0, 4, 3), (1, 32, 128, 16, 0, 32, 3), (5, 32, 256, 32, 0, 16, 3),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("path", ["direct", "tc", "tc2", "tc-fp16", "tc2-fp16"])
def test_conv_forward(case, path):
    N, H, W, C0, C1, Cout, ks = case
    dt = 2 if path.endswith("-fp16") else 0            # fp16 operands: same kernels, kind::f16 with the fp16 format code
    path = path.split("-")[0]
    if dt == 2 and CONV_CASES.index(case) % 2:
        pytest.skip("fp16 operands: every second case")
    if path == "tc2" and (H % 16 or W % 8):
        pytest.skip("v2 tile is 8x16")
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x0 = r16(torch.randn(N, C0, H, W, generator=g), dt)
    x1 = r16(torch.randn(N, C1, H, W, generator=g), dt) if C1 else None
    w = torch.randn(Cout, C0 + C1, ks, ks, generator=g) / np.sqrt((C0 + C1) * ks * ks)
    b = torch.randn(Cout, generator=g) * 0.1
    xin = torch.cat([x0, x1], 1) if C1 else x0
    pk = pack_conv_weights(w.to(DEV), [C0, C1] if C1 else [C0], dt)
    CoutP = pk["CoutP"]
    bias = torch.zeros(CoutP, device=DEV)
    bias[:Cout] = b.to(DEV)
    s0 = nhwc(x0, T16[dt]).to(DEV)
    s1 = nhwc(x1, T16[dt]).to(DEV) if C1 else None
    fp32_out = Cout == 4
    out = torch.zeros((N, Cout, H, W), device=DEV) if fp32_out else torch.zeros((N, H, W, Cout), device=DEV, dtype=T16[dt])
    if path in ("tc", "tc2"):
        import ctypes
        rows = ctypes.c_int(0)
        parts = torch.zeros(592 * 2 * CoutP, device=DEV)
        extra = (parts, ctypes.addressof(rows)) if path == "tc2" else ()
        call("wsl_conv_tc2" if path == "tc2" else "wsl_conv_tc", s0, C0, s1, C1, pk["bf"], bias, out, 1 if fp32_out else 0,
             N, H, W, CoutP, Cout, ks, dt, *extra)
        wref = r16(w, dt)   # tensor-core path multiplies 16-bit weights
        if path == "tc2" and not fp32_out:
            # fused BatchNorm statistics: rows of per-CTA (sum, sum of squares) of the stored outputs
            torch.cuda.synchronize()
            st = parts[: rows.value * 2 * CoutP].view(rows.value, 2, CoutP).double().sum(0).cpu()
            o = nchw(out.float().cpu()).double()
            assert rows.value >= 1
            assert torch.allclose(st[0, :Cout], o.sum((0, 2, 3)), rtol=1e-5, atol=1e-3)
            assert torch.allclose(st[1, :Cout], (o * o).sum((0, 2, 3)), rtol=1e-5, atol=1e-3)
    else:
        call("wsl_conv_direct", s0, C0, s1, C1, 0, pk["wf"], bias, out, 1 if fp32_out else 0, N, H, W, pk["CinP"], CoutP, Cout, ks)
        wref = w
    torch.cuda.synchronize()
    ref = F.conv2d(xin.double(), wref.double(), b.double(), padding=ks // 2).float()
    got = out.cpu() if fp32_out else nchw(out.float().cpu())
    tol = 1e-4 if fp32_out else 2 * ULP[dt]
    err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-9)
    assert err < tol, (case, path, err)


@pytest.mark.parametrize("case", [(2, 16, 16, 16, 16, 16, 3), (1, 16, 16, 128, 128, 128, 3), (1, 8, 16, 256, 0, 128, 1),
                                  (1, 16, 32, 16, 0, 4, 3), (2, 16, 16, 32, 0, 64, 3)])
@pytest.mark.parametrize("path", ["direct", "tc", "tc2", "tc2-fp16"])
def test_conv_dgrad(case, path):
    N, H, W, C0, C1, Cout, ks = case
    dt = 2 if path.endswith("-fp16") else 0
    path = path.split("-")[0]
    if path == "tc2" and (H % 16 or W % 8):
        pytest.skip("v2 tile is 8x16")
    g = torch.Generator().manual_seed(11)
    Cin = C0 + C1
    w = torch.randn(Cout, Cin, ks, ks, generator=g) / np.sqrt(Cin * ks * ks)
    CoutP = (Cout + 15) // 16 * 16
    dy = torch.zeros(N, CoutP, H, W)
    dy[:, :Cout] = r16(torch.randn(N, Cout, H, W, generator=g), dt)
    pk = pack_conv_weights(w.to(DEV), [C0, C1] if C1 else [C0], dt)
    dyd = nhwc(dy, T16[dt]).to(DEV)
    wr = r16(w, dt) if path != "direct" else w
    ref = F.conv_transpose2d(dy[:, :Cout].double(), wr.double(), padding=ks // 2).float()
    beg = 0
    for i, c in enumerate([C0, C1] if C1 else [C0]):
        sp = (c + 15) // 16 * 16
        out = torch.zeros((N, H, W, c), device=DEV, dtype=T16[dt])
        if path != "direct":
            extra = (None, None) if path == "tc2" else ()
            call("wsl_conv_tc2" if path == "tc2" else "wsl_conv_tc", dyd, CoutP, None, 0, pk["bd"][i], None, out, 0, N, H, W, sp, c, ks, dt, *extra)
        else:
            call("wsl_conv_direct", dyd, CoutP, None, 0, 0, pk["wd"][i], None, out, 0, N, H, W, CoutP, sp, c, ks)
        torch.cuda.synchronize()
        r = ref[:, beg:beg + c]
        err = (nchw(out.float().cpu()) - r).abs().max().item() / (r.abs().max().item() + 1e-9)
        assert err < 2 * ULP[dt], (case, path, i, err)
        beg += c


@pytest.mark.parametrize("case", [(2, 16, 16, 16, 16, 16, 3), (1, 16, 16, 64, 0, 64, 3), (2, 8, 16, 32, 0, 16, 1),
                                  (2, 32, 32, 16, 0, 4, 3), (3, 24, 40, 1, 0, 16, 3)])
def test_wgrad_direct(case):
    N, H, W, C0, C1, Cout, ks = case
    g = torch.Generator().manual_seed(5)
    Cin = C0 + C1
    f32src = C0 == 1
    x = torch.randn(N, Cin, H, W, generator=g)
    if not f32src:
        x = bf16_round(x)
    CoutP = (Cout + 15) // 16 * 16
    dy = torch.zeros(N, CoutP, H, W)
    dy[:, :Cout] = bf16_round(torch.randn(N, Cout, H, W, generator=g))
    dw = torch.zeros(Cout, Cin, ks, ks, device=DEV)
    db = torch.zeros(Cout, device=DEV)
    if f32src:
        s0, s1 = x.to(DEV).contiguous(), None
    else:
        s0 = nhwc(x[:, :C0]).to(DEV)
        s1 = nhwc(x[:, C0:]).to(DEV) if C1 else None
    call("wsl_wgrad_direct", s0, C0, s1, C1, 1 if f32src else 0, nhwc(dy).to(DEV), 0, CoutP, dw, db, N, H, W, Cout, ks)
    torch.cuda.synchronize()
    xr = x.double().requires_grad_(False)
    wz = torch.zeros(Cout, Cin, ks, ks, dtype=torch.double, requires_grad=True)
    bz = torch.zeros(Cout, dtype=torch.double, requires_grad=True)
    out = F.conv2d(xr, wz, bz, padding=ks // 2)
    gw, gb = torch.autograd.grad(out, [wz, bz], dy[:, :Cout].double())
    assert rel_l2(dw.cpu(), gw.float()) < 1e-5
    assert rel_l2(db.cpu(), gb.float()) < 1e-5


WGRAD_TC_CASES = [
    (2, 16, 16, 16, 0, 16, 3), (2, 16, 32, 16, 0, 32, 3), (1, 32, 32, 32, 0, 32, 3), (2, 16, 16, 64, 0, 64, 3),
    (1, 16, 16, 128, 0, 128, 3), (1, 8, 16, 256, 0, 256, 3), (1, 16, 16, 128, 128, 128, 3), (2, 16, 16, 16, 16, 16, 3),
    (1, 16, 32, 32, 32, 32, 3), (2, 16, 16, 64, 64, 64, 3), (1, 8, 16, 256, 0, 128, 1), (2, 16, 16, 32, 0, 16, 1),
    (2, 16, 16, 64, 0, 32, 1), (1, 32, 32, 16, 0, 4, 3), (3, 8, 16, 32, 0, 64, 3), (2, 16, 16, 64, 0, 128, 3),
]


WGRAD_TC_CASES += [(2, 32, 32, 16, 0, 16, 3), (1, 64, 32, 32, 32, 32, 3), (2, 32, 16, 64, 0, 128, 3), (1, 32, 32, 128, 128, 128, 3),
                   (1, 16, 16, 256, 0, 256, 3), (2, 32, 32, 16, 0, 4, 3), (1, 48, 24, 32, 0, 64, 3)]


@pytest.mark.parametrize("case", WGRAD_TC_CASES)
@pytest.mark.parametrize("ver", ["wsl_wgrad_tc", "wsl_wgrad_tc2", "wsl_wgrad_tc3", "wsl_wgrad_tc3-fp16"])
def test_wgrad_tc(case, ver):
    """wgmma weight gradient vs fp64 autograd on the same 16-bit inputs; fp32 accumulation -> 1e-4 relative."""
    N, H, W, C0, C1, Cout, ks = case
    dt = 2 if ver.endswith("-fp16") else 0
    ver = ver.split("-")[0]
    if ver != "wsl_wgrad_tc" and (ks != 3 or H % 16 or W % 8):
        pytest.skip("v2: 3x3, 8x16 chunks")
    if ver == "wsl_wgrad_tc" and (H % 8 or W % 16):
        pytest.skip("v1: 16x8 chunks")
    g = torch.Generator().manual_seed(17)
    Cin = C0 + C1
    x = r16(torch.randn(N, Cin, H, W, generator=g), dt)
    CoutP = (Cout + 15) // 16 * 16
    dy = torch.zeros(N, CoutP, H, W)
    dy[:, :Cout] = r16(torch.randn(N, Cout, H, W, generator=g), dt)
    dw = torch.zeros(Cout, Cin, ks, ks, device=DEV)
    s0 = nhwc(x[:, :C0], T16[dt]).to(DEV)
    s1 = nhwc(x[:, C0:], T16[dt]).to(DEV) if C1 else None
    dyd = nhwc(dy, T16[dt]).to(DEV)
    extra = ()
    if ver in ("wsl_wgrad_tc3", "wsl_wgrad_tc"):   # deterministic split-K: partial tiles + fixed-order finalize (None -> atomics)
        pw = torch.empty(8 * 1024 * 1024, device=DEV) if (hash(case) % 3) else None
        extra = (pw, pw.numel() if pw is not None else 0)
    call(ver, s0, C0, s1, C1, dyd, CoutP, dw, N, H, W, Cout, ks, dt, *extra)
    db = torch.zeros(Cout, device=DEV)
    call("wsl_channel_sum", dyd, dt, N * H * W, CoutP, Cout, db, workspace("csum") if (hash(case) % 2) else None)
    torch.cuda.synchronize()
    wz = torch.zeros(Cout, Cin, ks, ks, dtype=torch.double, requires_grad=True)
    bz = torch.zeros(Cout, dtype=torch.double, requires_grad=True)
    out = F.conv2d(x.double(), wz, bz, padding=ks // 2)
    gw, gb = torch.autograd.grad(out, [wz, bz], dy[:, :Cout].double())
    assert rel_l2(dw.cpu(), gw.float()) < 1e-4, (case, rel_l2(dw.cpu(), gw.float()))
    assert rel_l2(db.cpu(), gb.float()) < 1e-5
    # accumulation semantics: a second call doubles the result
    call(ver, s0, C0, s1, C1, dyd, CoutP, dw, N, H, W, Cout, ks, dt, *extra)
    torch.cuda.synchronize()
    assert rel_l2(dw.cpu(), 2 * gw.float()) < 1e-4
    if extra and extra[0] is not None:   # bit-stable: two fresh runs give identical bits
        d1, d2 = torch.zeros_like(dw), torch.zeros_like(dw)
        call(ver, s0, C0, s1, C1, dyd, CoutP, d1, N, H, W, Cout, ks, dt, *extra)
        call(ver, s0, C0, s1, C1, dyd, CoutP, d2, N, H, W, Cout, ks, dt, *extra)
        torch.cuda.synchronize()
        assert torch.equal(d1, d2)


SPLIT_CASES = [(2, 16, 16, 16, 0, 16, 3), (1, 16, 32, 32, 32, 32, 3), (1, 8, 16, 256, 0, 128, 1), (1, 16, 16, 128, 128, 128, 3),
               (2, 32, 32, 16, 0, 4, 3), (1, 8, 16, 256, 0, 256, 3), (2, 16, 16, 64, 0, 32, 1)]


@pytest.mark.parametrize("case", SPLIT_CASES)
def test_split_convolutions(case):
    """fp16 hi/lo split ("fp16x3") tensor-core convolutions on fp32 operands vs fp64: forward, data gradient and weight
    gradient must be fp32-accurate (the dropped lo*lo term is 2^-22 relative)."""
    N, H, W, C0, C1, Cout, ks = case
    g = torch.Generator().manual_seed(23)
    Cin, T, P = C0 + C1, ks * ks, N * H * W
    CoutP = (Cout + 15) // 16 * 16
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, ks, ks, generator=g) / np.sqrt(Cin * T)
    b = torch.randn(Cout, generator=g) * 0.1
    dy = torch.zeros(N, CoutP, H, W)
    dy[:, :Cout] = torch.randn(N, Cout, H, W, generator=g)
    s0 = nhwc(x[:, :C0], torch.float32).to(DEV)
    s1 = nhwc(x[:, C0:], torch.float32).to(DEV) if C1 else None
    f3 = torch.zeros(T * CoutP * 3 * Cin, device=DEV, dtype=torch.float16)
    d3 = [torch.zeros(T * c * 3 * CoutP, device=DEV, dtype=torch.float16) for c in ([C0, C1] if C1 else [C0])]
    beg = 0
    for i, c in enumerate([C0, C1] if C1 else [C0]):
        call("wsl_pack_split_weights", w.to(DEV), Cout, Cin, ks, CoutP, Cin, beg, c, f3 if i == 0 else None, d3[i])
        beg += c
    bias = torch.zeros(CoutP, device=DEV)
    bias[:Cout] = b.to(DEV)
    sx = torch.zeros((P, 2 * Cin), device=DEV, dtype=torch.float16)
    kx = torch.zeros(3, device=DEV)
    call("wsl_split_f32", s0, C0, s1, C1, P, sx, kx)
    torch.cuda.synchronize()
    xs = sx.float().cpu()
    amax = x.abs().max().item()
    assert 2 ** 13 <= amax * kx[0].item() < 2 ** 14 and kx[0].item() * kx[1].item() == 1.0
    assert ((xs[:, :Cin] + xs[:, Cin:]) * kx[1].item() - nhwc(x, torch.float32).reshape(P, Cin)).abs().max().item() < 1e-6 * amax
    # forward
    fp32_nchw = Cout == 4
    out = torch.zeros((N, Cout, H, W) if fp32_nchw else (N, H, W, Cout), device=DEV)
    call("wsl_conv_tc_split", sx, Cin, kx[1:], f3, bias, out, 1 if fp32_nchw else 2, N, H, W, CoutP, Cout, ks, 1)
    torch.cuda.synchronize()
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=ks // 2).float()
    got = out.cpu() if fp32_nchw else nchw(out.cpu())
    assert (got - ref).abs().max().item() < 2e-5 * ref.abs().max().item(), (got - ref).abs().max().item() / ref.abs().max().item()
    # data gradient per concatenated source
    sg = torch.zeros((P, 2 * CoutP), device=DEV, dtype=torch.float16)
    kg = torch.zeros(3, device=DEV)
    call("wsl_split_f32", (nhwc(dy, torch.float32) * 1e-6).to(DEV), CoutP, None, 0, P, sg, kg)      # tiny gradients: the per-tensor scale must cope
    dy = dy * 1e-6
    refd = F.conv_transpose2d(dy[:, :Cout].double(), w.double(), padding=ks // 2).float()
    beg = 0
    for i, c in enumerate([C0, C1] if C1 else [C0]):
        o = torch.zeros((N, H, W, c), device=DEV)
        call("wsl_conv_tc_split", sg, CoutP, kg[1:], d3[i], None, o, 2, N, H, W, c, c, ks, 1)
        torch.cuda.synchronize()
        r = refd[:, beg:beg + c]
        assert (nchw(o.cpu()) - r).abs().max().item() < 2e-5 * r.abs().max().item()
        beg += c
    # weight gradient
    dw = torch.zeros(Cout, Cin, ks, ks, device=DEV)
    call("wsl_wgrad_tc_split", sx, Cin, kx[1:], sg, CoutP, kg[1:], dw, N, H, W, Cout, ks, 1)
    torch.cuda.synchronize()
    wz = torch.zeros(Cout, Cin, ks, ks, dtype=torch.double, requires_grad=True)
    (gw,) = torch.autograd.grad(F.conv2d(x.double(), wz, None, padding=ks // 2), wz, dy[:, :Cout].double())
    assert rel_l2(dw.cpu(), gw.float()) < 2e-6, rel_l2(dw.cpu(), gw.float())


@pytest.mark.parametrize("shape", [(2, 32, 32), (3, 24, 40), (1, 7, 9)])
def test_first_layer_kernels(shape):
    N, H, W = shape
    g = torch.Generator().manual_seed(21)
    x = torch.rand(N, 1, H, W, generator=g)
    w = torch.randn(16, 1, 3, 3, generator=g) * 0.5
    b = torch.randn(16, generator=g) * 0.1
    y = torch.zeros((N, H, W, 16), device=DEV, dtype=BF)
    import ctypes
    rows = ctypes.c_int(0)
    parts = torch.zeros(592 * 2 * 16, device=DEV)
    call("wsl_conv_first", x.to(DEV), w.to(DEV), b.to(DEV), y, 0, N, H, W, 16, parts, ctypes.addressof(rows))
    torch.cuda.synchronize()
    ref = F.conv2d(x, w, b, padding=1)
    assert (nchw(y.cpu()) - ref).abs().max().item() <= 2 ** -8 * ref.abs().max().item()
    st = parts[: rows.value * 32].view(rows.value, 2, 16).double().sum(0).cpu()        # fused BatchNorm statistics of the stored values
    o = nchw(y.cpu()).double()
    assert torch.allclose(st[0], o.sum((0, 2, 3)), rtol=1e-5, atol=1e-3) and torch.allclose(st[1], (o * o).sum((0, 2, 3)), rtol=1e-5, atol=1e-3)
    dy = bf16_round(torch.randn(N, 16, H, W, generator=g))
    dw = torch.zeros(16, 1, 3, 3, device=DEV)
    call("wsl_wgrad_first", x.to(DEV), nhwc(dy).to(DEV), 0, dw, N, H, W, 16)
    torch.cuda.synchronize()
    wz = torch.zeros(16, 1, 3, 3, dtype=torch.double, requires_grad=True)
    (gw,) = torch.autograd.grad(F.conv2d(x.double(), wz, None, padding=1), wz, dy.double())
    assert rel_l2(dw.cpu(), gw.float()) < 1e-5


@pytest.mark.parametrize("shape", [(2, 16, 16, 16), (3, 8, 24, 64), (1, 4, 4, 256), (2, 32, 32, 32), (8, 64, 64, 16)])
def test_bn_stats_and_act(shape):
    N, H, W, C = shape
    g = torch.Generator().manual_seed(2)
    y = bf16_round(torch.randn(N, C, H, W, generator=g) * 1.7 + 0.3)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    yd = nhwc(y).to(DEV)
    save, ss = torch.zeros(2 * C, device=DEV), torch.zeros(2 * C, device=DEV)
    rmd, rvd = rm.to(DEV), rv.to(DEV)
    nbt = torch.zeros((), dtype=torch.int64, device=DEV)
    call("wsl_bn_stats", yd, 0, N * H * W, C, gamma.to(DEV), beta.to(DEV), rmd, rvd, nbt, 0.1, 1e-5, save, ss, workspace("bn"), None)
    rm2, rv2 = rm.clone(), rv.clone()
    ref = F.batch_norm(y, rm2, rv2, gamma, beta, True, 0.1, 1e-5)
    torch.cuda.synchronize()
    assert nbt.item() == 1
    assert torch.allclose(rmd.cpu(), rm2, atol=1e-5) and torch.allclose(rvd.cpu(), rv2, rtol=1e-4, atol=1e-5)
    mean = y.mean((0, 2, 3))
    assert torch.allclose(save[:C].cpu(), mean, atol=1e-5)
    # activation + dropout mask + pool
    p = 0.3
    mask = (torch.rand(N, C, H, W, generator=g) >= p)
    act = torch.zeros((N, H, W, C), device=DEV, dtype=BF)
    pooled = torch.zeros((N, H // 2, W // 2, C), device=DEV, dtype=BF)
    pidx = torch.zeros((N, H // 2, W // 2, C), device=DEV, dtype=torch.uint8)
    mk = mask.permute(0, 2, 3, 1).contiguous().to(torch.uint8).to(DEV)
    call("wsl_bn_act_fwd", yd, 0, ss, N, H, W, C, 0.01, p, mk, 0, None, act, pooled, pidx)
    torch.cuda.synchronize()
    ra = F.leaky_relu(ref, 0.01) * mask / (1 - p)
    assert (nchw(act.cpu()) - ra).abs().max().item() <= 2 ** -8 * ra.abs().max().item() + 1e-6
    rp, ri = F.max_pool2d(nchw(act.cpu()), 2, return_indices=True)
    assert torch.equal(nchw(pooled.cpu()), rp)
    # pool index k = 2*dy+dx inside the window must point at a maximal element
    a = nchw(act.cpu())
    k = pidx.cpu().permute(0, 3, 1, 2).long()
    yy = torch.arange(H // 2).view(1, 1, -1, 1) * 2 + (k >> 1)
    xx = torch.arange(W // 2).view(1, 1, 1, -1) * 2 + (k & 1)
    picked = a.flatten(2).gather(2, (yy * W + xx).flatten(2)).view_as(rp)
    assert torch.equal(picked, rp)
    # counter-RNG dropout keeps ~ (1-p) of the elements and is reproduced by the same seed
    a1 = torch.zeros_like(act)
    a2 = torch.zeros_like(act)
    call("wsl_bn_act_fwd", yd, 0, ss, N, H, W, C, 0.01, p, None, 1234, None, a1, None, None)
    call("wsl_bn_act_fwd", yd, 0, ss, N, H, W, C, 0.01, p, None, 1234, None, a2, None, None)
    torch.cuda.synchronize()
    assert torch.equal(a1, a2)
    frac = (a1 != 0).float().mean().item()
    assert abs(frac - (1 - p)) < 0.05


@pytest.mark.parametrize("shape", [(2, 16, 16, 16), (2, 8, 24, 64), (2, 32, 32, 32)])
def test_bn_backward_chain(shape):
    """dY, dgamma, dbeta of conv-out -> BN(train) -> LeakyReLU -> dropout -> {identity, channel-scale, maxpool}."""
    N, H, W, C = shape
    g = torch.Generator().manual_seed(9)
    y = bf16_round(torch.randn(N, C, H, W, generator=g) * 1.3 + 0.2)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    p = 0.2
    mask = (torch.rand(N, C, H, W, generator=g) >= p)
    cs = (torch.rand(N, C, generator=g) >= 0.5).float() * 2
    g0 = bf16_round(torch.randn(N, C, H, W, generator=g))
    g1 = bf16_round(torch.randn(N, C, H, W, generator=g))
    gp = bf16_round(torch.randn(N, C, H // 2, W // 2, generator=g))
    # reference with autograd (fp64)
    yr = y.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = F.batch_norm(yr, None, None, gr, br, True, 0.1, 1e-5)
    a = F.leaky_relu(z, 0.01) * mask / (1 - p)
    a_bf = a.detach().float().to(BF).double()           # the stored activation the pool sees
    _, idx = F.max_pool2d(a_bf, 2, return_indices=True)
    pool_grad = torch.zeros(N, C, H * W, dtype=torch.double).scatter_(2, idx.flatten(2), gp.double().flatten(2)).view(N, C, H, W)
    upstream = g0.double() + g1.double() * cs.double()[:, :, None, None] + pool_grad
    dyr, dgr, dbr = torch.autograd.grad(a, [yr, gr, br], upstream)
    # kernels
    yd = nhwc(y).to(DEV)
    save, ss = torch.zeros(2 * C, device=DEV), torch.zeros(2 * C, device=DEV)
    call("wsl_bn_stats", yd, 0, N * H * W, C, gamma.to(DEV), beta.to(DEV), None, None, None, 0.1, 1e-5, save, ss, workspace("bn"), None)
    act = torch.zeros((N, H, W, C), device=DEV, dtype=BF)
    pooled = torch.zeros((N, H // 2, W // 2, C), device=DEV, dtype=BF)
    pidx = torch.zeros((N, H // 2, W // 2, C), device=DEV, dtype=torch.uint8)
    mk = mask.permute(0, 2, 3, 1).contiguous().to(torch.uint8).to(DEV)
    call("wsl_bn_act_fwd", yd, 0, ss, N, H, W, C, 0.01, p, mk, 0, None, act, pooled, pidx)
    dgam, dbet, coef = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(2 * C, device=DEV)
    dy = torch.zeros((N, H, W, C), device=DEV, dtype=BF)
    call("wsl_bn_bwd", yd, 0, ss, save, nhwc(g0).to(DEV), nhwc(g1).to(DEV), cs.to(DEV), nhwc(gp).to(DEV), pidx, mk, 0, None, p,
         0.01, N, H, W, C, dgam, dbet, coef, dy, workspace("bn"), 0)
    torch.cuda.synchronize()
    assert rel_l2(dgam.cpu(), dgr.float()) < 1e-4
    assert rel_l2(dbet.cpu(), dbr.float()) < 1e-4
    assert rel_l2(nchw(dy.cpu()), dyr.float()) < 2 ** -8


@pytest.mark.parametrize("shape", [(2, 16, 16), (3, 24, 40), (2, 64, 128)])
@pytest.mark.parametrize("dt", [0, 1])
def test_first_layer_fused_backward(shape, dt):
    """wsl_bn_bwd_first: conv(1->16) -> BN(train) -> LeakyReLU -> dropout; dgamma, dbeta and the convolution's weight gradient
    against fp64 autograd (dY itself is never materialised)."""
    N, H, W = shape
    C = 16
    g = torch.Generator().manual_seed(41)
    x = torch.rand(N, 1, H, W, generator=g)
    w = torch.randn(C, 1, 3, 3, generator=g) * 0.5
    b = torch.randn(C, generator=g) * 0.1
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    p = 0.05
    mask = (torch.rand(N, C, H, W, generator=g) >= p)
    g0 = torch.randn(N, C, H, W, generator=g)
    tdt = torch.float32 if dt == 1 else BF
    y = F.conv2d(x, w, b, padding=1).to(tdt).float()           # the stored convolution output
    g0 = g0.to(tdt).float()
    wr = w.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    yr = F.conv2d(x.double(), wr, b.double(), padding=1)
    yr = yr + (y.double() - yr).detach()                        # evaluate at the stored values, differentiate through the conv
    a = F.leaky_relu(F.batch_norm(yr, None, None, gr, br, True, 0.1, 1e-5), 0.01) * mask / (1 - p)
    dwr, dgr, dbr = torch.autograd.grad(a, [wr, gr, br], g0.double())
    yd = nhwc(y, tdt).to(DEV)
    save, ss = torch.zeros(2 * C, device=DEV), torch.zeros(2 * C, device=DEV)
    call("wsl_bn_stats", yd, dt, N * H * W, C, gamma.to(DEV), beta.to(DEV), None, None, None, 0.1, 1e-5, save, ss, workspace("bn"), None)
    mk = mask.permute(0, 2, 3, 1).contiguous().to(torch.uint8).to(DEV)
    dgam, dbet, coef = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(2 * C, device=DEV)
    dw = torch.zeros(C, 1, 3, 3, device=DEV)
    call("wsl_bn_bwd_first", yd, dt, ss, save, nhwc(g0, tdt).to(DEV), mk, 0, None, p, 0.01, N, H, W, dgam, dbet, coef, x.to(DEV), dw,
         workspace("bn"), 0)
    torch.cuda.synchronize()
    tol = 1e-4 if dt == 1 else 2 ** -7
    assert rel_l2(dgam.cpu(), dgr.float()) < tol and rel_l2(dbet.cpu(), dbr.float()) < tol
    assert rel_l2(dw.cpu(), dwr.float()) < tol, rel_l2(dw.cpu(), dwr.float())


def test_bn_backward_is_well_conditioned_at_the_baseline_shape():
    """4 x 256 x 256 x 16 in fp32 storage with a channel mean of several standard deviations (first-layer convolution outputs on
    non-negative images look like this): dgamma / dbeta / dY against fp64.  The reduction accumulates sum(dz*z) on the normalised
    value; the raw-moment form sum(dz*y) - mean*sum(dz) lost two to three digits here."""
    N, H, W, C = 4, 256, 256, 16
    g = torch.Generator().manual_seed(31)
    y = torch.randn(N, C, H, W, generator=g) * 0.4 + torch.linspace(-3, 3, C).view(1, C, 1, 1)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    g0 = torch.randn(N, C, H, W, generator=g) * 1e-3
    yr = y.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    a = F.leaky_relu(F.batch_norm(yr, None, None, gr, br, True, 0.1, 1e-5), 0.01)
    dyr, dgr, dbr = torch.autograd.grad(a, [yr, gr, br], g0.double())
    yd = nhwc(y, torch.float32).to(DEV)
    save, ss = torch.zeros(2 * C, device=DEV), torch.zeros(2 * C, device=DEV)
    call("wsl_bn_stats", yd, 1, N * H * W, C, gamma.to(DEV), beta.to(DEV), None, None, None, 0.1, 1e-5, save, ss, workspace("bn"), None)
    dgam, dbet, coef = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(2 * C, device=DEV)
    dy = torch.zeros((N, H, W, C), device=DEV)
    call("wsl_bn_bwd", yd, 1, ss, save, nhwc(g0, torch.float32).to(DEV), None, None, None, None, None, 0, None, 0.0, 0.01, N, H, W, C,
         dgam, dbet, coef, dy, workspace("bn"), 0)
    torch.cuda.synchronize()
    e = (rel_l2(dgam.cpu(), dgr.float()), rel_l2(dbet.cpu(), dbr.float()), rel_l2(nchw(dy.cpu()), dyr.float()))
    print("bn_bwd at 4x256x256x16, fp32: rel-L2 dgamma %.2e dbeta %.2e dY %.2e" % e)
    assert e[0] < 3e-4 and e[1] < 3e-4 and e[2] < 3e-4, e      # measured 7e-5 / 1e-4 / 6e-5


@pytest.mark.parametrize("shape", [(2, 4, 4, 16), (1, 16, 8, 32), (2, 2, 2, 128)])
def test_upsample(shape):
    N, h, w, C = shape
    g = torch.Generator().manual_seed(4)
    t = bf16_round(torch.randn(N, C, h, w, generator=g))
    u = torch.zeros((N, 2 * h, 2 * w, C), device=DEV, dtype=BF)
    call("wsl_upsample2x_fwd", nhwc(t).to(DEV), 0, N, h, w, C, u)
    tr = t.clone().requires_grad_(True)
    ref = F.interpolate(tr, scale_factor=2, mode="bilinear", align_corners=True)
    torch.cuda.synchronize()
    assert (nchw(u.cpu()) - ref.detach()).abs().max().item() <= 2 ** -8 * ref.abs().max().item()
    du = bf16_round(torch.randn(N, C, 2 * h, 2 * w, generator=g))
    (gt,) = torch.autograd.grad(ref, tr, du)
    dt = torch.zeros((N, h, w, C), device=DEV, dtype=BF)
    call("wsl_upsample2x_bwd", nhwc(du).to(DEV), 0, N, h, w, C, dt)
    torch.cuda.synchronize()
    assert rel_l2(nchw(dt.cpu()), gt) < 2 ** -8


def test_sgd_matches_torch():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(10007, generator=g)
    ref = torch.nn.Parameter(w.clone())
    opt = torch.optim.SGD([ref], lr=0.01, momentum=0.9, weight_decay=1e-4)
    p, m = w.to(DEV), torch.zeros(10007, device=DEV)
    lr_dev = torch.tensor([0.01], device=DEV)
    for it in range(3):
        gr = torch.randn(10007, generator=g)
        ref.grad = gr.clone()
        opt.step()
        call("wsl_sgd_step", p, gr.to(DEV), m, 10007, lr_dev if it % 2 else None, 0.01, 0.9, 1e-4, 1.0)
    torch.cuda.synchronize()
    assert torch.allclose(p.cpu(), ref.data, atol=2e-7)


def test_chan_dropout():
    N, H, W, C = 3, 8, 8, 32
    cs = torch.zeros(N * C, device=DEV)
    call("wsl_chan_mask_gen", 42, None, N * C, 0.5, cs)
    torch.cuda.synchronize()
    vals = set(cs.cpu().unique().tolist())
    assert vals <= {0.0, 2.0} and len(vals) == 2
    a = bf16_round(torch.randn(N, C, H, W))
    d = torch.zeros((N, H, W, C), device=DEV, dtype=BF)
    call("wsl_chan_scale", nhwc(a).to(DEV), 0, cs, N, H, W, C, d)
    torch.cuda.synchronize()
    assert torch.equal(nchw(d.cpu()), a * cs.cpu().view(N, C, 1, 1))


@pytest.mark.parametrize("dt", [0, 1, 2])
@pytest.mark.parametrize("C,Creal", [(320, 320), (128, 128), (16, 4), (48, 40)])
@pytest.mark.parametrize("det", [False, True])
def test_channel_sum_any_width(dt, C, Creal, det):
    """bias gradient of the 1x1 heads: channel counts that do not divide the 256-thread block (PNet2D's 320-channel concat head, 40
    pixel groups) and more than 256 real channels in the deterministic last-block combine"""
    P = 2 * 40 * 24
    g = torch.Generator().manual_seed(C + dt)
    x = torch.randn(P, C, generator=g)
    xd = x.to({0: torch.bfloat16, 1: torch.float32, 2: torch.float16}[dt]).to(DEV)
    out = torch.ones(Creal, device=DEV)
    for _ in range(2):                    # accumulates, and the workspace ticket resets
        call("wsl_channel_sum", xd, dt, P, C, Creal, out, workspace("csum") if det else None)
    torch.cuda.synchronize()
    want = 1 + 2 * xd.double().sum(0)[:Creal].cpu()
    assert (out.cpu().double() - want).abs().max().item() < 1e-3, (out.cpu().double() - want).abs().max().item()


@pytest.mark.parametrize("dil", [2, 4, 16])
@pytest.mark.parametrize("dt", [0, 2])
def test_dilated_convolution(dil, dt):
    """PNet2D's dilated 3x3 blocks (networks/pnet.py:25-28) on the per-tap wgmma kernel: forward, data gradient and weight gradient
    against fp64 F.conv2d(dilation=d, padding=d) on the same 16-bit inputs."""
    N, H, W, C, Cout, ks = 2, 32, 32, 64, 64, 3
    g = torch.Generator().manual_seed(100 + dil)
    x = r16(torch.randn(N, C, H, W, generator=g), dt)
    w = torch.randn(Cout, C, ks, ks, generator=g) / np.sqrt(C * 9)
    b = torch.randn(Cout, generator=g) * 0.1
    dy = r16(torch.randn(N, Cout, H, W, generator=g), dt)
    pk = pack_conv_weights(w.to(DEV), [C], dt)
    xd, dyd = nhwc(x, T16[dt]).to(DEV), nhwc(dy, T16[dt]).to(DEV)
    out = torch.zeros((N, H, W, Cout), device=DEV, dtype=T16[dt])
    call("wsl_conv_tc_dil", xd, C, None, 0, pk["bf"], b.to(DEV), out, 0, N, H, W, Cout, Cout, ks, dt, dil)
    dx = torch.zeros((N, H, W, C), device=DEV, dtype=T16[dt])
    call("wsl_conv_tc_dil", dyd, Cout, None, 0, pk["bd"][0], None, dx, 0, N, H, W, C, C, ks, dt, dil)
    dw = torch.zeros(Cout, C, ks, ks, device=DEV)
    pw = torch.empty(8 * 1024 * 1024, device=DEV)
    call("wsl_wgrad_tc_dil", xd, C, None, 0, dyd, Cout, dw, N, H, W, Cout, ks, dt, dil, pw, pw.numel())
    torch.cuda.synchronize()
    xr = x.double().requires_grad_(True)
    wr = r16(w, dt).double().requires_grad_(True)
    ref = F.conv2d(xr, wr, b.double(), padding=dil, dilation=dil)
    gx, gw = torch.autograd.grad(ref, [xr, wr], dy.double())
    assert (nchw(out.float().cpu()) - ref.detach().float()).abs().max().item() < 2 * ULP[dt] * ref.abs().max().item()
    assert (nchw(dx.float().cpu()) - gx.float()).abs().max().item() < 2 * ULP[dt] * gx.abs().max().item()
    assert rel_l2(dw.cpu(), gw.float()) < 1e-4
