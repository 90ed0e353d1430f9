"""The row convolution (conv_row, wsl_conv_tc2 at 16 / 32 output channels and 128-pixel rows) against fp64.

Each output row is rounded into a shared-memory slot in the output tensor map's swizzle and leaves through a TMA tensor
store, two slots per consumer warpgroup, while the next input row's MMA group runs.  The cases cover what that touches: 16
and 32 output channels (KBW 16 and 32 channel blocks, one to four of them, one and two sources), row segments of 16 and 32
rows, CTAs with one item and with several, a last wave in which only some CTAs take another item, stored channels fewer than
the padded ones (TMA clips them), bias on and off, BatchNorm statistics on and off, the fp32 NCHW logits, maps one and two
128-pixel strips wide, bf16 and fp16.  Outputs are held to the per-element bounds of tests/_conv_check.py; the statistics rows
to fp64 sums of the stored outputs."""
import ctypes
import math

import pytest
import torch

import _conv_check as CC
from _gpu_util import pack_conv_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200._lib import call

T16 = {0: torch.bfloat16, 2: torch.float16}

# (N, H, W, C0, C1, CoutStore, dtype, out_mode, bias, stats); "rs32" cases set N from the SM count (see _shape)
CASES = {
    "nt16-kb1-one-item-per-cta": (3, 64, 256, 16, 0, 16, 0, 0, True, True),
    "nt16-kb4-two-sources-ragged": (20, 128, 256, 32, 32, 16, 2, 0, True, True),
    "nt16-kb2-clipped-no-bias": (4, 32, 128, 32, 0, 8, 0, 0, False, True),
    "nt16-kb3-fp16-no-stats": (6, 48, 128, 48, 0, 16, 2, 0, True, False),
    "nt32-kbw32-kb1-rs32": (None, 256, 128, 32, 0, 32, 0, 0, True, True),
    "nt32-kbw32-kb2-two-sources-ragged": (40, 64, 128, 32, 32, 32, 0, 0, True, False),
    "nt32-kbw16-kb3-two-sources": (8, 64, 256, 32, 16, 32, 2, 0, False, True),
    "nt32-kbw16-kb4-two-sources-fp16-rs32": (None, 64, 256, 48, 16, 32, 2, 0, True, True),
    "nt32-kbw16-kb1-clipped": (5, 16, 128, 16, 0, 24, 0, 0, True, True),
    "logits-fp32-bf16": (6, 64, 256, 16, 0, 4, 0, 1, True, False),
    "logits-fp32-fp16-ragged": (70, 32, 256, 16, 0, 4, 2, 1, True, False),
}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shape(name):
    N, H, W, *rest = CASES[name]
    if N is None:            # the smallest batch whose 32-row items reach 4 per SM (the dispatcher's RS = 32 threshold)
        per = (W // 128) * (H // 32)
        N = -(-4 * _sms() // per)
    return (N, H, W, *rest)


def _plan(C0, C1, N, H, W, CoutP):
    """the row kernel's RS and channel block, as wsl_conv_tc2 chooses them"""
    assert CoutP in (16, 32) and W % 128 == 0 and H % 16 == 0 and C0 + C1 <= 64
    rs = 32 if H % 32 == 0 and N * (W // 128) * (H // 32) >= 4 * _sms() else 16
    kbw = 32 if CoutP == 32 and C0 % 32 == 0 and C1 % 32 == 0 else 16
    return rs, kbw


@pytest.mark.parametrize("name", list(CASES))
def test_conv_row_epilogue(name):
    N, H, W, C0, C1, Cs, dt, mode, with_bias, stats = _shape(name)
    Cin = C0 + C1
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    x = (torch.randn(N, H, W, Cin, device=DEV, generator=g) * 2.0 ** (torch.rand(Cin, device=DEV, generator=g) * 4 - 2)).to(T16[dt])
    w = torch.randn(Cs, Cin, 3, 3, device=DEV, generator=g) / math.sqrt(Cin * 9)
    w64 = w.to(T16[dt]).double()
    pk = pack_conv_weights(w, [Cin], dt)
    CoutP = pk["CoutP"]
    bias = b64 = None
    if with_bias:
        b = torch.randn(Cs, device=DEV, generator=g) * 2
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = b
        b64 = b.double()
    s0 = x[..., :C0].contiguous()
    s1 = x[..., C0:].contiguous() if C1 else None
    out = torch.full((N, Cs, H, W) if mode == 1 else (N, H, W, Cs), float("nan"), device=DEV,
                     dtype=torch.float32 if mode == 1 else T16[dt])
    parts = torch.full((592 * 2 * CoutP,), float("nan"), device=DEV) if stats else None
    rows = ctypes.c_int(-1)
    call("wsl_conv_tc2", s0, C0, s1, C1, pk["bf"], bias, out, mode, N, H, W, CoutP, Cs, 3, dt, parts, ctypes.addressof(rows))
    torch.cuda.synchronize()

    rs, kbw = _plan(C0, C1, N, H, W, CoutP)
    items, grid = N * (W // 128) * (H // rs), rows.value
    assert 1 <= grid <= items
    if "rs32" in name:
        assert rs == 32 and items >= 2 * grid, (rs, items, grid)
    if "one-item" in name:
        assert items == grid, (items, grid)
    if "ragged" in name:
        assert items > grid and items % grid, (items, grid)
    if "clipped" in name:
        assert Cs < CoutP
    if "kbw" in name:
        assert f"kbw{kbw}" in name, (name, kbw)

    ref, S = CC.reference(x.permute(0, 3, 1, 2).double(), w64, b64)
    got = (out if mode == 1 else out.permute(0, 3, 1, 2)).double()
    rep = CC.check_output(got, ref, S, CC.UNIT_ROUNDOFF[T16[dt]] if mode == 0 else 0.0, CC.SLACK_16,
                          CC.Tiling(H, W, rs, 128, CoutP, grid, "xy"))
    assert rep["bad"] == 0, f"{name}: {CC.describe(rep)}"
    if stats:
        st = parts[: grid * 2 * CoutP].view(grid, 2, CoutP).double().sum(0)
        ssum, sabs, ssq = got.sum((0, 2, 3)), got.abs().sum((0, 2, 3)), (got * got).sum((0, 2, 3))
        # fp32 running sums over a few thousand pixels per thread, then an fp32 combine: 1e-5 of the magnitude
        assert ((st[0, :Cs] - ssum).abs() <= 1e-5 * sabs + 1e-6).all(), name
        assert ((st[1, :Cs] - ssq).abs() <= 1e-5 * ssq + 1e-6).all(), name
        assert torch.isfinite(st[:, :Cs]).all()
