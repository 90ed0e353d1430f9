"""The halo convolution's (conv_tc2) pipelined epilogue against fp64.

The kernel rounds a finished tile into registers, issues the next tile's first MMA group, and then accumulates the tile's
BatchNorm sums and writes it through a shared-memory staging buffer and TMA tensor stores while that group runs.  The cases
cover what that adds: CTAs with exactly one tile and a last wave in which only some CTAs take a second tile, stored channels
fewer than the padded ones (TMA clips them; the 128-channel tile is stored as two 64-channel boxes), bias absent and present,
BatchNorm statistics on and off, the fp32 NCHW logits epilogue, 1x1 and 3x3, bf16 and fp16.  Outputs are held to the
per-element bounds of tests/_conv_check.py; the statistics rows to fp64 sums of the stored outputs."""
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

# (N, H, W, Cin, CoutStore, ks, dtype, out_mode, bias, stats)
CASES = {
    "3x3-nt128-ragged-wave": (5, 64, 64, 64, 128, 3, 0, 0, True, True),
    "3x3-nt128-clipped-box": (2, 32, 32, 64, 120, 3, 2, 0, True, True),
    "3x3-mt2-one-tile-per-cta": (1, 32, 16, 32, 64, 3, 2, 0, False, False),
    "3x3-mt4-nt32": (2, 64, 64, 16, 32, 3, 2, 0, True, True),
    "3x3-no-bias-stats": (6, 32, 32, 128, 64, 3, 0, 0, False, True),
    "1x1-nt128": (4, 16, 16, 256, 128, 1, 0, 0, True, True),
    "1x1-clipped": (3, 64, 64, 16, 24, 1, 2, 0, True, True),
    "1x1-no-stats": (2, 32, 32, 64, 64, 1, 0, 0, True, False),
    "3x3-logits-fp32": (2, 64, 64, 16, 4, 3, 0, 1, True, False),
    "1x1-logits-fp32": (3, 32, 32, 32, 4, 1, 2, 1, True, False),
}


def _plan(Cin, H, CoutP, ks):
    """the halo kernel's tile (16*MT rows) and N tile, as wsl_conv_tc2 chooses them"""
    kblk = 64
    while kblk > 16 and Cin % kblk:
        kblk //= 2
    mt = {64: 1, 32: 2, 16: 4}[kblk]
    while mt > 1 and H % (16 * mt):
        mt //= 2
    nt = min(128, CoutP)
    while nt > 16 and (CoutP % nt or ks * ks * Cin * nt * 2 > 148 * 1024 or mt * nt > 128):
        nt //= 2
    return mt, nt


@pytest.mark.parametrize("name", list(CASES))
def test_conv_tc2_epilogue(name):
    N, H, W, Cin, Cs, ks, dt, mode, with_bias, stats = CASES[name]
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    x = (torch.randn(N, H, W, Cin, device=DEV, generator=g) * 2.0 ** (torch.rand(Cin, device=DEV, generator=g) * 4 - 2)).to(T16[dt])
    w = torch.randn(Cs, Cin, ks, ks, device=DEV, generator=g) / math.sqrt(Cin * ks * ks)
    w64 = w.to(T16[dt]).double()
    pk = pack_conv_weights(w, [Cin], dt)
    CoutP = pk["CoutP"]
    bias = b64 = None
    if with_bias:
        b = torch.randn(Cs, device=DEV, generator=g) * 2
        bias = torch.zeros(CoutP, device=DEV)
        bias[:Cs] = b
        b64 = b.double()
    out = torch.full((N, Cs, H, W) if mode == 1 else (N, H, W, Cs), float("nan"), device=DEV,
                     dtype=torch.float32 if mode == 1 else T16[dt])
    parts = torch.full((592 * 2 * CoutP,), float("nan"), device=DEV) if stats else None
    rows = ctypes.c_int(-1)
    call("wsl_conv_tc2", x, Cin, None, 0, pk["bf"], bias, out, mode, N, H, W, CoutP, Cs, ks, dt, parts, ctypes.addressof(rows))
    torch.cuda.synchronize()

    mt, nt = _plan(Cin, H, CoutP, ks)
    tiles, grid = N * (W // 8) * (H // (16 * mt)), rows.value
    assert 1 <= grid <= tiles
    if name.endswith("ragged-wave"):
        assert tiles > grid and tiles % grid, (tiles, grid)
    if name.endswith("one-tile-per-cta"):
        assert tiles == grid, (tiles, grid)
    if name.endswith("clipped-box") or name.endswith("clipped"):
        assert Cs < CoutP

    ref, S = CC.reference(x.permute(0, 3, 1, 2).double(), w64, b64)
    got = (out if mode == 1 else out.permute(0, 3, 1, 2)).double()
    rep = CC.check_output(got, ref, S, CC.UNIT_ROUNDOFF[T16[dt]] if mode == 0 else 0.0, CC.SLACK_16,
                          CC.Tiling(H, W, 16 * mt, 8, nt, grid))
    assert rep["bad"] == 0, f"{name}: {CC.describe(rep)}"
    if stats:
        st = parts[: grid * 2 * CoutP].view(grid, 2, CoutP).double().sum(0)
        ssum, sabs, ssq = got.sum((0, 2, 3)), got.abs().sum((0, 2, 3)), (got * got).sum((0, 2, 3))
        # fp32 running sums over at most a few hundred pixels per thread, then an fp32 combine: 1e-5 of the magnitude
        assert ((st[0, :Cs] - ssum).abs() <= 1e-5 * sabs + 1e-6).all(), name
        assert ((st[1, :Cs] - ssq).abs() <= 1e-5 * ssq + 1e-6).all(), name
        assert torch.isfinite(st[:, :Cs]).all()
