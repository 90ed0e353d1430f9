"""The checker of tests/test_gpu_conv_at_scale.py, on the CPU: correctly rounded fp64 convolutions pass, and the mistakes a
pipelined tensor-core kernel makes when a CTA walks several tiles (a stale stage, a missing k-block or tap, a zeroed channel
group, a split-K chunk left out of the weight gradient) are flagged at the tile that holds them.  Likewise for the CUDA-core direct
convolution: an fp32 restatement of its accumulation order passes its bound at the fp32 mode's depths, and its own mistakes (a second
source read without the C0 offset, a dropped 16-channel chunk, a thread's second pixel row stored over its first, a skipped
weight-gradient split, dbias added by every ci block or missing one split) are flagged."""
import pytest
import torch

import _conv_check as CC

N, H, W, CIN, COUT, KS = 2, 32, 256, 32, 32, 3
TILINGS = {
    "conv_tc2": CC.Tiling(H, W, 32, 8, 16, grid=10),              # MT = 2 halo tiles, two N tiles of 16, 10 persistent CTAs
    "conv_row": CC.Tiling(H, W, 16, 128, 32, grid=3, order="xy"),  # (image, 128-pixel strip, 16-row segment) items
    "conv_tc": CC.Tiling(H, W, 8, 16, 32),                        # one CTA per 8 x 16 tile
}


def _r16(t):
    return t.to(torch.bfloat16).double()


@pytest.fixture(scope="module")
def case():
    g = torch.Generator().manual_seed(3)
    scale = 2.0 ** (torch.rand(CIN, generator=g, dtype=torch.float64) * 8 - 4)     # per input channel, 2^-4 .. 2^4
    x = _r16(torch.randn(N, CIN, H, W, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1))
    w = _r16(torch.randn(COUT, CIN, KS, KS, generator=g, dtype=torch.float64) / (CIN * KS * KS) ** 0.5)
    b = torch.randn(COUT, generator=g, dtype=torch.float64)
    ref, S = CC.reference(x, w, b)
    return x, w, b, ref, S, _r16(ref)


def _origin(tl, t):
    ty, tx = tl.H // tl.th, tl.W // tl.tw
    n, r = divmod(t, ty * tx)
    y, x = divmod(r, tx) if tl.order == "yx" else divmod(r, ty)[::-1]
    return n, y * tl.th, x * tl.tw


def _region(tl, t):
    n, y0, x0 = _origin(tl, t)
    return n, slice(y0, y0 + tl.th), slice(x0, x0 + tl.tw)


def _check(got, ref, S, tl):
    return CC.check_output(got, ref, S, CC.UNIT_ROUNDOFF[torch.bfloat16], CC.SLACK_16, tl)


def _flagged_tiles(rep):
    return sorted({t for t, _ in rep["tiles"]})


@pytest.mark.parametrize("kind", list(TILINGS))
def test_correct_results_pass(case, kind):
    _, _, _, ref, S, got = case
    rep = _check(got, ref, S, TILINGS[kind])
    assert rep["bad"] == 0 and rep["worst"] <= 1.0, rep
    # fp32 outputs of the split path: fp32 rounding of the exact result is inside the allowance
    rep = CC.check_output(ref.float(), ref, S, 0.0, CC.split_slack(CIN * KS * KS))
    assert rep["bad"] == 0, rep


def test_split_slack():
    assert CC.split_slack(16) < 2.0 ** -19 and 2.0 ** -18 < CC.split_slack(2304) < 2.0 ** -16
    # a whole 16-channel k-block of hi x hi products left out stays far above the allowance at the deepest layer
    assert 1 / (2304 / 16) > 100 * CC.split_slack(2304)


def test_tile_numbering():
    tl = TILINGS["conv_row"]
    # item = (n * strips + strip) * segments + segment; 2 strips x 2 segments per image
    assert [tl.tile(1, 16, 128), tl.tile(0, 16, 0), tl.tile(0, 0, 128)] == [7, 1, 2]
    tl = TILINGS["conv_tc2"]
    assert tl.tile(1, 0, 0) == tl.tiles_per_image == 32 and tl.tile(0, 0, 8) == 1
    assert tl.owner(1, 5, 17, 20) == (34, 1, 4)


@pytest.mark.parametrize("kind", list(TILINGS))
def test_stale_stage_is_flagged_at_its_tile(case, kind):
    """tile t holds its neighbour's values: the stage of the previous tile was read again"""
    _, _, _, ref, S, good = case
    tl = TILINGS[kind]
    for t in (1, tl.tiles_per_image + 3):
        got = good.clone()
        n, ys, xs = _region(tl, t)
        m, ys0, xs0 = _region(tl, t - 1)
        got[n, :, ys, xs] = good[m, :, ys0, xs0]
        rep = _check(got, ref, S, tl)
        assert _flagged_tiles(rep) == [t], (kind, t, CC.describe(rep))
        assert rep["owner"][0] == t and rep["owner"][2] == (t % tl.grid if tl.grid else t)


@pytest.mark.parametrize("kind", list(TILINGS))
def test_missing_k_block_or_tap_is_flagged_at_its_tile(case, kind):
    x, w, b, ref, S, good = case
    tl = TILINGS[kind]
    t = 5
    n, ys, xs = _region(tl, t)
    variants = []
    for kb in range(CIN // 16):                   # one 16-channel k-block of the input never accumulated
        xk = x[n:n + 1].clone()
        xk[:, kb * 16:(kb + 1) * 16] = 0
        variants.append(("k-block %d" % kb, xk, w))
    for tap in (0, 4, 8):                         # one of the nine taps skipped
        wt = w.clone()
        wt[:, :, tap // 3, tap % 3] = 0
        variants.append(("tap %d" % tap, x[n:n + 1], wt))
    for what, xv, wv in variants:
        wrong, _ = CC.reference(xv, wv, b)
        got = good.clone()
        got[n, :, ys, xs] = _r16(wrong[0, :, ys, xs])
        rep = _check(got, ref, S, tl)
        assert _flagged_tiles(rep) == [t], (kind, what, CC.describe(rep))


@pytest.mark.parametrize("kind", list(TILINGS))
def test_zeroed_channel_group_is_flagged_at_its_tile(case, kind):
    _, _, _, ref, S, good = case
    tl = TILINGS[kind]
    t, c0 = 6, 24                                 # channels 24 .. 31: one 8-channel store group
    n, ys, xs = _region(tl, t)
    got = good.clone()
    got[n, c0:c0 + 8, ys, xs] = 0
    rep = _check(got, ref, S, tl)
    assert rep["tiles"] == [(t, c0 // tl.nt)], (kind, CC.describe(rep))
    assert rep["first"][3] >= c0


def test_unwritten_tile_fails(case):
    _, _, _, ref, S, good = case
    tl = TILINGS["conv_tc2"]
    got = good.clone()
    n, ys, xs = _region(tl, 9)
    got[n, :, ys, xs] = float("nan")
    rep = _check(got, ref, S, tl)
    assert _flagged_tiles(rep) == [9] and rep["worst"] == float("inf")


@pytest.mark.parametrize("sign", [-1, 1])
def test_split_k_chunk_left_out_or_doubled_is_flagged(sign):
    """dw with one 16 x 8 pixel chunk left out (sign -1) or added twice (+1) in one output tile of the split-K kernel"""
    g = torch.Generator().manual_seed(7)
    n_, h, w_, cin, cout = 2, 32, 64, 32, 32
    scale = 2.0 ** (torch.rand(cin, generator=g, dtype=torch.float64) * 8 - 4)
    x = _r16(torch.randn(n_, cin, h, w_, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1))
    dy = _r16(torch.randn(n_, cout, h, w_, generator=g, dtype=torch.float64))
    ref = CC.wgrad_reference(x, dy, 3)
    assert CC.check_wgrad(ref.float(), ref, 16, 16)["bad"] == []
    margin = CC.chunks_missing_margin(n_ * h * w_)
    assert margin > 50 * CC.WGRAD_TOL
    for cb, ib, (cn, cy, cx) in ((0, 0, (0, 0, 0)), (1, 1, (1, 16, 56)), (1, 0, (0, 16, 24))):
        mask = torch.zeros_like(dy)
        mask[cn, :, cy:cy + 16, cx:cx + 8] = 1
        part = CC.wgrad_reference(x, dy * mask, 3)
        got = ref.clone()
        blk = (slice(cb * 16, cb * 16 + 16), slice(ib * 16, ib * 16 + 16))
        got[blk] += sign * part[blk]
        rep = CC.check_wgrad(got.float(), ref, 16, 16)
        assert [(c, i) for c, i, _ in rep["bad"]] == [(cb, ib)], rep
        assert rep["bad"][0][2] > 0.2 * margin    # the chunk's size is what sqrt(128 / P) predicts, not a borderline hit


# ---------------------------------------------------------------------------------------------------- CUDA-core direct convolution
DIRECT_TILE = 16                                  # conv_direct_kernel: one CTA per 16 x 16 pixels x 16 output channels


def _direct_fp32(x, w, b):
    """conv_direct_kernel's arithmetic on the CPU: per output, one fp32 FMA per (16-channel chunk, channel, tap) in that order
    (the product of two fp32 values is exact in fp64, the sum is rounded to fp32), then the bias added in fp32"""
    N, Cin, H, W = x.shape
    Cout, _, ks, _ = w.shape
    pad = ks // 2
    xp = torch.nn.functional.pad(x.double(), (pad, pad, pad, pad))
    acc = torch.zeros(N, Cout, H, W, dtype=torch.float32)
    for c in range(Cin):
        for t in range(ks * ks):
            dy, dx = divmod(t, ks)
            acc = (acc.double() + xp[:, c:c + 1, dy:dy + H, dx:dx + W] * w[:, c, dy, dx].double().view(1, -1, 1, 1)).float()
    return acc if b is None else (acc.double() + b.double().view(1, -1, 1, 1)).float()


def test_direct_slack():
    assert CC.direct_slack(9) == 2.0 ** -20 and 10 * 2.0 ** -24 < CC.direct_slack(9)      # the image layer's 9 FMAs + bias
    for K in (9 * 16, 9 * 64, 9 * 512, 9 * 1024):
        # below one average term S / K at every depth the fp32 mode runs, the discriminator's last layer included
        assert CC.direct_slack(K) * K < 0.2, K
    assert CC.direct_slack(9 * 1024) > 5 * 2.0 ** -20


@pytest.mark.parametrize("cin,ks,hw,same_sign", [(1, 3, 64, True), (48, 3, 32, False), (32, 1, 32, False), (1024, 3, 16, False),
                                                 (1024, 3, 16, True)])
def test_direct_fp32_emulation_passes(cin, ks, hw, same_sign):
    """the kernel's own fp32 accumulation order passes the direct bound at the fp32 mode's depths, also with same-signed operands
    (partial sums growing to S: the most rounding noise)"""
    g = torch.Generator().manual_seed(cin + ks)
    scale = 2.0 ** (torch.rand(cin, generator=g, dtype=torch.float64) * 8 - 4)
    x = (torch.randn(1, cin, hw, hw, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1)).float()
    w = (torch.randn(16, cin, ks, ks, generator=g, dtype=torch.float64) / (cin * ks * ks) ** 0.5).float()
    if same_sign:
        x, w = x.abs(), w.abs()
    b = torch.randn(16, generator=g).float()
    ref, S = CC.reference(x.double(), w.double(), b.double())
    got = _direct_fp32(x, w, b)
    rep = CC.check_output(got, ref, S, CC.direct_u(torch.float32), CC.direct_slack(cin * ks * ks),
                          CC.Tiling(hw, hw, DIRECT_TILE, DIRECT_TILE, 16))
    print(f"K = {cin * ks * ks}{' same-signed' if same_sign else ''}: worst error / bound {rep['worst']:.3g}")
    assert rep["bad"] == 0, CC.describe(rep)


DN, DH, DW, DC0, DC1, DCOUT = 2, 32, 64, 16, 32, 32
DTILING = CC.Tiling(DH, DW, DIRECT_TILE, DIRECT_TILE, 16)


@pytest.fixture(scope="module")
def direct_case():
    """a two-source fp32 forward (torch.cat([x0, x1], 1)) and its correctly rounded fp32 output"""
    g = torch.Generator().manual_seed(11)
    cin = DC0 + DC1
    scale = 2.0 ** (torch.rand(cin, generator=g, dtype=torch.float64) * 8 - 4)
    x = (torch.randn(DN, cin, DH, DW, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1)).float().double()
    w = (torch.randn(DCOUT, cin, 3, 3, generator=g, dtype=torch.float64) / (cin * 9) ** 0.5).float().double()
    b = torch.randn(DCOUT, generator=g, dtype=torch.float64).float().double()
    ref, S = CC.reference(x, w, b)
    return x, w, b, ref, S, ref.float().double()


def _direct_check(got, ref, S):
    return CC.check_output(got, ref, S, CC.direct_u(torch.float32), CC.direct_slack(9 * (DC0 + DC1)), DTILING)


def test_direct_correct_output_passes(direct_case):
    _, _, _, ref, S, good = direct_case
    rep = _direct_check(good, ref, S)
    assert rep["bad"] == 0 and rep["worst"] <= 1.0, CC.describe(rep)


def _direct_wrong_tile(case, t, x_wrong):
    x, w, b, ref, S, good = case
    n, ys, xs = _region(DTILING, t)
    wrong, _ = CC.reference(x_wrong[n:n + 1], w, b)
    got = good.clone()
    got[n, :, ys, xs] = wrong[0, :, ys, xs].float().double()
    return _direct_check(got, ref, S)


def test_direct_second_source_without_offset_is_flagged_at_its_tile(direct_case):
    """src1 read at pix * C1 + c instead of pix * C1 + (c - C0): the second source's channels come out shifted by C0 elements"""
    x = direct_case[0]
    flat = x[:, DC0:].permute(0, 2, 3, 1).reshape(-1)
    idx = torch.arange(flat.numel()).view(DN, DH, DW, DC1) + DC0
    x1 = torch.where(idx < flat.numel(), flat[idx.clamp_max(flat.numel() - 1)], torch.zeros((), dtype=flat.dtype))
    xw = x.clone()
    xw[:, DC0:] = x1.permute(0, 3, 1, 2)
    for t in (3, DTILING.tiles_per_image + 5):
        rep = _direct_wrong_tile(direct_case, t, xw)
        assert _flagged_tiles(rep) == [t], (t, CC.describe(rep))


@pytest.mark.parametrize("chunk", range((DC0 + DC1) // 16))
def test_direct_dropped_input_chunk_is_flagged_at_its_tile(direct_case, chunk):
    xw = direct_case[0].clone()
    xw[:, chunk * 16:(chunk + 1) * 16] = 0
    t = 6
    rep = _direct_wrong_tile(direct_case, t, xw)
    assert _flagged_tiles(rep) == [t], (chunk, CC.describe(rep))


def test_direct_second_pixel_row_written_to_the_first_is_flagged_at_its_tile(direct_case):
    """each thread owns rows py and py + 8 of its tile; row py + 8's values stored at row py leave rows 8 .. 15 unwritten"""
    _, _, _, ref, S, good = direct_case
    for t in (0, 9):
        n, y0, x0 = _origin(DTILING, t)
        got = good.clone()
        got[n, :, y0:y0 + 8, x0:x0 + 16] = good[n, :, y0 + 8:y0 + 16, x0:x0 + 16]
        got[n, :, y0 + 8:y0 + 16, x0:x0 + 16] = float("nan")
        rep = _direct_check(got, ref, S)
        assert _flagged_tiles(rep) == [t] and rep["worst"] == float("inf"), (t, CC.describe(rep))
        assert rep["first"][1] == y0, rep


def _wgrad_direct_case():
    g = torch.Generator().manual_seed(13)
    n_, h, w_, cin, cout = 2, 32, 64, 32, 32
    scale = 2.0 ** (torch.rand(cin, generator=g, dtype=torch.float64) * 8 - 4)
    x = (torch.randn(n_, cin, h, w_, generator=g, dtype=torch.float64) * scale.view(1, -1, 1, 1)).float().double()
    dy = torch.randn(n_, cout, h, w_, generator=g, dtype=torch.float64).float().double()
    return x, dy


def test_direct_skipped_weight_gradient_split_is_flagged_at_its_block():
    """wgrad_direct_kernel: CTA (co block, ci block, split s) sums the 8 x 16 pixel tiles t with t % splits == s; one CTA that never
    adds its split leaves those tiles out of one 16 x 16 block of dw"""
    x, dy = _wgrad_direct_case()
    n_, _, h, w_ = x.shape
    ref = CC.wgrad_reference(x, dy, 3)
    assert CC.check_wgrad(ref.float(), ref, 16, 16)["bad"] == []
    tx, ty = w_ // 16, h // 8
    ntiles, splits = n_ * tx * ty, 5                       # 32 tiles over 5 splits: a ragged last split
    tile = torch.arange(ntiles).view(n_, ty, tx).repeat_interleave(8, 1).repeat_interleave(16, 2)
    for cb, ib, s in ((0, 0, 0), (1, 0, 4), (1, 1, 2)):
        part = CC.wgrad_reference(x, dy * (tile % splits == s).unsqueeze(1).double(), 3)
        got = ref.clone()
        blk = (slice(cb * 16, cb * 16 + 16), slice(ib * 16, ib * 16 + 16))
        got[blk] -= part[blk]
        rep = CC.check_wgrad(got.float(), ref, 16, 16)
        assert [(c, i) for c, i, _ in rep["bad"]] == [(cb, ib)], rep


def test_direct_bias_gradient_added_once_per_ci_block_is_flagged():
    """dbias is added by the ci block 0 CTAs only; adding it from every ci block multiplies it by the number of ci blocks"""
    _, dy = _wgrad_direct_case()
    ref = dy.sum((0, 2, 3))
    mag = dy.abs().sum((0, 2, 3))
    good = dy.float().sum((0, 2, 3))
    assert CC.check_sums(good, ref, mag)["bad"] == []
    ci_blocks = 2
    rep = CC.check_sums(ci_blocks * good, ref, mag)
    assert rep["bad"] == list(range(dy.shape[1])), rep


def test_direct_bias_gradient_with_a_lost_split_is_flagged():
    """with a per-channel mean in dY (as the scale test draws it), leaving one split's tiles out of dbias fails every channel"""
    _, dy = _wgrad_direct_case()
    n_, c, h, w_ = dy.shape
    mean = torch.where(torch.arange(c) % 2 == 0, -2.0, 2.0).double()
    dy = dy + mean.view(1, -1, 1, 1)
    ref, mag = dy.sum((0, 2, 3)), dy.abs().sum((0, 2, 3))
    tx, ty = w_ // 16, h // 8
    tile = torch.arange(n_ * tx * ty).view(n_, ty, tx).repeat_interleave(8, 1).repeat_interleave(16, 2)
    splits = 5
    lost = (dy * (tile % splits == splits - 1).unsqueeze(1).double()).sum((0, 2, 3))
    assert CC.check_sums((ref - lost).float(), ref, mag)["bad"] == list(range(c))
    assert CC.check_sums((ref + lost).float(), ref, mag)["bad"] == list(range(c))
