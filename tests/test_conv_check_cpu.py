"""The checker of tests/test_gpu_conv_at_scale.py, on the CPU: correctly rounded fp64 convolutions pass, and the mistakes a
pipelined tensor-core kernel makes when a CTA walks several tiles (a stale stage, a missing k-block or tap, a zeroed channel
group, a split-K chunk left out of the weight gradient) are flagged at the tile that holds them."""
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
