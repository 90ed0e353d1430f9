"""CPU self-test of tests/_netop_check.py: the counter-RNG restatement reproduces the published SplitMix64 vectors and agrees with
a big-integer form, and the bounds flag the usual kernel mistakes at the right (n, y, x, c) / channel.  Every "kernel" here is an
fp32 emulation on the CPU, correct or with one planted fault."""
import numpy as np
import pytest
import torch

import _netop_check as K

SEED = 0x5DEECE66D


def test_splitmix64_matches_the_published_vectors():
    assert K.splitmix64_int(K.GOLDEN) == 0xE220A8397B1DCDAF
    assert int(K.splitmix64(np.uint64(K.GOLDEN))) == 0xE220A8397B1DCDAF
    state, outs = 1234567, []
    for _ in range(3):
        state = (state + K.GOLDEN) & K.M64
        outs.append(K.splitmix64_int(state))
    assert outs == [6457827717110365317, 3203168211198807973, 9817491932198370423]


def test_vectorised_rng_equals_the_big_int_form():
    seed = 0xFFFFFFFFFFFFFFF0 + 7          # seed + vec * golden wraps
    vec = np.array([0, 1, 2, 12345, 0xFFFFFFFF], dtype=np.uint64)
    got = K.rand8x16(seed, vec)
    for i, v in enumerate(vec.tolist()):
        a = K.splitmix64_int(seed + v * K.GOLDEN)
        b = K.splitmix64_int(a + 0xD1B54A32D192ED03)
        want = [(a >> (16 * j)) & 0xFFFF for j in range(4)] + [(b >> (16 * j)) & 0xFFFF for j in range(4)]
        assert got[i].tolist() == want
    u = K.uniform(seed, 4)
    for i in range(4):
        x = (seed * K.GOLDEN + i) & K.M64
        x ^= x >> 33
        x = (x * 0xFF51AFD7ED558CCD) & K.M64
        x ^= x >> 33
        x = (x * 0xC4CEB9FE1A85EC53) & K.M64
        x ^= x >> 33
        assert u[i] == np.float32(((x & 0xFFFFFFFF) >> 8) / 16777216.0)
    assert K.drop_threshold(0.5) == 32768 and K.drop_threshold(0.05) == int(np.float32(0.05) * np.float32(65536))
    keep = K.keep_mask(SEED, 4096, 16, 0.3)
    assert abs(keep.mean() - 0.7) < 0.02


def _case(N=2, H=8, W=8, C=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    sig = 2.0 ** (torch.rand(C, generator=g) * 8 - 4)
    mu = sig * (torch.rand(C, generator=g) * 16 - 8)
    y = (torch.randn(N * H * W, C, generator=g) * sig + mu).to(torch.bfloat16).float()
    return y, g


def _act_fp32(y, sc, sh, slope, keep, p):
    """fp32 emulation of bn_act_fwd's element arithmetic"""
    z = torch.addcmul(sh, y, sc)                                   # fp32 (an fmaf rounds once; this rounds twice at most)
    a = torch.where(z > 0, z, z * np.float32(slope))
    return torch.where(torch.from_numpy(keep), a * np.float32(K.inv_keep(p)), torch.zeros_like(a))


def _ss(y, g):
    m = y.double().mean(0)
    inv = 1.0 / (y.double().var(0, unbiased=False) + 1e-5).sqrt()
    gamma = 0.5 + torch.rand(y.shape[1], generator=g)
    beta = 0.4 * torch.rand(y.shape[1], generator=g) - 0.2
    sc = (gamma * inv.float()).float()
    sh = (beta - m.float() * sc).float()
    return sc, sh, m.float(), inv.float()


def test_act_bound_passes_fp32_arithmetic_and_flags_a_shifted_dropout_vector():
    N, H, W, C, p = 2, 8, 8, 16, 0.3
    y, g = _case(N, H, W, C)
    sc, sh, _, _ = _ss(y, g)
    keep = K.keep_mask(SEED, N * H * W, C, p)
    ref = K.act_ref(y, sc, sh, 0.01, torch.from_numpy(keep), p)
    good = _act_fp32(y, sc, sh, 0.01, keep, p).to(torch.bfloat16)
    assert K.report(good, ref, K.act_bound(ref, 0), (N, H, W))["bad"] == 0
    shifted = K.keep_mask(SEED, N * H * W, C, p, vec_offset=1)     # vector index off by one
    bad = _act_fp32(y, sc, sh, 0.01, shifted, p).to(torch.bfloat16)
    lay = K.Layout("rows", C, 3)
    rep = K.report(bad, ref, K.act_bound(ref, 0), (N, H, W), lay)
    assert rep["bad"] > 0
    n, yy, xx, c0 = rep["first"]
    p0 = rep["p"]
    assert keep[p0, c0] != shifted[p0, c0]                           # the first flagged element is a flipped keep bit
    assert f"block {lay.block(p0, c0)}" in rep["msg"]


def test_swapped_channel_groups_are_flagged_in_the_first_group():
    N, H, W, C = 2, 8, 8, 16
    y, g = _case(N, H, W, C, 1)
    sc, sh, _, _ = _ss(y, g)
    keep = np.ones((N * H * W, C), dtype=bool)
    ref = K.act_ref(y, sc, sh, 0.01, torch.from_numpy(keep), 0.0)
    out = _act_fp32(y, sc, sh, 0.01, keep, 0.0)
    out = torch.cat([out[:, 8:], out[:, :8]], 1).to(torch.bfloat16)
    rep = K.report(out, ref, K.act_bound(ref, 0), (N, H, W))
    assert rep["bad"] > 0 and "(n, y, x, c) = (0, 0, 0, " in rep["msg"] and "8-channel group 0" in rep["msg"]


def test_pool_index_on_the_second_of_two_tied_maxima_is_flagged():
    N, H, W, C = 2, 4, 4, 16
    act = torch.randn(N, H, W, C).to(torch.bfloat16)
    act[1, 2, 0, 11] = act[1, 3, 0, 11] = 7.0          # window (n=1, yp=1, xp=0): elements k = 0 and k = 2 tie
    pooled, idx, ties = K.pool_ref(act)
    assert ties >= 1 and idx[1, 1, 0, 11].item() == 0 and pooled[1, 1, 0, 11].item() == 7.0
    wrong = idx.clone()
    wrong[1, 1, 0, 11] = 2
    rep = K.exact(wrong, idx, (N, H // 2, W // 2), what="pool_idx")
    assert rep["bad"] == 1 and "(n, y, x, c) = (1, 1, 0, 11)" in rep["msg"]


def test_a_missing_block_partial_is_flagged():
    N, H, W, C, grid = 4, 16, 16, 16, 7
    y, g = _case(N, H, W, C, 2)
    P = N * H * W
    lay = K.Layout("rows", C, grid)
    blk = torch.tensor([lay.block(p, 0) for p in range(P)])
    parts = torch.stack([torch.stack([y[blk == b].sum(0), (y[blk == b] ** 2).sum(0)]) for b in range(grid)])   # fp32 rows
    s, a, sq = K.stats_ref(y)
    full = parts.double().sum(0)
    assert K.sums(full[0], s, a)["bad"] == 0 and K.sums(full[1], sq, sq)["bad"] == 0
    short = parts[torch.arange(grid) != 5].double().sum(0)         # block 5's row left out
    assert K.sums(short[0], s, a)["bad"] > 0 and K.sums(short[1], sq, sq)["bad"] == C
    mean, var = short[0] / P, short[1] / P - (short[0] / P) ** 2
    rep, _, _ = K.check_mean_invstd(mean, 1 / (var + 1e-5).sqrt(), s, sq, P, 1e-5)
    assert rep["bad"] == 1


def _bwd_case(N=4, H=8, W=8, C=16, p=0.2, seed=3):
    y, g = _case(N, H, W, C, seed)
    sc, sh, mean, inv = _ss(y, g)
    gs = 2.0 ** (torch.rand(C, generator=g) * 8 - 4)
    g0 = (torch.randn(N * H * W, C, generator=g) * gs).to(torch.bfloat16).double()
    keep = torch.from_numpy(K.keep_mask(SEED, N * H * W, C, p))
    return y, sc, sh, mean, inv, g0, keep


def test_ignored_accumulate_is_flagged():
    N, H, W, C, p = 4, 8, 8, 16, 0.2
    y, sc, sh, mean, inv, g0, keep = _bwd_case(N, H, W, C, p)
    r = K.bn_bwd_ref(y, sc, sh, mean, inv, g0, g0.abs(), keep, p, 0.01, N * H * W)
    once = r["dgamma"].float()                            # a second call that overwrote instead of adding
    assert K.sums(2 * once, 2 * r["dgamma"], 2 * r["dgamma_mag"])["bad"] == 0
    assert K.sums(once, 2 * r["dgamma"], 2 * r["dgamma_mag"])["bad"] > 0


def test_per_sample_scale_from_the_neighbouring_image_is_flagged():
    N, H, W, C = 3, 4, 4, 16
    a = torch.randn(N, H, W, C).to(torch.bfloat16)
    cs = torch.rand(N, C) * 2
    ref = (a.float() * cs.view(N, 1, 1, C)).to(torch.bfloat16)
    bad = (a.float() * cs.roll(-1, 0).view(N, 1, 1, C)).to(torch.bfloat16)
    assert K.exact(ref, ref)["bad"] == 0
    rep = K.exact(bad.view(-1, C), ref.view(-1, C), (N, H, W), K.Layout("vec", C, 5), what="chan_scale")
    assert rep["bad"] > 0 and "(n, y, x, c) = (0, 0, 0, 0)" in rep["msg"]


def test_sync_coefficients_from_the_local_pixel_count_are_flagged():
    N, H, W, C, p = 4, 8, 8, 16, 0.2
    y, sc, sh, mean, inv, g0, keep = _bwd_case(N, H, W, C, p, seed=5)
    P = N * H * W
    r = K.bn_bwd_ref(y, sc, sh, mean, inv, g0, g0.abs(), keep, p, 0.01, P)
    ref, bound = K.dy_ref(r, sc, mean, inv, P, 0)
    half = P // 2                                          # two ranks; rank 0 forms c1, c2 from the global sums over its own P
    good = sc.double() * (r["dz"] - r["dbeta"] / P - r["xhat"] * (r["dgamma"] / P))
    assert K.report(good[:half].to(torch.bfloat16), ref[:half], bound[:half], (N // 2, H, W))["bad"] == 0
    local = sc.double() * (r["dz"] - r["dbeta"] / half - r["xhat"] * (r["dgamma"] / half))
    rep = K.report(local[:half].to(torch.bfloat16), ref[:half], bound[:half], (N // 2, H, W))
    assert rep["bad"] > 0


@pytest.mark.parametrize("dt", [0, 2])
def test_dy_bound_accepts_fp32_evaluation(dt):
    N, H, W, C, p = 4, 8, 8, 16, 0.1
    y, sc, sh, mean, inv, g0, keep = _bwd_case(N, H, W, C, p, seed=7)
    P = N * H * W
    r = K.bn_bwd_ref(y, sc, sh, mean, inv, g0, g0.abs(), keep, p, 0.01, P)
    ref, bound = K.dy_ref(r, sc, mean, inv, P, dt)
    c1, c2 = (r["dbeta"] / P).float(), (r["dgamma"] / P).float()
    B = (-sc.double() * c2.double() * inv.double()).float()
    D = (-sc.double() * c1.double() + sc.double() * c2.double() * mean.double() * inv.double()).float()
    got = (r["dz"].float() * sc + (y * B + D)).to(K.TORCH_T[dt])
    assert K.report(got, ref, bound, (N, H, W))["bad"] == 0
