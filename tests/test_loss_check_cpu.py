"""CPU self-test of tests/_loss_check.py: at small shapes, an fp32 emulation of each loss kernel passes its bound and the same
emulation with one planted fault fails it (a dropped Gated CRF tap, a halo row from the wrong tile, a lost block partial, TV's
tie rule, the UAMT Monte-Carlo row layout, truncated bf16 stores, S2L's class rule)."""
import numpy as np
import pytest
import torch

import _loss_check as L


def _logits(N, H, W, seed, sat=True):
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 ** (torch.rand(N, 1, H, W, generator=g) * 9 - 4)
    x = torch.randn(N, 4, H, W, generator=g) * scale
    if sat:
        x[:, :, : H // 4, : W // 4] = torch.tensor([200.0, -200.0, -200.0, -200.0]).view(1, 4, 1, 1)    # exact 1 / 0 plateau
    return x


def _image(N, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    lev = torch.rand(N, 1, H // 8, W // 8, generator=g)
    img = torch.nn.functional.interpolate(lev, size=(H, W), mode="nearest")              # flat regions with edges
    img[:, :, : H // 4, : W // 4] = 0.0                                                   # dark top-left corner
    return img


def test_crf_bound_passes_fp32_and_flags_a_dropped_tap_and_a_wrong_seam_row():
    N, H, W = 1, 64, 64
    y = torch.softmax(_logits(N, H, W, 1, sat=False), 1)
    img = _image(N, H, W, 2)
    loss, ksum, ref, mag, lmag = L.crf_ref(y, img)
    gscale = -2.0 / (N * H * W)
    s = L.crf_s(y, img)
    assert torch.allclose(gscale * s, ref, rtol=1e-12, atol=0)               # the tap-by-tap restatement is the autograd gradient
    bound = L.CRF_REL * mag
    good = (gscale * s).float()
    assert L.report(good.view(-1, 4), ref.view(-1, 4), bound.view(-1, 4))["bad"] == 0
    for fault in ({"drop": (5, 5)}, {"seam": (32, 32)}):
        bad = (gscale * L.crf_s(y, img, **fault)).float()
        rep = L.report(bad.view(-1, 4), ref.view(-1, 4), bound.view(-1, 4))
        assert rep["bad"] > 0, fault
        assert rep["worst"] > 50, (fault, rep["worst"])
    pair = (s * y.double()).sum().item()
    assert L.scalar((ksum - pair) / (N * H * W), loss, lmag, "crf")["bad"] == 0


def test_a_lost_block_partial_is_flagged():
    N, H, W, grid = 4, 32, 32, 7
    x = _logits(N, H, W, 3)
    lab = torch.randint(0, 5, (N, H, W), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    loss, cnt, mag = L.pce_ref(x, lab, 4)
    xs = x.float()
    nll = (torch.logsumexp(xs, 1) - xs.gather(1, lab.long().clamp(max=3).unsqueeze(1))[:, 0]) * L.labelled(lab, 4)
    quad = torch.arange(N * H * W) // 4
    blk = (quad // 256) % grid                                                # grid-stride: thread = quad, block = thread // 256
    parts = torch.stack([nll.reshape(-1)[blk == b].sum() for b in range(grid)]).double()
    assert L.scalar(parts.sum() / cnt, loss, mag / cnt, "pce")["bad"] == 0
    assert L.scalar(parts[1:].sum() / cnt, loss, mag / cnt, "pce")["bad"] == 1


def test_tv_routing_to_the_last_extremum_is_flagged():
    g = torch.Generator().manual_seed(5)
    p = torch.randint(0, 3, (3, 16, 16), generator=g).float() / 2                 # three levels: ties everywhere
    p[1] = torch.rand(16, 16, generator=g)
    loss, mag, ref = L.tv_ref(p, 1e-2)
    gscale = 1e-2 / p.numel()
    first = L.tv_route(p, gscale)
    assert torch.allclose(first, ref, rtol=1e-12, atol=1e-18)                  # autograd routes to the first extremum too
    b = L.tv_bound(ref, gscale)
    assert L.report(first.float().view(-1, 1), ref.view(-1, 1), b.view(-1, 1))["bad"] == 0
    assert L.report(L.tv_route(p, gscale, last=True).float().view(-1, 1), ref.view(-1, 1), b.view(-1, 1))["bad"] > 0


def test_uamt_sample_major_rows_are_flagged():
    T, B, H, W = 8, 3, 16, 16
    rows = L.mc_rows(T, B)
    assert torch.equal(rows, torch.arange(T).view(T, 1) * B + torch.arange(B).view(1, B))   # the kernel's layout is t * B + b
    mc = _logits(T * B, H, W, 6, sat=False)
    unc, band = L.uncertainty_ref(mc, T, B)
    thr = float(np.float32(unc.median().item()))
    rep, frac = L.mask_check((L.uncertainty_fp32(mc, T, B) < thr).to(torch.uint8), unc, band, thr)
    assert rep["bad"] == 0 and frac < 0.01
    rep, _ = L.mask_check((L.uncertainty_fp32(mc, T, B, "sample_major") < thr).to(torch.uint8), unc, band, thr)
    assert rep["bad"] > 0


@pytest.mark.parametrize("dt", [0, 2])
def test_truncated_16bit_stores_are_flagged(dt):
    N, H, W = 2, 16, 16
    x = _logits(N, H, W, 7)
    p = torch.softmax(x, 1)
    lab = torch.randint(0, 5, (N, H, W), generator=torch.Generator().manual_seed(8), dtype=torch.uint8)
    gp = torch.randn(N, 4, H, W, generator=torch.Generator().manual_seed(9))
    cnt = int(L.labelled(lab, 4).sum())
    S = 1024.0 if dt == 2 else 1.0
    ref, mag = L.head_bwd_ref(p, lab, 4, S, cnt, gp, 0.1 * S)
    d = ref.float()
    for trunc, fails in ((False, False), (True, True)):
        d16 = torch.zeros(N, H, W, 16, dtype=L.TORCH_T[dt])
        d16[..., :4] = L.round16(d.permute(0, 2, 3, 1), dt, truncate=trunc)
        reps = L.check_nhwc16(d16, ref, mag, dt, "nhwc16")
        assert (sum(r["bad"] for r in reps) > 0) == fails
    d16[..., 7] = 1.0
    assert L.check_nhwc16(d16, ref, mag, dt, "nhwc16")[1]["bad"] == N * H * W


def test_s2l_first_class_wins_is_flagged():
    N, H, W, thr = 2, 16, 16, 0.8
    g = torch.Generator().manual_seed(10)
    weight = torch.rand(N, H, W, 4, generator=g)
    weight[0, 0, :4, :] = float(np.float32(thr))                                     # exactly at thr_conf: not a u-label (strict >)
    scr = torch.where(torch.rand(N, H, W, generator=g) < 0.2, torch.randint(0, 4, (N, H, W), generator=g), 4).to(torch.uint8)
    r = L.s2l_ref(_logits(N, H, W, 11), scr, weight, thr, 0.5)
    assert int((r["ulab"][0, 0, :4] != 4).sum()) == 0
    assert L.exact(r["ulab"].view(-1, 1), r["ulab"].view(-1, 1))["bad"] == 0
    assert L.exact(L.u_labels_first_wins(weight, scr, thr).view(-1, 1), r["ulab"].view(-1, 1), (N, H, W))["bad"] > 0


def test_documented_divergences():
    """class variance: where a class's std is 0, torch.std's backward leaves the intra term out (finite gradient), as the kernel
    does; pCE of no labelled pixel is NaN with a zero CE gradient"""
    N, H, W = 2, 16, 16
    x = _logits(N, H, W, 12, sat=False)
    x[0, 3] = -300.0
    p = torch.softmax(x, 1)
    img = _image(N, H, W, 13) + 0.1
    r = L.variance_ref(img, p, 1.0)
    assert bool(r["zero"][0, 3]) and bool(torch.isfinite(r["grad"]).all())
    v = img.double() * p.double()                                      # sample 0, class 3: only the inter term remains
    mean, mbar, sdn = r["mean"][0], r["mean"][0].mean(), r["sdn"][0]
    inter = (mean[3] - mbar) / (3 * sdn * v[0, 3].numel() * N) * img.double()[0, 0]
    assert torch.allclose(r["grad"][0, 3], inter, rtol=1e-9, atol=1e-15)
    lab = torch.full((N, H, W), 4, dtype=torch.uint8)
    loss, cnt, _ = L.pce_ref(x, lab, 4)
    assert cnt == 0 and loss != loss
    ref, _ = L.head_bwd_ref(p, lab, 4, 1.0, cnt, None, 0.0)
    assert torch.equal(ref, torch.zeros_like(ref))
