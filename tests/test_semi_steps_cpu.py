"""The mean-teacher and entropy-minimisation step bodies of the CPU oracle (semi_oracle.mt_losses / em_losses on the functional
UNet) against one step of each script on the unmodified reference modules (tests/golden/semi_steps.npz, written by
oracle/make_golden_semi.py), in fp32 and fp64.  CPU only."""
import os

import numpy as np
import pytest
import torch

import semi_oracle as S
import wsl_oracle as O

torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))


def _masks(seed, n, h, w):
    """make_golden.elem_masks: keep masks of the five encoder nn.Dropout layers from a numpy stream"""
    rs = np.random.RandomState(seed)
    names = ["encoder.in_conv.conv_conv.3"] + [f"encoder.down{i}.maxpool_conv.1.conv_conv.3" for i in range(1, 5)]
    return {nm: torch.from_numpy((rs.uniform(size=(n, O.FT[i], h >> i, w >> i)) >= O.ENC_DROP[i]).astype(np.uint8))
            for i, nm in enumerate(names)}


def _fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "semi_steps.npz"))
    B, hw, it, s_student, s_teacher, s_batch, s_noise, m_l, m_u, m_t = (int(v) for v in z["seeds"])
    x, y = O.synth_batch(2 * B, hw, hw, seed=s_batch, dense=True)
    g = torch.Generator().manual_seed(s_noise)
    noise = torch.clamp(torch.randn(B, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2)
    return z, dict(B=B, hw=hw, it=it, s_student=s_student, s_teacher=s_teacher, x_l=x[:B], y_l=y[:B], x_u=x[B:].contiguous(),
                   noise=noise, masks=[_masks(m, B, hw, hw) for m in (m_l, m_u, m_t)])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["mt", "em"])
def test_oracle_step_matches_reference_fixture(golden_dir, method, dtype):
    z, f = _fixture(golden_dir)
    p = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in O.synth_params(1, 4, ("decoder",), f["s_student"]).items()}
    leaves = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v) for k, v in p.items()}
    ns1, ns2 = {}, {}
    out_l = O.unet_forward(leaves, f["x_l"].to(dtype), True, f["masks"][0], ns1)
    out_u = O.unet_forward({**leaves, **ns1}, f["x_u"].to(dtype), True, f["masks"][1], ns2)
    if method == "mt":
        pt = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in O.synth_params(1, 4, ("decoder",), f["s_teacher"]).items()}
        with torch.no_grad():
            ema_out = O.unet_forward(pt, (f["x_u"] + f["noise"]).to(dtype), True, f["masks"][2])
        loss, sup, cons, _ = S.mt_losses(out_l, out_u, ema_out, f["y_l"], f["it"])
    else:
        loss, sup, cons, _ = S.em_losses(out_l, out_u, f["y_l"], f["it"])
    for name, v in (("loss", loss), ("supervised", sup), ("consistency", cons)):
        ref = float(z[f"{method}/{name}"])
        assert abs(v.item() - ref) <= 2e-5 * abs(ref), (name, v.item(), ref)
    keys = [str(k) for k in z[f"{method}/grad_keys"]]
    grads = torch.autograd.grad(loss, [leaves[k] for k in keys])
    for k, gr, (l2, asum) in zip(keys, grads, z[f"{method}/grad_stats"]):
        assert abs(gr.double().norm().item() - l2) <= 2e-3 * l2 + 1e-5, k      # conv biases in front of BatchNorm: ~1e-7 noise
        assert abs(gr.double().abs().sum().item() - asum) <= 2e-3 * asum + 1e-4, k
    stats = [k for k in z.files if k.startswith(f"{method}/stat/")]
    assert len(stats) == 2 * 18
    for k in stats:
        assert np.allclose(ns2[k.split("/", 2)[2]].double().numpy(), z[k], rtol=1e-4, atol=1e-5), k


@pytest.mark.parametrize("method", ["mt", "em"])
def test_losses_fp64_agree_with_fp32(method):
    g = torch.Generator().manual_seed(17)
    out_l, out_u, ema = (torch.randn(3, 4, 16, 16, generator=g, dtype=torch.float64) * 3 for _ in range(3))
    y = torch.randint(0, 4, (3, 16, 16), generator=g, dtype=torch.uint8)
    res = {}
    for dt in (torch.float32, torch.float64):
        a, b = out_l.to(dt).requires_grad_(True), out_u.to(dt).requires_grad_(True)
        r = S.mt_losses(a, b, ema.to(dt), y, 60000) if method == "mt" else S.em_losses(a, b, y, 60000)
        ga, gb = torch.autograd.grad(r[0], [a, b])
        res[dt] = (r[:3], ga, gb, r[3])
    (v32, ga32, gb32, w32), (v64, ga64, gb64, w64) = res[torch.float32], res[torch.float64]
    assert w32 == w64 == pytest.approx(0.1)
    for x32, x64 in zip(v32, v64):
        assert x32.dtype == torch.float32 and x64.dtype == torch.float64
        assert abs(x32.item() - x64.item()) <= 1e-6 * abs(x64.item())
    for x32, x64 in ((ga32, ga64), (gb32, gb64)):
        assert (x32.double() - x64).abs().max().item() <= 1e-5 * x64.abs().max().item()
