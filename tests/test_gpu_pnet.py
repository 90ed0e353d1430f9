"""PNet2D (SURVEY 8(f) rank 4; reference networks/pnet.py, net_factory.py:18-19) on the planned executor: dilated 3x3 blocks on the per-tap
wgmma kernel, concat + 1x1 heads, Dropout2d -- against the fixture generated from the unmodified reference class."""
import os

import numpy as np
import pytest
import torch

import wsl_oracle as O
from _gpu_util import cosine

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200 import functional as Fn
    from wsl4mis_b200.networks.net_factory import net_factory
    from wsl4mis_b200.networks.pnet import PNet2D


def _case(golden_dir, precision):
    g = np.load(os.path.join(golden_dir, "pnet.npz"))
    n = int(g["n"])
    p = O.pnet_synth_params(1, 4, int(g["pseed"]))
    m = PNet2D(1, 4, 64, [1, 2, 4, 8, 16])
    m.load_state_dict(p)
    m = m.to(DEV).set_precision(precision)
    rs = np.random.RandomState(int(g["cseed"]))
    keeps = [torch.from_numpy((rs.uniform(size=(n, c)) >= 0.3).astype(np.uint8)) for c in (128, 64)]
    m.channel_keep = [k.to(DEV) for k in keeps]
    return g, p, m, keeps


def test_pnet_fp16x3_matches_the_reference_fixture(golden_dir):
    g, p, m, _ = _case(golden_dir, "fp16x3")
    x, lab = torch.from_numpy(g["image"]).to(DEV), torch.from_numpy(g["label"]).to(DEV)
    m.eval()
    with torch.no_grad():
        ev = m(x)
    ref = torch.from_numpy(g["eval"])
    assert (ev.cpu() - ref).abs().max().item() < 1e-3 * ref.abs().max().item()
    m.train()
    o = m(x)
    ref = torch.from_numpy(g["train"])
    err = (o.detach().cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-3, err
    assert torch.equal(o.detach().cpu().argmax(1), ref.argmax(1))
    loss, _ = Fn.softmax_pce(o, lab)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - float(g["loss"])) < 1e-4 * abs(float(g["loss"]))
    named = dict(m.named_parameters())
    errs = {}
    for k, (_, asum, l2) in zip([str(k) for k in g["grad_keys"]], g["grad_stats"]):
        if k.startswith("block") and k.endswith(".bias") and ".conv" in k:
            continue                      # conv bias in front of BatchNorm: true gradient 0 (the reference holds rounding noise)
        assert named[k].grad is not None, k
        errs[k] = abs(named[k].grad.double().norm().item() - l2) / (l2 + 1e-12)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print(f"[pnet fp16x3] logits {err:.2e} of scale; worst gradient-norm errors:", [(k, f"{v:.2e}") for k, v in worst])
    bad = {k: v for k, v in errs.items() if v > (2e-3 if named[k].dim() == 4 else 1e-2)}
    assert not bad, bad


def test_pnet_bf16_matches_the_storage_emulating_oracle(golden_dir):
    g, p, m, keeps = _case(golden_dir, "bf16")
    x = torch.from_numpy(g["image"])
    m.train()
    o = m(x.to(DEV))
    loss, _ = Fn.softmax_pce(o, torch.from_numpy(g["label"]).to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    O.QUANT = True
    try:
        leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
        q = O.pnet2d_forward(leaves, x, True, keeps)
        lq = O.pce_loss(q, torch.from_numpy(g["label"]))
        ks = [k for k, v in leaves.items() if v.requires_grad]
        gq = dict(zip(ks, torch.autograd.grad(lq, [leaves[k] for k in ks])))
    finally:
        O.QUANT = None
    err = (o.detach().float().cpu() - q.detach()).abs().max().item() / q.detach().abs().max().item()
    named = dict(m.named_parameters())
    worst = min(cosine(named[k].grad.detach().cpu(), v) for k, v in gq.items() if named[k].dim() == 4)
    print(f"[pnet bf16] logits vs the bf16-emulating oracle {err:.3f} of scale, worst conv-weight gradient cosine {worst:.4f}")
    assert err < 0.06 and worst > 0.9


def test_net_factory_pnet_trains():
    torch.manual_seed(1)
    m = net_factory("pnet", in_chns=1, class_num=4)
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    img, lab = O.synth_batch(4, 64, 64, seed=2, frac=0.1)
    img, lab = img.to(DEV), lab.to(DEV)
    m.train()
    hist = []
    for _ in range(8):
        loss = torch.nn.CrossEntropyLoss(ignore_index=4)(m(img), lab.long())
        opt.zero_grad()
        loss.backward()
        opt.step()
        hist.append(loss.item())
    assert hist[-1] < hist[0], hist


def test_pnet_step_time_at_256():
    """eager module API (forward + CrossEntropy + backward + SGD) at 16 x 256 x 256, bf16 tensor-core mode: a reported number"""
    torch.manual_seed(3)
    m = net_factory("pnet", in_chns=1, class_num=4)
    opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    img, lab = O.synth_batch(16, 256, 256, seed=4, frac=0.05)
    img, lab = img.to(DEV), lab.to(DEV).long()
    ce = torch.nn.CrossEntropyLoss(ignore_index=4)
    m.train()

    def step():
        loss = ce(m(img), lab)
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss
    for _ in range(3):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(10):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print(f"[pnet bf16] 16x256x256 eager step {ms:.2f} ms = {16e3 / ms:.0f} img/s, loss {loss.item():.4f}")
    assert torch.isfinite(loss)
