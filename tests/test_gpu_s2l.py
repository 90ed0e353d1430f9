"""Scribble2Label (code/train_s2l.py, code/dataloaders/dataset_s2l.py) on the fused path: the batch transform of the image, scribble
and prediction memory, the u-label / two-term CE head, the per-sample BatchNorm forward, the batched ensemble refresh, the whole
step against the CPU oracle (s2l_oracle.py), graph == eager, the epoch-snapshot visibility of the memory, and the reference's
unchanged train_s2l.py."""
import os
import random

import numpy as np
import pytest
import torch
from scipy.ndimage import zoom

import s2l_oracle as S
import wsl_oracle as O
from _gpu_util import ENC_MASK_KEYS, cosine, elem_masks_nchw

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    from wsl4mis_b200._lib import call, workspace
    from wsl4mis_b200.dataloaders.dataset import RandomGenerator, S2LLoader, SliceStore
    from wsl4mis_b200.engine import S2LStep
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT


def _slices(n, seed, shapes=((40, 36), (36, 44), (50, 30), (33, 47), (44, 44))):
    rs = np.random.RandomState(seed)
    ims, masks, scrs = [], [], []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        ims.append(rs.rand(h, w).astype(np.float32))
        masks.append(rs.randint(0, 4, (h, w)).astype(np.uint8))
        scrs.append(np.where(rs.rand(h, w) < 0.3, masks[-1], 4).astype(np.uint8))
    return ims, masks, scrs


def _store_with_memory(ims, masks, scrs, seed):
    store = SliceStore.from_arrays(ims, masks, device=DEV, scribbles=scrs)
    rs = np.random.RandomState(seed)
    mems = [rs.rand(*m.shape, 4).astype(np.float32) for m in masks]
    for i, m in enumerate(mems):
        store.weight(i).copy_(torch.from_numpy(m))
    return store, mems


# ---------------------------------------------------------------- augmentation
def test_augment_matches_reference_fixture(golden_dir):
    """the reference's own RandomGenerator_s2l output (tests/golden/s2l_augment.npz) == SliceStore.augment_s2l, bit for bit"""
    z = np.load(os.path.join(golden_dir, "s2l_augment.npz"))
    n, seed, hw = int(z["n"]), int(z["seed"]), tuple(int(v) for v in z["out_hw"])
    store = SliceStore.from_arrays([z[f"in{i}_image"] for i in range(n)], [z[f"in{i}_mask"] for i in range(n)], device=DEV,
                                   scribbles=[z[f"in{i}_scribble"] for i in range(n)])
    for i in range(n):
        store.weight(i).copy_(torch.from_numpy(z[f"in{i}_weight"]))
    params = []
    for i in range(n):
        random.seed(seed + i)
        np.random.seed(seed + i)
        params.append(RandomGenerator.draw(False))
    assert {p[0] for p in params} == {0, 1, 2}
    img, scr, wgt = store.augment_s2l(list(range(n)), params, hw, which="live")
    for i in range(n):
        assert np.array_equal(img[i, 0].cpu().numpy(), z[f"out{i}_image"][0]), i
        assert np.array_equal(scr[i].cpu().numpy(), z[f"out{i}_scribble"]), i
        assert np.array_equal(wgt[i].cpu().numpy(), z[f"out{i}_weight"]), i


def test_augment_every_decision_matches_oracle():
    """every rot90 count x flip axis and every angle in [-20, 20), on ragged slices, against the scipy restatement"""
    ims, masks, scrs = _slices(5, 3)
    store, mems = _store_with_memory(ims, masks, scrs, 4)
    decisions = [(0, 0, 0, 0, 0)] + [(1, k, a, 0, 0) for k in range(4) for a in range(2)] + [(2, 0, 0, ang, 0) for ang in range(-20, 20)]
    out_hw = (64, 48)
    idx = [d % len(ims) for d in range(len(decisions))]
    img, scr, wgt = store.augment_s2l(idx, decisions, out_hw, which="live")
    img, scr, wgt = img.cpu().numpy(), scr.cpu().numpy(), wgt.cpu().numpy()

    for b, (i, d) in enumerate(zip(idx, decisions)):
        mode, k, axis, ang, _ = d
        # feed the oracle's random.random / np.random.randint calls with this decision
        rnd = [0.9] if mode == 1 else ([0.1, 0.9] if mode == 2 else [0.1, 0.1])
        ints = [k, axis] if mode == 1 else ([ang] if mode == 2 else [])
        r_saved, n_saved = random.random, np.random.randint
        random.random = lambda: rnd.pop(0)
        np.random.randint = lambda lo, hi=None: ints.pop(0)
        try:
            oi, _, os_, ow = S.transform(ims[i], masks[i], scrs[i], mems[i], out_hw)
        finally:
            random.random, np.random.randint = r_saved, n_saved
        assert np.array_equal(img[b, 0], oi), d
        assert np.array_equal(scr[b], os_), d
        assert np.array_equal(wgt[b], ow), d


# ---------------------------------------------------------------- loss head
def _head_inputs(seed, n=2, hw=32):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, 4, hw, hw, generator=g) * 3
    scr = torch.full((n, hw, hw), 4, dtype=torch.uint8)
    lab = torch.rand(n, hw, hw, generator=g) < 0.1
    scr[lab] = torch.randint(0, 4, (int(lab.sum()),), generator=g, dtype=torch.uint8)
    weight = torch.rand(n, hw, hw, 4, generator=g)
    weight[:, ::3, ::5, 1] = 0.8                 # exactly at thr_conf (fp32): not above it
    return logits, scr, weight


def _run_head(logits, scr, weight, thr, w_u):
    n, _, h, w = logits.shape
    ctrl = torch.tensor([thr, w_u], dtype=torch.float32, device=DEV)
    probs = torch.empty(n, 4, h, w, device=DEV)
    ulab = torch.empty(n, h, w, dtype=torch.uint8, device=DEV)
    st = torch.empty(5, device=DEV)
    call("wsl_s2l_fwd", logits.to(DEV), scr.to(DEV), weight.to(DEV).contiguous(), ctrl, n, 4, h, w, probs, ulab, st, workspace("t_s2l", DEV))
    d = torch.empty(n, 4, h, w, device=DEV)
    call("wsl_s2l_head_bwd", probs, scr.to(DEV), ulab, st, ctrl, 1.0, n, 4, h, w, d, None, 1)
    torch.cuda.synchronize()
    return st.cpu(), ulab.cpu(), d.cpu()


@pytest.mark.parametrize("thr", [0.8, 0.3])
def test_u_labels_bit_exact(thr):
    logits, scr, weight = _head_inputs(1)
    _, ulab, _ = _run_head(logits, scr, weight, thr, 0.5)
    ref = S.u_labels(weight, scr, thr)
    assert torch.equal(ulab.long(), ref)
    if thr == 0.3:                                 # several classes qualify: the last one wins
        assert int(((weight > thr).sum(-1) > 1).sum()) > 100


@pytest.mark.parametrize("after", [False, True])
def test_losses_and_gradient_match_autograd(after):
    logits, scr, weight = _head_inputs(2)
    st, _, d = _run_head(logits, scr, weight, 0.8, 0.5 if after else 0.0)
    x = logits.clone().requires_grad_(True)
    loss, ce, lu = S.step_loss(x, scr, weight, 6000 if after else 0, 6000, 0.8)
    g, = torch.autograd.grad(loss, x)
    assert abs(st[4].item() - loss.item()) <= 2e-5 * abs(loss.item())
    assert abs(st[0].item() - ce.item()) <= 2e-5 * abs(ce.item())
    if after:
        assert abs(st[2].item() - lu.item()) <= 2e-5 * abs(lu.item())
    assert (d - g).abs().max().item() < 1e-6


def test_no_qualifying_pixel_gives_nan_loss_and_pce_gradient():
    logits, scr, weight = _head_inputs(3)
    weight.zero_()
    st, ulab, d = _run_head(logits, scr, weight, 0.8, 0.5)
    assert torch.isnan(st[4]) and torch.isnan(st[2]) and st[3].item() == 0 and int((ulab != 4).sum()) == 0
    x = logits.clone().requires_grad_(True)
    loss, _, _ = S.step_loss(x, scr, weight, 6000, 6000, 0.8)
    assert torch.isnan(loss)
    x2 = logits.clone().requires_grad_(True)
    g, = torch.autograd.grad(torch.nn.functional.cross_entropy(x2, scr.long(), ignore_index=4), x2)
    assert (d - g).abs().max().item() < 1e-6


# ---------------------------------------------------------------- per-sample BatchNorm forward
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bn_per_sample_forward_equals_batch1_forwards(precision):
    B, hw = 3, 64
    torch.manual_seed(21)
    m = UNet(1, 4)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV).set_precision(precision)
    x = torch.rand(B, 1, hw, hw, generator=torch.Generator().manual_seed(4)) * torch.tensor([1.0, 3.0, 0.5]).view(B, 1, 1, 1)
    em = elem_masks_nchw(6, B, hw, hw)
    masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    outs, _ = m.executor.forward(x.to(DEV), True, False, masks, None, bn_per_sample=True)
    got = outs[0].cpu()
    torch.cuda.synchronize()
    O.QUANT = True if precision == "bf16" else None
    try:
        ref = []
        for i in range(B):
            ns = {}
            with torch.no_grad():
                ref.append(O.unet_forward(p, x[i:i + 1], True, {k: e[i:i + 1] for k, e in zip(ENC_MASK_KEYS, em)}, ns))
            p.update(ns)
    finally:
        O.QUANT = None
    ref = torch.cat(ref)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < (1e-5 if precision == "fp32" else 0.08), err
    sd = m.state_dict()
    worst = 0.0
    for k in p:
        if "running" in k:
            a, b = sd[k].cpu().double(), p[k].double()
            worst = max(worst, ((a - b).norm() / b.norm()).item())
        elif k.endswith("num_batches_tracked"):
            assert int(sd[k]) == B, k
    # fp32 mode: the BatchNorm inputs already differ from the oracle's in the last bits of the fp32 convolutions (~1e-6)
    assert worst < (5e-6 if precision == "fp32" else 2e-2), worst
    print(f"[bn_per_sample {precision}] logits {err:.2e} of scale, running statistics {worst:.2e} rel")


# ---------------------------------------------------------------- ensemble refresh
def test_refresh_index_map_bit_exact():
    """large-margin one-hot logits: the refreshed memory (alpha = 1) is the scipy zoom-back of the class pattern, with zoom's 0 fill"""
    shapes = [(216, 256), (256, 216), (174, 208), (82, 89), (300, 120)]
    ims = [np.zeros(s, np.float32) for s in shapes]
    store = SliceStore.from_arrays(ims, [np.zeros(s, np.uint8) for s in shapes], device=DEV, scribbles=[np.zeros(s, np.uint8) for s in shapes])
    yy, xx = np.mgrid[0:256, 0:256]
    pat = ((yy * 7 + xx * 3) % 4).astype(np.int64)
    logits = torch.nn.functional.one_hot(torch.from_numpy(pat), 4).permute(2, 0, 1).float() * 60.0
    logits = logits.unsqueeze(0).repeat(len(shapes), 1, 1, 1).contiguous().to(DEV)
    tab = store.table(list(range(len(shapes))), [(0, 0, 0, 0, 0)] * len(shapes))
    call("wsl_s2l_refresh", logits, tab, len(shapes), 256, max(h * w for h, w in shapes), 1.0, 0.0, store.weight_live)
    torch.cuda.synchronize()
    onehot = np.eye(4, dtype=np.float32)[pat].transpose(2, 0, 1)
    for i, (h, w) in enumerate(shapes):
        ref = zoom(onehot, (1, h / 256, w / 256), order=0).transpose(1, 2, 0)
        got = store.weight(i).cpu().numpy()
        assert np.array_equal(got.argmax(-1), ref.argmax(-1)), (h, w)
        assert np.array_equal(got.max(-1) > 0.5, ref.max(-1) > 0.5), (h, w)      # rows / columns of zoom's fill
    assert np.array_equal(store.weight(0).cpu().numpy()[-1], np.zeros((256, 4), np.float32))  # h = 216: last row reads the fill


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
def test_refresh_matches_per_slice_loop(precision):
    n = 5
    ims, masks, scrs = _slices(n, 8, shapes=((216, 256), (256, 216), (174, 208), (232, 256), (224, 154)))
    store, mems = _store_with_memory(ims, masks, scrs, 9)
    torch.manual_seed(22)
    m = UNet(1, 4)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV).set_precision(precision)
    step = S2LStep(m, graph=False)
    em = elem_masks_nchw(10, n, 256, 256)
    step.refresh(store, alpha=0.2, chunk=2, masks={i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)})
    torch.cuda.synchronize()
    ref = S.refresh(p, ims, [mm.copy() for mm in mems], 0.2, [{k: e[i:i + 1] for k, e in zip(ENC_MASK_KEYS, em)} for i in range(n)])
    worst = max(np.abs(store.weight(i).cpu().numpy() - ref[i]).max() for i in range(n))
    assert worst < 1e-5, worst
    sd = m.state_dict()
    rs = 0.0
    for k in p:
        if "running" in k:
            a, b = sd[k].cpu().double(), p[k].double()
            rs = max(rs, ((a - b).norm() / b.norm()).item())
        elif k.endswith("num_batches_tracked"):
            assert int(sd[k]) == n, k
    assert rs < 1e-5, rs
    print(f"[refresh {precision}] memory max error {worst:.2e}, running statistics {rs:.2e} rel")


# ---------------------------------------------------------------- whole step
@pytest.mark.parametrize("after", [False, True])
def test_step_matches_oracle(after):
    n, hw = 4, 64
    torch.manual_seed(5)
    m = UNet(1, 4)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV).set_precision("fp32")
    em = elem_masks_nchw(5, n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    image, label = O.synth_batch(n, hw, hw, seed=11, frac=0.05)
    weight = torch.rand(n, hw, hw, 4, generator=torch.Generator().manual_seed(12)) ** 0.3
    step = S2LStep(m, thr_iter=6000, thr_conf=0.8, base_lr=0.01, graph=False)
    if after:
        step.iter_num = 6000
    loss = step(image.to(DEV), label.to(DEV), weight.to(DEV)).item()
    leaves = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in p.items()}
    out = O.unet_forward(leaves, image, True, {k: e for k, e in zip(ENC_MASK_KEYS, em)})
    ref, _, lu = S.step_loss(out, label, weight, step.iter_num - 1, 6000, 0.8)
    assert (lu is not None) == after and (not after or int((S.u_labels(weight, label, 0.8) != 4).sum()) > 0)
    names = [k for k, v in leaves.items() if v.requires_grad]
    grads = dict(zip(names, torch.autograd.grad(ref, [leaves[k] for k in names])))
    assert abs(loss - ref.item()) < 2e-5 * abs(ref.item()) + 1e-6, (loss, ref.item())
    # per-parameter SGD updates (the fp32 mode's weight gradients accumulate with atomics: parameters with tiny gradients carry
    # ~1e-3 relative noise), and the whole update vector
    named = dict(m.named_parameters())
    ds, rds = [], []
    for k, g in grads.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue
        delta, ref_delta = named[k].detach().cpu() - p[k], -0.01 * (g + 1e-4 * p[k])
        assert cosine(delta, ref_delta) > 0.99, k
        assert abs(delta.norm().item() - ref_delta.norm().item()) < 5e-2 * ref_delta.norm().item() + 1e-9, k
        ds.append(delta.flatten())
        rds.append(ref_delta.flatten())
    d, rd = torch.cat(ds).double(), torch.cat(rds).double()
    assert ((d - rd).norm() / rd.norm()).item() < 1e-3


def test_graph_replay_equals_eager_across_thr_iter():
    n, hw = 2, 64
    img, lab = O.synth_batch(n, hw, hw, seed=13, frac=0.05)
    weight = torch.rand(n, hw, hw, 4, generator=torch.Generator().manual_seed(14)) ** 0.3
    img, lab, weight = img.to(DEV), lab.to(DEV), weight.to(DEV)
    steps = {}
    for graph in (False, True):
        torch.manual_seed(31)
        steps[graph] = S2LStep(UNet(1, 4).to(DEV).set_precision("fp32"), thr_iter=4, graph=graph)
    e, c = steps[False], steps[True]
    for i in range(7):
        le, lc = e(img, lab, weight).item(), c(img, lab, weight).item()
        torch.cuda.synchronize()
        assert abs(le - lc) < 1e-4 * abs(le), (i, le, lc)
        for name in ("flat", "mom"):
            a, b = getattr(c, name), getattr(e, name)
            assert ((a - b).norm() / b.norm().clamp_min(1e-30)).item() < 1e-5, (i, name)
            a.copy_(b)
    assert c._graphs[0] is not None and c._w_u == 0.5


def test_rejects_two_head_models():
    with pytest.raises(ValueError):
        S2LStep(UNet_CCT(1, 4).to(DEV))
    with pytest.raises(NotImplementedError):
        S2LStep(UNet(1, 4).to(DEV), world_size=2)


# ---------------------------------------------------------------- visibility of the memory
@pytest.mark.parametrize("visibility", ["epoch", "live"])
def test_refresh_visibility(visibility):
    ims, masks, scrs = _slices(4, 15)
    store = SliceStore.from_arrays(ims, masks, device=DEV, scribbles=scrs)
    loader = S2LLoader(store, 2, output_size=(32, 32), shuffle=False, visibility=visibility)
    it = iter(loader)
    assert float(next(it)["weight"].abs().sum()) == 0.0
    store.weight_live.fill_(0.5)                      # what a refresh in mid-epoch does
    second = next(it)["weight"]
    if visibility == "epoch":
        assert float(second.abs().sum()) == 0.0
    else:
        assert float(second.max()) == 0.5
    assert float(next(iter(loader))["weight"].max()) == 0.5          # the next epoch sees it either way


# ---------------------------------------------------------------- the reference's unchanged script
def test_reference_train_s2l_runs_unchanged(tmp_path):
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    try:
        import build_ref
        import stage_s2l
        code = build_ref.extract(str(tmp_path))
        if code is not None and not stage_s2l.extract(code):
            code = None
    finally:
        sys.path.pop(0)
    if code is None:
        pytest.skip("reference scripts not staged (run __graft_entry__.build() where the reference exists)")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(root, "dropin"), root, os.path.join(root, "tests", "harness")])
    r = subprocess.run([sys.executable, "-m", "wsl4mis_b200.run", "train_s2l.py", "--root_path", "synthetic:30", "--max_iterations", "12",
                        "--thr_iter", "6", "--period_iter", "4", "--batch_size", "4"], cwd=code, env=env, capture_output=True, text=True,
                       timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "update weight end" in out, out[-3000:]
