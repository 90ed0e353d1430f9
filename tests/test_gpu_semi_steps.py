"""The mean-teacher and entropy-minimisation steps (engine.MeanTeacherStep / EntropyMinStep, train_mean_teacher_2D.py:138-180 and
train_entropy_minimization_2D.py:121-150), the partially supervised script's body on TrainStep('ce_dice'), one captured graph per
batch shape for every semi-supervised step, and the two-stream feed zip(cycle(labelled), unlabelled) of those scripts."""
import itertools
import os
import socket

import pytest
import torch
import torch.nn.functional as F

import semi_oracle as S
import wsl_oracle as O
from _gpu_util import ENC_MASK_KEYS, cosine, elem_masks_nchw, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _models(precision, seed_s=7, seed_t=8):
    from wsl4mis_b200.networks.unet import UNet
    s, t = UNet(1, 4), UNet(1, 4)
    s.load_state_dict(O.synth_params(1, 4, ("decoder",), seed_s))
    t.load_state_dict(O.synth_params(1, 4, ("decoder",), seed_t))
    return s.to(DEV).set_precision(precision), t.to(DEV).set_precision(precision)


def _inject(m, seed, B, hw):
    """fixed dropout keep masks for every training forward of `m` -> the same masks in the oracle's layout"""
    em = elem_masks_nchw(seed, B, hw, hw)
    m.dropout_masks = {i: em[i].permute(0, 2, 3, 1).contiguous().to(DEV) for i in range(5)}
    return {k: em[i].to(DEV) for i, k in enumerate(ENC_MASK_KEYS)}


def _batch(B_l, B_u, hw, seed=3):
    x, y = O.synth_batch(B_l + B_u, hw, hw, seed=seed, dense=True)
    g = torch.Generator().manual_seed(seed + 1)
    noise = torch.clamp(torch.randn(B_u, 1, hw, hw, generator=g) * 0.1, -0.2, 0.2)
    return x[:B_l].to(DEV), y[:B_l].to(DEV), x[B_l:].contiguous().to(DEV), noise.to(DEV)


def _step(method, student, teacher, **kw):
    from wsl4mis_b200.engine import EntropyMinStep, MeanTeacherStep
    return MeanTeacherStep(student, teacher, **kw) if method == "mt" else EntropyMinStep(student, **kw)


def _call(method, step, x_l, y_l, x_u, noise):
    return step(x_l, y_l, x_u, [noise]) if method == "mt" else step(x_l, y_l, x_u)


# ---- the consistency kernel's unmasked mode ------------------------------------------------------------------------------------
def test_unmasked_consistency_kernel_against_fp64():
    """T = 0: torch.mean((softmax(s) - softmax(t))^2) over B*C*H*W (train_mean_teacher_2D.py:169-170) and w times its gradient,
    at 6 x 4 x 256 x 256, with the weight from device memory and from the host argument"""
    from wsl4mis_b200._lib import call, workspace
    B, C, H, W = 6, 4, 256, 256
    g = torch.Generator().manual_seed(61)
    s, t = (torch.randn(B, C, H, W, generator=g) * 2.5).to(DEV), (torch.randn(B, C, H, W, generator=g) * 2.5).to(DEV)
    w = 0.0713
    sd = s.double().requires_grad_(True)
    ref = torch.mean((torch.softmax(sd, 1) - torch.softmax(t.double(), 1)) ** 2)
    (gref,) = torch.autograd.grad(w * ref, sd)
    out3 = torch.empty(3, device=DEV)
    call("wsl_uamt_consistency_fwd", s, t, None, 0, B, C, H, W, None, 0.0, None, out3, workspace("uamt", DEV))
    grads = []
    for wptr, wh in ((torch.tensor([w], dtype=torch.float32, device=DEV), 0.0), (None, w)):
        d = torch.full((B, C, H, W), float("nan"), device=DEV)
        call("wsl_uamt_consistency_bwd", s, t, None, out3, wptr, wh, B, C, H, W, d)
        grads.append(d)
    torch.cuda.synchronize()
    assert out3[1].item() == B * C * H * W
    assert abs(out3[2].item() - ref.item()) <= 1e-6 * ref.item(), (out3.tolist(), ref.item())
    assert abs(out3[0].item() - ref.item() * B * C * H * W) <= 1e-6 * ref.item() * B * C * H * W
    assert torch.equal(grads[0], grads[1]), "device and host weight differ"
    err = (grads[0].double() - gref).abs().max().item()
    assert err <= 1e-6 * gref.abs().max().item(), (err, gref.abs().max().item())
    # a different device weight is read at run time (what a captured graph replays)
    wptr = torch.tensor([2 * w], dtype=torch.float32, device=DEV)
    call("wsl_uamt_consistency_bwd", s, t, None, out3, wptr, 0.0, B, C, H, W, grads[1])
    torch.cuda.synchronize()
    assert (grads[1].double() - 2 * gref).abs().max().item() <= 2e-6 * gref.abs().max().item()


# ---- fp32 steps against the fp64 oracle ----------------------------------------------------------------------------------------
def _oracle_iteration(method, ps, pt, x_l, y_l, x_u, noise, masks, tmasks, iter_num):
    """one step body of the script in fp64 from the given state -> (loss, student gradients, running statistics after both
    student forwards)"""
    leaves = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v) for k, v in ps.items()}
    ns1, ns2 = {}, {}
    out_l = O.unet_forward(leaves, x_l, True, masks, ns1)
    out_u = O.unet_forward({**leaves, **ns1}, x_u, True, masks, ns2)
    if method == "mt":
        with torch.no_grad():
            ema = O.unet_forward(pt, x_u + noise, True, tmasks)
        loss = S.mt_losses(out_l, out_u, ema, y_l, iter_num)[0]
    else:
        loss = S.em_losses(out_l, out_u, y_l, iter_num)[0]
    names = [k for k, v in leaves.items() if isinstance(v, torch.Tensor) and v.requires_grad]
    grads = dict(zip(names, torch.autograd.grad(loss, [leaves[k] for k in names])))
    return loss.item(), grads, ns2


@pytest.mark.parametrize("method", ["mt", "em"])
def test_fp32_step_matches_fp64_oracle_for_three_iterations(method):
    """three consecutive fp32 steps, each checked against one fp64 oracle iteration started from the step's own state: loss,
    the gradient bucket, and the BatchNorm running statistics after the two student forwards (the DAN step's fp32 pair: its size
    and bounds)"""
    B, hw = 2, 256
    student, teacher = _models("fp32")
    masks = _inject(student, 11, B, hw)
    tmasks = _inject(teacher, 12, B, hw)
    x_l, y_l, x_u, noise = _batch(B, B, hw)
    step = _step(method, student, teacher, max_iterations=90000, graph=False)
    step.iter_num = 60000                   # iter_num // 300 = 200: the ramp weight is at its full 0.1
    pt = {k: (v.detach().double() if v.is_floating_point() else v.detach().clone()) for k, v in teacher.state_dict().items()}
    names = [k for k, _ in student.named_parameters()]
    feeds_bn = lambda k: ".conv_conv." in k and k.endswith((".0.bias", ".4.bias"))
    for it in range(3):
        ps = {k: (v.detach().double() if v.is_floating_point() else v.detach().clone()) for k, v in student.state_dict().items()}
        lr = step.lr_dev.item()
        assert lr == pytest.approx(0.01 if it == 0 else O.poly_lr(0.01, 60000 + it - 1, 90000), rel=1e-6)
        iter_num = step.iter_num
        loss = _call(method, step, x_l, y_l, x_u, noise).item()
        torch.cuda.synchronize()
        lo, grads, stats = _oracle_iteration(method, ps, pt, x_l.double(), y_l, x_u.double(), noise.double(), masks, tmasks, iter_num)
        assert step.parts["weight"] == pytest.approx(0.1)
        assert abs(loss - lo) <= 1e-5 * abs(lo), (it, loss, lo)
        gflat = step.ex.grads()[0]
        named = dict(student.named_parameters())
        view = lambda k: gflat[step.offsets[id(named[k])][0]: step.offsets[id(named[k])][0] + named[k].numel()].view_as(named[k])
        assert all(view(k).abs().max().item() == 0.0 for k in names if feeds_bn(k))
        errs = {k: rel_l2(view(k), grads[k]) for k in names if not feeds_bn(k)}
        worst = max(errs.items(), key=lambda kv: kv[1])
        bad = {k: e for k, e in errs.items() if e >= (1e-2 if it == 0 else 2e-2)}
        assert not bad, (it, bad)
        sd = student.state_dict()
        serr = max(rel_l2(sd[k], v) for k, v in stats.items())
        assert serr < 1e-4, (it, serr)
        print(f"[{method} fp32 iteration {it + 1}] loss {loss:.7f} / oracle {lo:.7f}; worst gradient {worst}; running statistics {serr:.2e}")


# ---- bf16 steps against the scripts' autograd bodies ---------------------------------------------------------------------------
def _update_check(tag, s1, s2, s0, loss, ref):
    """the UAMT step test's bf16 tolerances: loss within 3e-2, every parameter's update direction within cosine 0.85"""
    named2 = dict(s2.named_parameters())
    worst = 1.0
    for k, p in s1.named_parameters():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue                        # conv biases in front of training-mode BatchNorm: zero gradient, weight decay only
        c = cosine(p.detach() - s0[k], named2[k].detach() - s0[k])
        worst = min(worst, c)
        assert c > 0.85, (tag, k, c)
    whole = rel_l2(torch.cat([(p.detach() - s0[k]).flatten() for k, p in s1.named_parameters()]),
                   torch.cat([(named2[k].detach() - s0[k]).flatten() for k, _ in s1.named_parameters()]))
    print(f"[{tag} bf16 vs autograd] loss {loss:.7f} / {ref:.7f}; worst update cosine {worst:.5f}; whole update rel. L2 {whole:.2e}")
    assert abs(loss - ref) <= 3e-2 * abs(ref), (loss, ref)


@pytest.mark.parametrize("method", ["mt", "em"])
def test_bf16_step_matches_the_scripts_autograd_body(method):
    """one bf16 step against model(x_l), model(x_u), torch softmax / CrossEntropyLoss / DiceLoss / entropy_loss and
    torch.optim.SGD on the same modules, masks, noise and initial state"""
    from wsl4mis_b200.utils import losses
    B, hw = 2, 64
    x_l, y_l, x_u, noise = _batch(B, B, hw, seed=4)
    (s1, t1), (s2, t2) = _models("bf16"), _models("bf16")
    for s, t in ((s1, t1), (s2, t2)):
        _inject(s, 11, B, hw)
        _inject(t, 12, B, hw)
    s0 = {k: p.detach().clone() for k, p in s2.named_parameters()}
    step = _step(method, s1, t1, max_iterations=90000, graph=False)
    step.iter_num = 60000
    loss = _call(method, step, x_l, y_l, x_u, noise).item()
    opt = torch.optim.SGD(s2.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    s2.train()
    t2.train()
    outputs, outputs_unlabeled = s2(x_l), s2(x_u)
    sup = 0.5 * (losses.DiceLoss(4)(torch.softmax(outputs, 1), y_l.unsqueeze(1)) + F.cross_entropy(outputs, y_l.long()))
    if method == "mt":
        with torch.no_grad():
            ema_output = t2(x_u + noise)
        cons = torch.mean((torch.softmax(outputs_unlabeled, 1) - torch.softmax(ema_output, 1)) ** 2)
    else:
        cons = losses.entropy_loss(torch.softmax(outputs_unlabeled, 1), C=4)
    ref = sup + 0.1 * O.sigmoid_rampup(200, 200.0) * cons
    opt.zero_grad()
    ref.backward()
    opt.step()
    torch.cuda.synchronize()
    assert abs(step.parts["consistency"].item() - cons.item()) <= 3e-2 * abs(cons.item())
    _update_check(method, s1, s2, s0, loss, ref.item())


def test_partially_supervised_body_is_ce_dice():
    """train_partially_fully_supervised.py:130-142 (0.5 * (CE + Dice) on the labelled batch; the unlabelled batch is never used)
    against TrainStep(model, 'ce_dice') on the same labelled batch"""
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.utils import losses
    B, hw = 4, 64
    x_l, y_l, _, _ = _batch(B, 1, hw, seed=5)
    (s1, _), (s2, _) = _models("bf16"), _models("bf16")
    for s in (s1, s2):
        _inject(s, 13, B, hw)
    s0 = {k: p.detach().clone() for k, p in s2.named_parameters()}
    loss = TrainStep(s1, "ce_dice", graph=False)(x_l, y_l).item()
    opt = torch.optim.SGD(s2.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    s2.train()
    outputs = s2(x_l)
    ref = 0.5 * (losses.DiceLoss(4)(torch.softmax(outputs, 1), y_l.unsqueeze(1)) + torch.nn.CrossEntropyLoss()(outputs, y_l.long()))
    opt.zero_grad()
    ref.backward()
    opt.step()
    torch.cuda.synchronize()
    _update_check("partially supervised", s1, s2, s0, loss, ref.item())


# ---- one captured graph per batch shape ----------------------------------------------------------------------------------------
SHAPES = [(6, 6), (4, 6), (6, 6), (6, 3), (4, 3), (6, 6)]


def _graph_pair(method):
    """(eager step, graph step, input size, state names) built from the same seed.  256 x 256, where the default bf16 executor is
    deterministic (split-K weight gradients, fixed-order sums), as test_gpu_dan_step.py's graph test relies on"""
    from wsl4mis_b200.engine import DANStep, EntropyMinStep, MeanTeacherStep, UAMTStep
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    from wsl4mis_b200.networks.unet import UNet
    steps = []
    for graph in (False, True):
        torch.manual_seed(33)
        if method == "dan":
            steps.append(DANStep(UNet(1, 4).to(DEV), FCDiscriminator(4).to(DEV), graph=graph))
        elif method == "em":
            steps.append(EntropyMinStep(UNet(1, 4).to(DEV), graph=graph))
        else:
            cls = MeanTeacherStep if method == "mt" else UAMTStep
            steps.append(cls(UNet(1, 4).to(DEV), UNet(1, 4).to(DEV), graph=graph))
        steps[-1].iter_num = 297
    state = ("flat", "mom") + (("dflat", "exp_avg", "exp_avg_sq") if method == "dan" else ())
    return steps[0], steps[1], 256, state


@pytest.mark.parametrize("method", ["mt", "em", "uamt", "dan"])
def test_graph_per_batch_shape_equals_eager(method):
    """the batch shapes of a two-stream epoch (full, short labelled, short unlabelled, both short), three times over, from
    iteration 297 (the ramp's iter_num // 300 -- DAN's // 150 -- changes at 300): a graph step and an eager step in lockstep are
    bit-identical in loss, flat parameters and momentum at every step, and the graph step holds exactly four graphs"""
    eager, captured, hw, state = _graph_pair(method)
    x, y = O.synth_batch(12, hw, hw, seed=21, dense=True)
    x, y = x.to(DEV), y.to(DEV)
    for i, (bl, bu) in enumerate(SHAPES * 3):
        args = (x[:bl], y[:bl], x[6:6 + bu])
        le, lg = eager(*args), captured(*args)
        torch.cuda.synchronize()
        assert torch.equal(le, lg), (i, (bl, bu), le.item(), lg.item())
        for name in state:
            a, b = getattr(captured, name), getattr(eager, name)
            assert torch.equal(a, b), (i, (bl, bu), name, (a - b).abs().max().item())
    assert captured.iter_num == eager.iter_num == 297 + 3 * len(SHAPES)
    assert len(captured._graphs) == 4 and 0 in captured._graphs
    print(f"[{method} graph per shape] {len(captured._graphs)} graphs: {sorted(map(str, captured._graphs))}")


# ---- the two-stream feed -------------------------------------------------------------------------------------------------------
def test_two_stream_feed_replays_labelled_batches_within_an_epoch():
    """zip(cycle(GpuLoader(labelled, 6)), GpuLoader(unlabelled, 6)) over two epochs of synthetic:40: within an epoch the labelled
    batches after the first pass are the first pass's, bit for bit (cycle keeps them, DESIGN F19); the next epoch's cycle
    reshuffles and re-augments; an epoch is len(unlabelled loader) iterations"""
    from wsl4mis_b200.dataloaders.dataset import GpuLoader
    from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets
    torch.manual_seed(1)
    L = BaseDataSets(base_dir="synthetic:40", labeled_type="labeled", fold="fold2", split="train").to_slice_store()
    U = BaseDataSets(base_dir="synthetic:40", labeled_type="unlabeled", fold="fold2", split="train").to_slice_store()
    loader_l, loader_u = GpuLoader(L, 6), GpuLoader(U, 6)
    n_l = len(loader_l)
    assert len(loader_u) > n_l, (len(loader_u), n_l)           # the labelled stream wraps within the epoch
    firsts, shapes = [], set()
    for epoch in range(2):
        first_pass, n = [], 0
        for i, (bl, bu) in enumerate(zip(itertools.cycle(loader_l), loader_u)):
            shapes.add((bl["image"].shape[0], bu["image"].shape[0]))
            if i < n_l:
                first_pass.append(bl)
            else:
                ref = first_pass[i % n_l]
                assert torch.equal(bl["image"], ref["image"]) and torch.equal(bl["label"], ref["label"]) and bl["idx"] == ref["idx"]
            n += 1
        assert n == len(loader_u)
        firsts.append(first_pass[0])
    assert not torch.equal(firsts[0]["image"], firsts[1]["image"])
    print(f"[two-stream feed] {n_l} labelled / {len(loader_u)} unlabelled batches per epoch; batch shapes {sorted(shapes)}")


# ---- data parallel -------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ddp_worker(rank, world, port, method, out):
    import datetime
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev, timeout=datetime.timedelta(seconds=90))
    try:
        from wsl4mis_b200.engine import EntropyMinStep, MeanTeacherStep
        from wsl4mis_b200.networks.unet import UNet
        torch.manual_seed(7 + rank)         # different replicas: the construction broadcasts rank 0's student (and teacher)
        s, t = UNet(1, 4).to(dev), UNet(1, 4).to(dev)
        step = MeanTeacherStep(s, t, world_size=world) if method == "mt" else EntropyMinStep(s, world_size=world)
        x, y = O.synth_batch(8, 64, 64, seed=3, dense=True)
        lo, hi = rank * 4, rank * 4 + 2
        x_l, y_l, x_u = x[lo:hi].to(dev), y[lo:hi].to(dev), x[lo + 2:hi + 2].contiguous().to(dev)
        for _ in range(5):
            step(x_l, y_l, x_u)
        torch.cuda.synchronize()
        gathered = [torch.empty_like(step.flat) for _ in range(world)]
        dist.all_gather(gathered, step.flat)
        out[rank] = all(torch.equal(gathered[0], g) for g in gathered)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("method", ["mt", "em"])
def test_two_gpu_replicas_stay_bit_identical(method):
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    out = mp.Manager().dict()
    mp.spawn(_ddp_worker, args=(2, _free_port(), method, out), nprocs=2, join=True)
    assert out[0] and out[1]


# ---- rejections ----------------------------------------------------------------------------------------------------------------
def test_new_steps_reject_a_global_batch_mode():
    from wsl4mis_b200.engine import EntropyMinStep, MeanTeacherStep
    s, t = _models("bf16")
    with pytest.raises(NotImplementedError, match="global_batch"):
        MeanTeacherStep(s, t, global_batch=True)
    with pytest.raises(NotImplementedError, match="global_batch"):
        EntropyMinStep(s, global_batch=True)


def test_dan_graph_step_takes_short_batches_after_a_full_one():
    """DANStep(graph=True): the first batch must be full (B_u == B_l, test_gpu_dan_step.py::test_rejections); after it an epoch's
    short last unlabelled batch runs"""
    from wsl4mis_b200.engine import DANStep
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    from wsl4mis_b200.networks.unet import UNet
    torch.manual_seed(5)
    step = DANStep(UNet(1, 4).to(DEV), FCDiscriminator(4).to(DEV), graph=True)
    x, y = O.synth_batch(4, 256, 256, seed=6, dense=True)
    x, y = x.to(DEV), y.to(DEV)
    with pytest.raises(ValueError, match="B_u == B_l"):
        step(x[:2], y[:2], x[2:3])
    assert step.iter_num == 0
    for bu in (2, 1, 1, 1, 2, 2):           # each shape: two eager warm-up steps, then its graph
        assert torch.isfinite(step(x[:2], y[:2], x[2:2 + bu]))
    assert step.iter_num == 6 and len(step._graphs) == 2
