"""PNet2D (reference networks/pnet.py, net_factory.py:18-19) on the captured training steps: every TrainStep variant against the
fp64 oracle for three SGD iterations, the semi-supervised, USTM, DAN and Scribble2Label steps against their oracles composed with
`wsl_oracle.pnet2d_forward`, the per-sample (S2L refresh) forward against batch-1 training forwards, captured == eager bit for bit,
the bf16 step against the autograd module path, a census of the launches the PNet recipes make, and the trainer end to end."""
import gc
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dan_oracle as D
import s2l_oracle as S2
import semi_oracle as SO
import wsl_oracle as O
from _gpu_util import LaunchRecorder, cosine, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HW = 256
PNET_SEED = 43
KEEP_C = (128, 64)                          # channels of the output block's two Dropout2d layers

if torch.cuda.is_available():
    from wsl4mis_b200 import _lib, engine
    from wsl4mis_b200 import train as TR
    from wsl4mis_b200.networks.net_factory import net_factory
    from wsl4mis_b200.networks.pnet import PNet2D


@pytest.fixture(autouse=True)
def _release():
    """networks and executors reference each other: collect them after every test so the next one has the device's memory"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _pnet(precision, seed=PNET_SEED):
    p = O.pnet_synth_params(1, 4, seed)
    m = PNet2D(1, 4, 64, [1, 2, 4, 8, 16])
    m.load_state_dict(p)
    return m.to(DEV).set_precision(precision), p


def _keeps(n, seed):
    rs = np.random.RandomState(seed)
    return [torch.from_numpy((rs.uniform(size=(n, c)) >= 0.3).astype(np.uint8)).to(DEV) for c in KEEP_C]


def _p64(p):
    return {k: (v.to(DEV).double() if v.is_floating_point() else v.to(DEV)) for k, v in p.items()}


def _trained(p):
    return [k for k, v in p.items() if v.is_floating_point() and "running" not in k]


def _leaves(P):
    keys = set(_trained(P))
    return {k: (v.clone().requires_grad_(True) if k in keys else v) for k, v in P.items()}


def _fwd(P, x, keep):
    return O.pnet2d_forward(P, x, True, keep)


def _bucket(step, model):
    """the step's flat gradient bucket as {parameter name: gradient}"""
    gflat = step.ex.grads()[0]
    return {k: gflat[step.offsets[id(q)][0]: step.offsets[id(q)][0] + q.numel()].view_as(q) for k, q in model.named_parameters()}


def _feeds_bn(k):
    """a block convolution's bias: it feeds training-mode BatchNorm, so its true gradient is 0 (the executor leaves it at 0)"""
    return k.startswith("block") and ".conv" in k and k.endswith(".bias")


def _check_grads(step, model, grads, bound, where):
    got = _bucket(step, model)
    assert all(got[k].abs().max().item() == 0.0 for k in got if _feeds_bn(k)), where
    errs = {k: rel_l2(got[k], g) for k, g in grads.items() if not _feeds_bn(k)}
    worst = max(errs.items(), key=lambda kv: kv[1])
    assert worst[1] < bound, (where, sorted(errs.items(), key=lambda kv: -kv[1])[:4])
    return worst


# ---- 1. every TrainStep variant against fp64 ------------------------------------------------------------------------------------
def _oracle_loss(variant, logits, image, label, w_var):
    """the scripts' loss bodies (wsl_oracle's step_loss_* compositions; the Entropy_Mini script calls losses.entropy_loss)"""
    soft = torch.softmax(logits, 1)
    if variant == "pce":
        return O.pce_loss(logits, label)
    if variant == "pce_gatedcrf":
        return O.step_loss_pce_gatedcrf(logits, image, label)[0]
    if variant == "pce_ms":
        return O.step_loss_pce_ms(logits, image, label)[0]
    if variant == "pce_tv":
        return O.step_loss_pce_tv(logits, label)[0]
    if variant == "pce_entropy":
        return O.pce_loss(logits, label) + 0.1 * O.entropy_loss(soft, 4)
    if variant == "pce_variance":
        return O.pce_loss(logits, label) + w_var * O.class_variance_loss(soft, image)
    assert variant == "ce_dice"
    return 0.5 * (O.pce_loss(logits, label) + O.dice_loss(soft, label.long().unsqueeze(1)))


VARIANTS = ("pce", "pce_gatedcrf", "pce_ms", "pce_tv", "pce_entropy", "pce_variance", "ce_dice")


@pytest.mark.parametrize("variant", VARIANTS)
def test_train_step_matches_fp64_for_three_iterations(variant):
    """fp16x3 PNet2D, batch 4 at 256 x 256, Dropout2d keep masks injected: loss at each of three iterations and the parameters after
    them against O.pnet2d_forward + the loss + O.sgd_step in fp64 (on the GPU), at the step's own poly learning rates"""
    N, it0, max_it = 4, (4500 if variant == "pce_variance" else 0), 30000
    m, p = _pnet("fp16x3")
    keep = _keeps(N, 5)
    m.channel_keep = keep
    x, y = O.synth_batch(N, HW, HW, seed=11, frac=0.05, dense=variant == "ce_dice")
    x, y = x.to(DEV), y.to(DEV)
    step = engine.TrainStep(m, variant, base_lr=0.01, max_iterations=max_it, graph=False)
    step.iter_num = it0
    losses = [step(x, y).item() for _ in range(3)]
    torch.cuda.synchronize()
    P, moms, ref = _p64(p), {}, []
    keys = _trained(P)
    with torch.device(DEV):                 # the oracle's helper tensors (the CRF's coordinates) on the GPU as well
        for k in range(3):
            L = _leaves(P)
            w_var = 0.1 * O.sigmoid_rampup((it0 + k) // 150, 200.0)
            loss = _oracle_loss(variant, _fwd(L, x.double(), keep), x.double(), y, w_var)
            grads = dict(zip(keys, torch.autograd.grad(loss, [L[q] for q in keys])))
            lr = 0.01 if k == 0 else O.poly_lr(0.01, it0 + k - 1, max_it)
            params = {q: P[q] for q in keys}
            O.sgd_step(params, grads, moms, lr)
            P.update(params)
            ref.append(loss.item())
    lerr = max(abs(a - b) / abs(b) for a, b in zip(losses, ref))
    named = dict(m.named_parameters())
    p0 = _p64(p)
    errs = {k: rel_l2(named[k].detach().double() - p0[k], P[k] - p0[k]) for k in keys}
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"[pnet {variant} fp16x3] losses {losses} / fp64 {ref}: worst loss error {lerr:.2e}; worst update error {worst}")
    assert lerr < 2e-3, (losses, ref)
    assert worst[1] < 3e-2, sorted(errs.items(), key=lambda kv: -kv[1])[:4]


# ---- 2. the other step classes against their oracles ----------------------------------------------------------------------------
def _noises(B, g, T=8):
    return [torch.clamp(torch.randn(B, 1, HW, HW, generator=g) * 0.1, -0.2, 0.2).to(DEV)] + \
           [torch.clamp(torch.randn(2 * B, 1, HW, HW, generator=g) * 0.1, -0.2, 0.2).to(DEV) for _ in range(T // 2)]


def _teacher_passes(pt, img, noises, keep_t):
    with torch.no_grad():
        ema = _fwd(pt, img + noises[0], keep_t)
        if len(noises) == 1:
            return ema, None
        k2 = [k.repeat(2, 1) for k in keep_t]
        return ema, torch.cat([_fwd(pt, img.repeat(2, 1, 1, 1) + n, k2) for n in noises[1:]], 0)


@pytest.mark.parametrize("method", ["uamt", "mt", "em", "dan"])
def test_two_batch_steps_match_their_oracles(method):
    """one fp16x3 step of the UAMT / mean-teacher / entropy-minimisation / DAN body on PNet2D (batch 2 + 2, teacher noise and every
    Dropout2d mask injected) against wsl_oracle.uamt_losses / semi_oracle.mt_losses / em_losses / the DAN oracle body, composed with
    pnet2d_forward in fp64: loss and the student's gradient bucket"""
    B, it = 2, 900
    g = torch.Generator().manual_seed(5)
    x, y = O.synth_batch(2 * B, HW, HW, seed=3, dense=True)
    x_l, y_l, x_u = x[:B].to(DEV), y[:B].to(DEV), x[B:].contiguous().to(DEV)
    s, ps = _pnet("fp16x3", 7)
    s.channel_keep = keep_s = _keeps(B, 6)
    t, pt = _pnet("fp16x3", 8)
    t.channel_keep = keep_t = _keeps(B, 9)
    noises = _noises(B, g, 8 if method == "uamt" else 0)
    if method == "uamt":
        step = engine.UAMTStep(s, t, graph=False)
    elif method == "mt":
        step = engine.MeanTeacherStep(s, t, graph=False)
    elif method == "em":
        step = engine.EntropyMinStep(s, graph=False)
    else:
        from wsl4mis_b200.networks.discriminator import FCDiscriminator
        disc = FCDiscriminator(4)
        disc.load_state_dict(D.synth_params(101))
        disc = disc.to(DEV).set_precision("fp32")
        pd = {k: v.detach().double() for k, v in disc.named_parameters()}
        step = engine.DANStep(s, disc, graph=False)
    step.iter_num = it
    if method in ("uamt", "mt"):
        loss = step(x_l, y_l, x_u, noises).item()
    else:
        loss = step(x_l, y_l, x_u).item()
    torch.cuda.synchronize()
    P = _p64(ps)
    L = _leaves(P)
    out_l, out_u = _fwd(L, x_l.double(), keep_s), _fwd(L, x_u.double(), keep_s)
    if method == "uamt":
        ema, mc = _teacher_passes(_p64(pt), x_u.double(), [n.double() for n in noises], keep_t)
        ref = O.uamt_losses(out_l, out_u, ema, mc, y_l, it, 30000)[0]
    elif method == "mt":
        ema, _ = _teacher_passes(_p64(pt), x_u.double(), [noises[0].double()], keep_t)
        ref = SO.mt_losses(out_l, out_u, ema, y_l, it)[0]
    elif method == "em":
        ref = SO.em_losses(out_l, out_u, y_l, it)[0]
    else:
        w = 0.1 * O.sigmoid_rampup(it // 150, 200.0)
        adv = F.cross_entropy(D.forward(pd, torch.softmax(out_u, 1), x_u.double(), False), torch.ones(B, dtype=torch.long, device=DEV))
        ref = SO.supervised_half(out_l, y_l) + w * adv
    keys = _trained(P)
    grads = dict(zip(keys, torch.autograd.grad(ref, [L[k] for k in keys])))
    worst = _check_grads(step, s, grads, 3e-2, method)
    print(f"[pnet {method} fp16x3] loss {loss:.7f} / fp64 {ref.item():.7f}; worst gradient {worst}")
    assert abs(loss - ref.item()) < 2e-3 * abs(ref.item()) + 1e-6, (loss, ref.item())


def test_ustm_step_matches_its_oracle():
    """one fp16x3 USTM step on PNet2D (rot90 count 1, teacher noise and masks injected) against wsl_oracle.ustm_losses on
    pnet2d_forward in fp64: loss, the student's gradient bucket, and the teacher's EMA update"""
    B, it, k = 2, 3500, 1
    g = torch.Generator().manual_seed(15)
    x, y = O.synth_batch(B, HW, HW, seed=13, frac=0.05)
    x, y = x.to(DEV), y.to(DEV)
    s, ps = _pnet("fp16x3", 17)
    s.channel_keep = keep_s = _keeps(B, 16)
    t, pt = _pnet("fp16x3", 18)
    t.channel_keep = keep_t = _keeps(B, 19)
    noises = _noises(B, g)
    step = engine.USTMStep(s, t, graph=False)
    step.iter_num = it
    loss = step(x, y, noises, rot_times=k).item()
    torch.cuda.synchronize()
    P = _p64(ps)
    L = _leaves(P)
    out = _fwd(L, x.double(), keep_s)
    ema, mc = _teacher_passes(_p64(pt), torch.rot90(x.double(), k, [2, 3]), [n.double() for n in noises], keep_t)
    ref = O.ustm_losses(out, ema, mc, y, k, it, 60000)[0]
    keys = _trained(P)
    grads = dict(zip(keys, torch.autograd.grad(ref, [L[q] for q in keys])))
    worst = _check_grads(step, s, grads, 3e-2, "ustm")
    assert abs(loss - ref.item()) < 2e-3 * abs(ref.item()) + 1e-6, (loss, ref.item())
    # teacher <- alpha * teacher + (1 - alpha) * student after the student's SGD step
    alpha = min(1 - 1 / (it + 1), 0.99)
    tn, sn = dict(t.named_parameters()), dict(s.named_parameters())
    terr = max(rel_l2(tn[q].detach().double(), alpha * pt[q].to(DEV).double() + (1 - alpha) * sn[q].detach().double()) for q in keys)
    print(f"[pnet ustm fp16x3] loss {loss:.7f} / fp64 {ref.item():.7f}; worst gradient {worst}; teacher EMA {terr:.1e}")
    assert terr < 1e-6


def test_s2l_step_matches_its_oracle():
    """one fp16x3 Scribble2Label step on PNet2D past thr_iter (pCE + 0.5 * CE on the u-labels) against s2l_oracle.step_loss on
    pnet2d_forward in fp64"""
    B = 2
    x, y = O.synth_batch(B, HW, HW, seed=21, frac=0.05)
    g = torch.Generator().manual_seed(22)
    weight = torch.softmax(torch.rand(B, HW, HW, 4, generator=g) * 6, -1)
    x, y, weight = x.to(DEV), y.to(DEV), weight.to(DEV)
    m, p = _pnet("fp16x3", 23)
    m.channel_keep = keep = _keeps(B, 24)
    step = engine.S2LStep(m, thr_iter=0, thr_conf=0.5, graph=False)
    loss = step(x, y, weight).item()
    torch.cuda.synchronize()
    P = _p64(p)
    L = _leaves(P)
    ref, _, lu = S2.step_loss(_fwd(L, x.double(), keep), y, weight.double(), 0, thr_iter=0, thr_conf=0.5)
    assert lu is not None and torch.isfinite(lu)
    keys = _trained(P)
    grads = dict(zip(keys, torch.autograd.grad(ref, [L[q] for q in keys])))
    worst = _check_grads(step, m, grads, 3e-2, "s2l")
    print(f"[pnet s2l fp16x3] loss {loss:.7f} / fp64 {ref.item():.7f}; worst gradient {worst}")
    assert abs(loss - ref.item()) < 2e-3 * abs(ref.item()), (loss, ref.item())


def test_per_sample_forward_equals_batch_one_forwards():
    """forward(..., bn_per_sample=True), the S2L refresh's forward, against N batch-1 training forwards on the same executor state
    and masks, and against the fp64 oracle slice by slice with the running statistics updated in slice order"""
    N = 4
    x, _ = O.synth_batch(N, HW, HW, seed=31)
    x = x.to(DEV)
    keep = _keeps(N, 32)
    m1, p = _pnet("fp16x3", 33)
    m2, _ = _pnet("fp16x3", 33)
    with torch.no_grad():
        ps = m1.executor.forward(x, True, False, None, keep, bn_per_sample=True)[0][0].clone()
        one = torch.cat([m2.executor.forward(x[i:i + 1].contiguous(), True, False, None, [k[i:i + 1] for k in keep])[0][0].clone()
                         for i in range(N)], 0)
    torch.cuda.synchronize()
    P = _p64(p)
    ref = []
    with torch.no_grad():
        for i in range(N):
            ns = {}
            ref.append(O.pnet2d_forward(P, x[i:i + 1].double(), True, [k[i:i + 1] for k in keep], ns))
            P.update(ns)
    ref = torch.cat(ref, 0)
    scale = ref.abs().max().item()
    e_one = (ps.double() - one.double()).abs().max().item() / scale
    e_ref = (ps.double() - ref).abs().max().item() / scale
    sd1, sd2 = m1.state_dict(), m2.state_dict()
    e_run = max(rel_l2(sd1[k].double(), P[k]) for k in P if "running" in k)
    e_run12 = max(rel_l2(sd1[k].double(), sd2[k].double()) for k in P if "running" in k)
    nbt = {int(v) - int(p[k]) for k, v in sd1.items() if k.endswith("num_batches_tracked")}
    print(f"[pnet per-sample forward] vs batch-1 forwards {e_one:.1e}, vs fp64 {e_ref:.1e} of scale; running statistics vs fp64 "
          f"{e_run:.1e}, vs batch-1 forwards {e_run12:.1e}; num_batches_tracked {nbt}")
    assert e_one < 1e-3 and e_ref < 1e-3
    assert e_run < 1e-4 and e_run12 < 1e-4
    assert nbt == {N}


# ---- 3. captured == eager ---------------------------------------------------------------------------------------------------------
def _graph_pair(method):
    """(eager step, graph step) on PNet2D built from one seed, bf16 (device-drawn dropout masks and teacher noise)"""
    steps = []
    for graph in (False, True):
        torch.manual_seed(33)
        s = net_factory("pnet", 1, 4)
        if method in ("pce_variance", "pce", "ce_dice"):
            steps.append(engine.TrainStep(s, method, graph=graph))
        elif method == "s2l":
            steps.append(engine.S2LStep(s, thr_iter=3, thr_conf=0.5, graph=graph))
        elif method == "em":
            steps.append(engine.EntropyMinStep(s, graph=graph))
        elif method == "dan":
            from wsl4mis_b200.networks.discriminator import FCDiscriminator
            steps.append(engine.DANStep(s, FCDiscriminator(4).to(DEV), graph=graph))
        else:
            cls = {"mt": engine.MeanTeacherStep, "uamt": engine.UAMTStep, "ustm": engine.USTMStep}[method]
            steps.append(cls(s, net_factory("pnet", 1, 4), graph=graph))
    return steps


RAMP_START = {"pce_variance": 295, "dan": 145, "ustm": 995, "mt": 296, "uamt": 296, "em": 296}
TWO_STREAM = [(2, 2), (2, 2), (2, 2), (2, 1), (2, 1), (2, 1), (1, 1), (1, 1), (1, 1), (2, 2)]


ATOMIC = "block1.conv1.weight"     # its weight gradient (1 input channel, from the fp32 image) is summed with atomics


@pytest.mark.parametrize("method", ["pce", "pce_variance", "ce_dice", "s2l", "ustm", "mt", "uamt", "em", "dan"])
def test_graph_equals_eager(method):
    """ten steps of a graph step and an eager step in lockstep on bf16 PNet2D: across a change of the ramp weight (and S2L's switch
    at thr_iter), and for the two-stream steps across the short last batches of an epoch.  The loss is bit-identical at every step,
    and so are the flat parameters, momentum and teacher, except the slice of `ATOMIC`: the module path's weight gradient of the
    image layer adds its partial sums with atomics, which differs in the last bits from run to run (eager against eager as well).
    That slice agrees to 1e-6 and is copied from the eager step to the graph step after every step, so each step starts from the
    same state.  DAN's discriminator (which reads the updated student's maps) and USTM's EMA teacher (a different arithmetic
    form when captured) agree to the same 1e-6 and are copied likewise."""
    eager, captured = _graph_pair(method)
    for st in (eager, captured):
        st.iter_num = RAMP_START.get(method, 0)
    x, y = O.synth_batch(8, HW, HW, seed=41, frac=0.05)
    _, yd = O.synth_batch(8, HW, HW, seed=42, dense=True)
    x, y, yd = x.to(DEV), y.to(DEV), yd.to(DEV)
    g = torch.Generator().manual_seed(43)
    weight = torch.softmax(torch.rand(2, HW, HW, 4, generator=g) * 6, -1).to(DEV)
    state = ("flat", "mom")
    # DAN's discriminator reads the updated student's maps; USTM's teacher takes the EMA update as wsl_ema_update when eager and
    # as a lerp with the factor from device memory when captured
    whole = {"dan": ("dflat", "exp_avg", "exp_avg_sq"), "ustm": ("tflat",)}.get(method, ())
    q = dict(eager.model.named_parameters())[ATOMIC]
    off, n = eager.offsets[id(q)]
    worst = 0.0
    for i in range(10):
        if method in ("mt", "uamt", "em", "dan"):
            bl, bu = TWO_STREAM[i]
            args, kw = (x[:bl], yd[:bl], x[4:4 + bu]), {}
        elif method == "s2l":
            args, kw = (x[:2], y[:2], weight), {}
        elif method == "ustm":
            args, kw = (x[:2], y[:2]), {"rot_times": i % 4}
        else:
            args, kw = (x[:2], (yd if method == "ce_dice" else y)[:2]), {}
        le, lg = eager(*args, **kw), captured(*args, **kw)
        torch.cuda.synchronize()
        assert torch.equal(le, lg), (method, i, le.item(), lg.item())
        for name in state:
            a, b = getattr(captured, name), getattr(eager, name)
            assert torch.equal(a[:off], b[:off]) and torch.equal(a[off + n:], b[off + n:]), (method, i, name)
            d = rel_l2(a[off:off + n], b[off:off + n])
            worst = max(worst, d)
            assert d < 1e-6, (method, i, name, d)
            a.copy_(b)
        for name in whole:
            a, b = getattr(captured, name), getattr(eager, name)
            d = rel_l2(a, b)
            worst = max(worst, d)
            assert d < 1e-6, (method, i, name, d)
            a.copy_(b)
    assert captured.iter_num == eager.iter_num
    # pce_variance runs eagerly by design (its ramp weight is a launch argument of the backward kernel)
    assert (len(captured._graphs) >= 1) == (method != "pce_variance"), captured._graphs
    print(f"[pnet {method} graph == eager] 10 steps, losses bit-identical, {len(captured._graphs)} graphs; {ATOMIC} (and the "
          f"teacher / D) within {worst:.1e}")


# ---- 4. bf16 step against the autograd module path ------------------------------------------------------------------------------
def test_bf16_pce_step_matches_the_module_path():
    """TrainStep('pce') on bf16 PNet2D against m(x) -> CrossEntropyLoss(ignore_index=4) -> torch.optim.SGD on the same weights and
    Dropout2d masks: the same kernels, so the loss agrees to 1e-6 and the update to the bf16 bound of the semi-step tests"""
    N = 4
    x, y = O.synth_batch(N, HW, HW, seed=51, frac=0.05)
    x, y = x.to(DEV), y.to(DEV)
    m1, p = _pnet("bf16", 52)
    m2, _ = _pnet("bf16", 52)
    m1.channel_keep = m2.channel_keep = _keeps(N, 53)
    s0 = {k: q.detach().clone() for k, q in m2.named_parameters()}
    loss = engine.TrainStep(m1, "pce", graph=False)(x, y).item()
    opt = torch.optim.SGD(m2.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    m2.train()
    ref = torch.nn.CrossEntropyLoss(ignore_index=4)(m2(x), y.long())
    opt.zero_grad()
    ref.backward()
    opt.step()
    torch.cuda.synchronize()
    assert abs(loss - ref.item()) < 1e-6 * abs(ref.item()), (loss, ref.item())
    n1, n2 = dict(m1.named_parameters()), dict(m2.named_parameters())
    # test_gpu_semi_steps.py's bf16 bound: every update direction within cosine 0.85 (block conv biases: weight decay only)
    cos = {k: cosine(n1[k].detach() - s0[k], n2[k].detach() - s0[k]) for k in n1 if not _feeds_bn(k)}
    worst = min(cos.items(), key=lambda kv: kv[1])
    whole = rel_l2(torch.cat([(n1[k].detach() - s0[k]).flatten() for k in n1]), torch.cat([(n2[k].detach() - s0[k]).flatten() for k in n1]))
    print(f"[pnet bf16 pce] loss {loss:.7f} / module path {ref.item():.7f}; worst update cosine {worst}; whole update rel. L2 {whole:.2e}")
    assert worst[1] > 0.85, sorted(cos.items(), key=lambda kv: kv[1])[:4]


def test_global_batch_and_sync_bn_are_rejected():
    m, _ = _pnet("bf16")
    with pytest.raises(NotImplementedError, match="PNet2D"):
        m.executor.sync_bn = (2, None)
    assert m.executor.sync_bn is None
    assert (m.executor.n_outputs, m.executor.aux_param_ids, m.executor.comm_split) == (1, set(), None)


def test_dmpls_needs_two_outputs():
    m, _ = _pnet("bf16")
    with pytest.raises(AssertionError, match="two-head"):
        engine.TrainStep(m, "dmpls", graph=False)


# ---- 5. launch census -----------------------------------------------------------------------------------------------------------
def _census():
    """{launch key: [where]} of one eager bf16 iteration of every PNet recipe at its own batch, the S2L refresh, one resident
    validation pass and one test-step volume"""
    from wsl4mis_b200 import test_2D, val_2D
    from wsl4mis_b200.dataloaders.dataset import BaseDataSets_s2l
    import test_gpu_conv_at_scale as CS
    seen = {}

    def rec(run, where):
        r, saved = LaunchRecorder(lambda name: True), _lib.PROFILE
        _lib.PROFILE = r
        try:
            run()
            torch.cuda.synchronize()
        finally:
            _lib.PROFILE = saved
        for key in r.launches:
            seen.setdefault(key, []).append(where)
    for script, recipe in TR.RECIPES.items():
        if recipe.step is TR._DMPLS:
            continue
        args = TR.parser_for(script).parse_args(["--model", "pnet"])
        B = TR.rank_batch(script, args.batch_size, 1)
        torch.manual_seed(0)
        model = net_factory("pnet", 1, 4).set_precision("bf16")
        step = recipe.step(args, model, 1)
        step.graph_enabled = False
        inputs = CS._census_inputs(script, recipe, args, B, torch.Generator().manual_seed(len(script)))
        rec(lambda: step(*inputs), f"{script} at batch {B}")
        if recipe.kind == "s2l":
            store = BaseDataSets_s2l(base_dir="synthetic:30", fold="fold1").to_slice_store()
            rec(lambda: step.refresh(store), f"S2L refresh of {len(store)} slices")
        del model, step, inputs
        gc.collect()
        torch.cuda.empty_cache()
    net = net_factory("pnet", 1, 4)
    rs = np.random.RandomState(5)
    shapes = [(30, 200, 180), (25, 256, 256), (20, 212, 240)]
    vs = val_2D.ValidationSet.from_arrays([rs.rand(*s).astype(np.float32) for s in shapes],
                                          [rs.randint(0, 4, s).astype(np.uint8) for s in shapes])
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    rec(lambda: vs.predict(net), f"validation pass (chunk {vs.chunk})")
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    vol = rs.rand(20, 230, 210).astype(np.float32)
    rec(lambda: test_2D.predict_volume(vol, net), f"test step (chunk {test_2D.CHUNK})")
    del net, vs
    torch.cuda.empty_cache()
    return seen, peak


# Launches over a bound, measured: catblock.conv1's weight gradient (1x1, 320 -> 320) at the pCE recipes' default batch 24 sums
# N*H*W = 1.57 M pixels per weight with up to twice the per-CTA split-K chain of batch 12 and reaches rel-L2 1.03e-4 against fp64
# on one call and 1.12e-4 accumulated over two (the deterministic and the atomics path alike), over _conv_check.WGRAD_TOL = 1e-4
# (measured on an H100 80GB HBM3 at 700 W).  Recorded here, not hidden: its error / bound must stay under 1.25.
OVER_BOUND = {("wsl_wgrad_tc", "24x256x256 320->320 k1"): 1.25}


def test_census_every_launch_of_the_pnet_recipes_is_replayed():
    """every convolution and network-op launch the PNet recipes' steps, the S2L refresh, the validation pass and the test step make
    is either one of the pnet2d-n12-* module-path harvests or is replayed here against fp64 with the at-scale files' bounds (the
    launches of OVER_BOUND: within their stated multiple of it)"""
    import test_gpu_conv_at_scale as CS
    import test_gpu_netops_at_scale as NS
    seen, peak = _census()
    print(f"\nvalidation pass at chunk 64: peak allocated {peak:.1f} GiB on {torch.cuda.get_device_name(0)}")
    harvested = set()
    for c in ("pnet2d-n12-bf16", "pnet2d-n12-fp16"):
        harvested |= set(CS._harvest(*CS.CONFIGS[c]))
        harvested |= set(NS._harvest(c)[0])
    conv = {k: w for k, w in seen.items() if k[0] in CS.HARVESTED}
    ops = {k: w for k, w in seen.items() if k[0] in NS.REPLAY}
    new_conv = {k: w for k, w in conv.items() if k not in harvested}
    new_ops = {k: w for k, w in ops.items() if k not in harvested}
    fails = []
    for key, where in sorted(new_conv.items(), key=repr):
        row, f = CS._replay(key)
        print(f"  {row['entry']:<19} {row['kernel']:<14} {row['dtype']:<6} {row['shape']:<28} error/bound {row['worst']:.3g}  <- "
              f"{', '.join(sorted(set(where)))[:120]}")
        limit = OVER_BOUND.get((row["entry"], row["shape"]))
        if limit is not None and all("over the bound" in m or "does not add on top" in m for m in f):
            assert row["worst"] < limit, (row["entry"], row["shape"], row["worst"])
            continue
        fails += [f"{row['entry']} {row['shape']}: {m}" for m in f]
    for key, where in sorted(new_ops.items(), key=repr):
        a = dict(key[1])
        row, f = NS._replay(key, a.get("N", 1))
        print(f"  {row['entry']:<28} {row['dtype']:<5} {row['shape']:<30} error/bound {row['worst']:.3g}  <- "
              f"{', '.join(sorted(set(where)))[:120]}")
        fails += [f"{row['entry']} {row['shape']}: {m}" for m in f]
    print(f"census: {len(conv)} convolution and {len(ops)} network-op launches, {len(new_conv)} + {len(new_ops)} replayed here")
    assert any(k[0] == "wsl_bn_stats_ps" and dict(k[1])["C"] == 64 for k in new_ops), "the refresh's per-sample BatchNorm is missing"
    assert not fails, "\n".join(fails[:40])


# ---- 6. the trainer -------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def workdir(tmp_path, monkeypatch):
    work = tmp_path / "code"
    work.mkdir()
    monkeypatch.chdir(work)
    return tmp_path


PNET_SCRIPTS = sorted(s for s, r in TR.RECIPES.items() if r.step is not TR._DMPLS) if torch.cuda.is_available() else []


@pytest.mark.parametrize("script", PNET_SCRIPTS)
def test_every_recipe_trains_pnet(workdir, script, monkeypatch):
    """four iterations of every recipe but pCE_ours_proposed with --model pnet on synthetic:30, validated at iteration 4 and saved:
    the checkpoints carry the reference's keys and load into a fresh net_factory('pnet').  pnet_best_model.pth is written on a
    strict improvement of the mean Dice over 0, as in the scripts, which four iterations need not reach."""
    monkeypatch.setattr(TR, "VAL_EVERY", 4)
    monkeypatch.setattr(TR, "SAVE_EVERY", 4)
    recipe = TR.RECIPES[script]
    bs = 4 if recipe.kind == "semi" else 2
    extra = ["--period_iter", "2"] if recipe.kind == "s2l" else []
    snap = TR.train([script, "--root_path", "synthetic:30", "--exp", "P/r", "--fold", "fold1", "--max_iterations", "4",
                     "--batch_size", str(bs), "--model", "pnet", *extra])
    log = open(os.path.join(snap, "log.txt")).read()
    dice = float(log.split("iteration 4 : mean_dice : ")[1].split()[0])
    files = os.listdir(snap)
    assert "iter_4.pth" in files and ("pnet_best_model.pth" in files) == (dice > 0), (files, dice)
    keys = list(net_factory("pnet", 1, 4).state_dict().keys())
    for f in [f for f in files if f.endswith(".pth")]:
        sd = torch.load(os.path.join(snap, f))
        assert list(sd.keys()) == keys
        net_factory("pnet", 1, 4).load_state_dict(sd)


def test_test_2D_scores_a_pnet_checkpoint(workdir):
    import shutil
    import wsl4mis_b200.test_2D as T2
    snap = TR.train(["train_weakly_supervised_pCE_2D.py", "--root_path", "synthetic:30", "--exp", "P/t", "--fold", "fold1",
                     "--max_iterations", "6", "--batch_size", "4", "--model", "pnet"])
    sd = torch.load(os.path.join(snap, "pnet_best_model.pth")) if os.path.exists(os.path.join(snap, "pnet_best_model.pth")) else None
    torch.save(sd if sd is not None else net_factory("pnet", 1, 4).state_dict(), os.path.join(snap, "iter_60000.pth"))
    F_ = T2.parser.parse_args(["--root_path", "synthetic:30", "--exp", "P/t", "--fold", "fold1", "--sup_type", "scribble",
                               "--model", "pnet"])
    torch.cuda.reset_peak_memory_stats()
    try:
        dice = T2.Inference(F_)
        assert np.isfinite(dice)
    except RuntimeError as e:          # medpy's behaviour on an empty predicted class, as the script's
        assert "does not contain any binary object" in str(e)
    print(f"[pnet test_2D] peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB at chunk {T2.CHUNK}")
    shutil.rmtree(snap)


def _ddp_worker(rank, world, port, base, argv):
    import test_gpu_train_ddp as TD
    TD._trainer_worker(rank, world, port, "nccl", base, argv)


def test_two_rank_pnet_replicas_stay_bit_identical(tmp_path):
    """torchrun-style two-rank run of the pCE recipe on PNet2D: the comm overlap is off (no encoder/decoder split), the whole bucket
    is all-reduced after backward, and the replicas are bit-identical after 5 steps"""
    import test_gpu_train_ddp as TD
    TD._need("nccl")
    argv = ["train_weakly_supervised_pCE_2D.py", "--root_path", "synthetic:30", "--exp", "DDP/p", "--fold", "fold1",
            "--max_iterations", "5", "--batch_size", "4", "--model", "pnet"]
    TD._spawn(_ddp_worker, 2, str(tmp_path), argv)
    s0, s1 = (torch.load(os.path.join(tmp_path, f"state{r}.pt")) for r in range(2))
    assert torch.equal(s0["flat"].view(torch.int32), s1["flat"].view(torch.int32))
