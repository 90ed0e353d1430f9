"""Data-parallel training on the GPU: the scaled Adam entry point, the trainer in a one-process group against the plain run, and two
ranks of DANStep, S2LStep (with its sharded refresh) and the trainer.

The two-rank tests run twice: over NCCL on two GPUs (skipped on a single-GPU box), and over gloo with both ranks sharing GPU 0,
which checks the same collectives' placement and arithmetic on any box with one GPU."""
import os
import re
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = "synthetic:100"
BACKENDS = ["nccl", "gloo"]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _strip(line):
    return re.sub(r"^\[\d\d:\d\d:\d\d\.\d{3}\] ", "", line)


def _need(backend):
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")


def _join(rank, world, port, backend, init=True):
    """torchrun's environment for `rank`, its device, and (init) the process group -> device"""
    import datetime
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if init:
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120),
                                **({"device_id": dev} if backend == "nccl" else {}))
    return dev


def _spawn(fn, world, *args):
    import torch.multiprocessing as mp
    mp.spawn(fn, args=(world, _free_port()) + args, nprocs=world, join=True)


# ---------------------------------------------------------------- Adam's gradient scale
def test_adam_grad_scale():
    from wsl4mis_b200._lib import call
    n = 100_003
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g).to(DEV)
    # gradients on a 2^-12 grid: their sum and its half are exact in fp32
    ga = (torch.randint(-4096, 4096, (n,), generator=g).float() / 4096).to(DEV)
    gb = (torch.randint(-4096, 4096, (n,), generator=g).float() / 4096).to(DEV)
    gsum, gmean = ga + gb, (ga + gb) * 0.5
    assert torch.equal(gsum * 0.5, gmean)

    def run(entry, grad, *scale, steps=4):
        p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        for t in range(1, steps + 1):
            call(entry, p, grad, m, v, n, None, 1e-4 / (1 - 0.9 ** t), (1 - 0.99 ** t) ** 0.5, 0.9, 0.99, 1e-8, *scale)
        return p, m, v

    base = run("wsl_adam_step", ga)
    for a, b in zip(base, run("wsl_adam_step_scaled", ga, 1.0)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for a, b in zip(run("wsl_adam_step_scaled", gsum, 0.5), run("wsl_adam_step", gmean)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    # the scale acts before the moments: Adam on the unscaled sum takes a different step (eps breaks scale invariance)
    assert not torch.equal(run("wsl_adam_step", gsum)[0], run("wsl_adam_step", gmean)[0])


# ---------------------------------------------------------------- a one-process group changes nothing
def _argv(script, exp, iters, bs):
    return [script, "--root_path", ROOT, "--exp", exp, "--fold", "fold1", "--max_iterations", str(iters), "--batch_size", str(bs)]


def _group_of_one(rank, world, port, workdir, argv):
    import torch.distributed as dist
    _join(rank, world, port, "nccl")
    try:
        os.makedirs(workdir, exist_ok=True)
        os.chdir(workdir)
        import wsl4mis_b200.train as TR
        TR.train(argv)
    finally:
        dist.destroy_process_group()


def _checkpoints(snap):
    return {f: torch.load(os.path.join(snap, f)) for f in sorted(os.listdir(snap)) if f.endswith(".pth")}


@pytest.mark.parametrize("script", ["train_weakly_supervised_pCE_2D.py", "train_mean_teacher_2D.py"])
def test_one_process_group_equals_the_plain_run(tmp_path, monkeypatch, script):
    import wsl4mis_b200.train as TR
    argv = _argv(script, "G1/r", 400, 12)
    _spawn(_group_of_one, 1, str(tmp_path / "group" / "code"), argv)
    monkeypatch.chdir(tmp_path)
    (tmp_path / "plain" / "code").mkdir(parents=True)
    monkeypatch.chdir(tmp_path / "plain" / "code")
    snap = TR.train(argv)
    a = os.path.join(tmp_path, "group", "code", snap)
    b = os.path.join(tmp_path, "plain", "code", snap)
    la, lb = ([_strip(l) for l in open(os.path.join(d, "log.txt")).read().splitlines()] for d in (a, b))
    assert la == lb and sum("mean_dice" in l for l in la) == 2
    ca, cb = _checkpoints(a), _checkpoints(b)
    assert list(ca) == list(cb) and ca
    for f in ca:
        assert list(ca[f]) == list(cb[f])
        assert all(torch.equal(ca[f][k], cb[f][k]) for k in ca[f]), f


# ---------------------------------------------------------------- two ranks of DANStep and S2LStep
N_RANK = 2          # images per rank and stream


def _dan_data(world):
    g = torch.Generator().manual_seed(21)
    n = N_RANK * world
    return (torch.rand(n, 1, 256, 256, generator=g), torch.randint(0, 4, (n, 256, 256), generator=g).to(torch.uint8),
            torch.rand(n, 1, 256, 256, generator=g))


def _dan_pair(dev, n):
    from _gpu_util import elem_masks_nchw
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    from wsl4mis_b200.networks.unet import UNet
    torch.manual_seed(7)
    s, d = UNet(1, 4).to(dev), FCDiscriminator(4).to(dev)
    em = elem_masks_nchw(11, n, 256, 256)
    s.dropout_masks = {i: em[i].permute(0, 2, 3, 1).contiguous().to(dev) for i in range(5)}
    rs = np.random.RandomState(17)
    d.channel_keep = [torch.from_numpy((rs.uniform(size=(2 * n, c)) >= 0.5).astype(np.uint8)).to(dev) for c in (128, 256)]
    return s, d


def _s2l_data(world):
    g = torch.Generator().manual_seed(31)
    n = N_RANK * world
    lab = torch.randint(0, 4, (n, 256, 256), generator=g).to(torch.uint8)
    scr = torch.where(torch.rand(n, 256, 256, generator=g) < 0.1, lab, torch.full_like(lab, 4))
    w = torch.rand(n, 256, 256, 4, generator=g)
    return torch.rand(n, 1, 256, 256, generator=g), scr, w / w.sum(-1, keepdim=True)


def _s2l_model(dev, n):
    from _gpu_util import elem_masks_nchw
    from wsl4mis_b200.networks.unet import UNet
    torch.manual_seed(9)
    m = UNet(1, 4).to(dev)
    em = elem_masks_nchw(12, n, 256, 256)
    m.dropout_masks = {i: em[i].permute(0, 2, 3, 1).contiguous().to(dev) for i in range(5)}
    return m


def _s2l_store(dev):
    from wsl4mis_b200.dataloaders.dataset import SliceStore
    rs = np.random.RandomState(5)
    shapes = ((216, 256), (256, 216), (174, 208), (232, 256), (224, 154))
    ims = [rs.rand(*shapes[i % 5]).astype(np.float32) for i in range(13)]
    labs = [rs.randint(0, 4, im.shape).astype(np.uint8) for im in ims]
    store = SliceStore.from_arrays(ims, labs, device=dev, scribbles=[np.where(rs.rand(*l.shape) < 0.3, l, 4).astype(np.uint8) for l in labs])
    store.weight_live.copy_(torch.from_numpy(rs.rand(*store.weight_live.shape).astype(np.float32)))
    return store


def _refresh_masks(dev, n):
    from _gpu_util import elem_masks_nchw
    return {i: e.permute(0, 2, 3, 1).contiguous().to(dev) for i, e in enumerate(elem_masks_nchw(13, n, 256, 256))}


def _step_worker(rank, world, port, backend, kind, out_dir):
    import torch.distributed as dist
    dev = _join(rank, world, port, backend)
    try:
        from wsl4mis_b200.engine import DANStep, S2LStep
        lo, hi = rank * N_RANK, (rank + 1) * N_RANK
        res = {}
        if kind == "dan":
            xl, yl, xu = (t[lo:hi].to(dev) for t in _dan_data(world))
            s, d = _dan_pair(dev, N_RANK)
            step = DANStep(s, d, graph=True, world_size=world)
            inputs = (xl, yl, xu)
        else:
            m = _s2l_model(dev, N_RANK)
            step = S2LStep(m, thr_iter=0, graph=True, world_size=world)
            store = _s2l_store(dev)
            step.refresh(store, alpha=0.2, chunk=4, masks=_refresh_masks(dev, len(store)))
            torch.cuda.synchronize()
            res["memory"] = store.weight_live.cpu()
            inputs = tuple(t[lo:hi].to(dev) for t in _s2l_data(world))
        for it in range(5):
            step(*inputs)
            if it == 0:
                torch.cuda.synchronize()
                res["bucket0"] = step.ex.grads()[0][: step.n_trained].cpu()
                if kind == "dan":
                    res["dbucket0"] = step.dgrad.cpu()
        torch.cuda.synchronize()
        res["graphs"] = len(step._graphs)
        res["flat"] = step.flat.cpu()
        res["mom"] = step.mom.cpu()
        if kind == "dan":
            res.update(dflat=step.dflat.cpu(), exp_avg=step.exp_avg.cpu(), exp_avg_sq=step.exp_avg_sq.cpu())
        torch.save(res, os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _two_ranks(tmp_path, backend, kind):
    _need(backend)
    _spawn(_step_worker, 2, backend, kind, str(tmp_path))
    return [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("backend", BACKENDS)
def test_two_rank_dan_step(tmp_path, backend):
    from wsl4mis_b200.engine import DANStep, _ramp
    res = _two_ranks(tmp_path, backend, "dan")
    assert res[0]["graphs"] == 1
    for k in ("flat", "mom", "dflat", "exp_avg", "exp_avg_sq"):
        assert _bits_equal(res[0][k], res[1][k]), k           # replicas bit-identical after five steps (three of them replays)
    # one process, the same weights: each shard's phase 1 from the same BatchNorm buffers, SGD on the mean of the two buckets, then
    # each shard's phase 2 with the running statistics its own rank holds
    xl, yl, xu = _dan_data(2)
    s, d = _dan_pair(DEV, N_RANK)
    st = DANStep(s, d, graph=False)
    st.ramp_dev.copy_(torch.tensor([_ramp(st.consistency, 0, 150, st.consistency_rampup), 0.0, 1.0]))   # iteration 0's weight
    buffers0 = [b.clone() for b in s.buffers()]
    shards, gsum, after = [], None, []
    for r in range(2):
        for b, b0 in zip(s.buffers(), buffers0):
            b.copy_(b0)
        sh = tuple(t[r * N_RANK:(r + 1) * N_RANK].to(DEV) for t in (xl, yl, xu))
        s.train()
        _, g = st._fwd_bwd(*sh)
        g = g[: st.n_trained].clone()
        gsum = g if gsum is None else gsum + g
        shards.append((sh, dict(st.parts)))
        after.append([b.clone() for b in s.buffers()])
    torch.cuda.synchronize()
    err = _rel(res[0]["bucket0"], gsum.cpu())
    print(f"[{backend}] DAN student bucket vs the sum of per-shard gradients: rel-L2 {err:.2e}")
    assert err < 2e-3, err
    st.world_size = 2                                   # SGD on the mean, once
    full = torch.zeros_like(st.flat)
    full[: st.n_trained] = gsum
    st._opt(full)
    st._opt = lambda g: None
    dsum = None
    for r, (sh, parts) in enumerate(shards):
        for b, b1 in zip(s.buffers(), after[r]):
            b.copy_(b1)
        st._inputs, st.parts = (sh[0], sh[2]), parts
        st._phase2(None)
        dsum = st.dgrad.clone() if dsum is None else dsum + st.dgrad
    torch.cuda.synchronize()
    err = _rel(res[0]["dbucket0"], dsum.cpu())
    print(f"[{backend}] DAN discriminator bucket vs the sum of per-shard gradients: rel-L2 {err:.2e}")
    assert err < 2e-3, err


@pytest.mark.parametrize("backend", BACKENDS)
def test_two_rank_s2l_step_and_refresh(tmp_path, backend):
    from wsl4mis_b200.engine import S2LStep
    res = _two_ranks(tmp_path, backend, "s2l")
    assert res[0]["graphs"] == 1
    for k in ("flat", "mom", "memory"):
        assert _bits_equal(res[0][k], res[1][k]), k
    m = _s2l_model(DEV, N_RANK)
    st = S2LStep(m, thr_iter=0, graph=False)
    store = _s2l_store(DEV)
    st.refresh(store, alpha=0.2, chunk=4, masks=_refresh_masks(DEV, len(store)))
    torch.cuda.synchronize()
    assert _bits_equal(res[0]["memory"], store.weight_live.cpu())      # the sharded refresh is the one-process refresh
    st.ctrl[1].fill_(0.5)
    data, gsum = _s2l_data(2), None
    for r in range(2):
        m.train()
        _, g = st._fwd_bwd(*(t[r * N_RANK:(r + 1) * N_RANK].to(DEV) for t in data))
        g = g[: st.n_trained].clone()
        gsum = g if gsum is None else gsum + g
    torch.cuda.synchronize()
    err = _rel(res[0]["bucket0"], gsum.cpu())
    print(f"[{backend}] S2L bucket vs the sum of per-shard gradients: rel-L2 {err:.2e}")
    assert err < 2e-3, err


# ---------------------------------------------------------------- two ranks of the trainer
def _trainer_worker(rank, world, port, backend, base, argv):
    import torch.distributed as dist
    _join(rank, world, port, backend, init=backend != "nccl")     # over NCCL the trainer creates and destroys the group itself
    work = os.path.join(base, f"rank{rank}", "code")
    os.makedirs(work)
    os.chdir(work)
    import wsl4mis_b200.train as TR
    orig = TR.Trainer.run

    def run(self):
        out = orig(self)
        torch.cuda.synchronize()
        st = {"flat": self.step.flat.cpu(), "n": self.n_per_epoch}
        if hasattr(self.step, "dflat"):
            st["dflat"] = self.step.dflat.cpu()
        torch.save(st, os.path.join(base, f"state{rank}.pt"))
        return out
    TR.Trainer.run = run
    try:
        TR.train(argv)
        if backend == "nccl":
            assert not dist.is_initialized()
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _files(root):
    return sorted(os.path.relpath(os.path.join(dp, f), root) for dp, _, fs in os.walk(root) for f in fs)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("script,bs", [("train_weakly_supervised_segmentation_pCE_ours_proposed.py", 8),
                                       ("train_deep_adversarial_network_2D.py", 8)])
def test_two_rank_trainer(tmp_path, backend, script, bs):
    _need(backend)
    argv = _argv(script, "DDP/r", 400, bs)
    _spawn(_trainer_worker, 2, backend, str(tmp_path), argv)
    s0, s1 = (torch.load(os.path.join(tmp_path, f"state{r}.pt")) for r in range(2))
    assert _bits_equal(s0["flat"], s1["flat"]) and ("dflat" not in s0 or _bits_equal(s0["dflat"], s1["dflat"]))
    assert _files(tmp_path / "rank1") == []
    r0 = _files(tmp_path / "rank0")
    assert r0 and all(f.startswith("model" + os.sep) for f in r0)
    import wsl4mis_b200.train as TR
    sup = TR.parse([script])[1].sup_type
    log = [_strip(l) for l in open(os.path.join(tmp_path, "rank0", "model", "DDP", "r_fold1", sup, "log.txt")).read().splitlines()]
    assert log[1] == f"{s0['n']} iterations per epoch"
    assert [int(l.split()[1]) for l in log if "mean_dice" in l] == [200, 400]
    it = [l for l in log if l.startswith("iteration ") and " : loss : " in l]
    assert [int(l.split()[1]) for l in it] == list(range(1, 401))

