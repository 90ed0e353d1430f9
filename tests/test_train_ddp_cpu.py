"""The trainer's data-parallel mode on the host (wsl4mis_b200/train.py): two gloo ranks through `train` with a fake step, fake
batches and a fake validator (only rank 0 logs, validates and saves, and its lines are those of a one-process run fed its inputs),
the batch-size rule, today's Namespace and loader sizes without a torchrun environment, the loaders' DistributedSampler partition
and their per-rank augmentation streams."""
import argparse
import os
import random
import re
import socket

import numpy as np
import pytest
import torch

import wsl4mis_b200.train as T
from wsl4mis_b200.dataloaders import dataset as D

SCRIPT = "train_weakly_supervised_pCE_2D.py"
TORCHRUN_VARS = ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _strip(line):
    return re.sub(r"^\[\d\d:\d\d:\d\d\.\d{3}\] ", "", line)


# ---------------------------------------------------------------- two gloo ranks through train()
class FakeStep:
    def __init__(self):
        self.loss_parts = {}

    def __call__(self, x):
        self.loss_parts = {"ce": torch.tensor(x * 0.5)}
        return torch.tensor(float(x))


class FakeValidator:
    calls = []

    def __init__(self, root_path, fold):
        pass

    def score(self, model, classes):
        FakeValidator.calls.append(model.training)
        d = 0.1 * len(FakeValidator.calls)
        return [[(d, 2.0 * d)] * (classes - 1)]


def _fake_build(script, args, precision, rank=0, world_size=1):
    """rank r's batches are numbered 1000 * r + i: a one-process run with rank=0 is fed what rank 0 of a group is fed"""
    torch.manual_seed(args.seed)
    model = torch.nn.Linear(2, 2)
    n = 7
    counter = iter(range(1000 * rank + 1, 1000 * rank + 10 ** 5))
    return model, FakeStep(), (lambda: ((next(counter),) for _ in range(n))), n, None


def _train_in(workdir, argv):
    import wsl4mis_b200.val_2D as V
    os.makedirs(workdir, exist_ok=True)
    old = os.getcwd()
    saved = (T.build, V.ValidationSet, T._summary_writer)
    T.build, V.ValidationSet, T._summary_writer = _fake_build, FakeValidator, (lambda path: None)
    os.chdir(workdir)
    try:
        return T.train(argv)
    finally:
        os.chdir(old)
        T.build, V.ValidationSet, T._summary_writer = saved


ARGV = [SCRIPT, "--exp", "DDP/fake", "--max_iterations", "450", "--batch_size", "4"]


def _rank_worker(rank, world, port, base):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _train_in(os.path.join(base, f"rank{rank}", "code"), ARGV)
        with open(os.path.join(base, f"validator{rank}.txt"), "w") as f:
            f.write(str(len(FakeValidator.calls)))
        assert dist.is_initialized()             # train() keeps a group its caller created
    finally:
        dist.destroy_process_group()


def _files(root):
    return sorted(os.path.relpath(os.path.join(dp, f), root) for dp, _, fs in os.walk(root) for f in fs)


def test_two_gloo_ranks_only_rank0_logs_validates_and_saves(tmp_path, monkeypatch):
    import torch.multiprocessing as mp
    for v in TORCHRUN_VARS:
        monkeypatch.delenv(v, raising=False)
    mp.spawn(_rank_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    snap = os.path.join("model", "DDP", "fake_fold1", "scribble")
    r0 = _files(tmp_path / "rank0")
    assert os.path.join(snap, "log.txt") in r0 and os.path.join(snap, "unet_best_model.pth") in r0
    assert any(re.fullmatch(r"iter_\d+_dice_[\d.]+\.pth", os.path.basename(f)) for f in r0)
    assert _files(tmp_path / "rank1") == [] and not os.path.exists(tmp_path / "rank1" / "model")
    assert (tmp_path / "validator0.txt").read_text() == "2" and (tmp_path / "validator1.txt").read_text() == "0"
    # the one-process run fed rank 0's inputs writes the same lines
    FakeValidator.calls = []
    _train_in(str(tmp_path / "single" / "code"), ARGV)
    got = [_strip(l) for l in (tmp_path / "rank0" / snap / "log.txt").read_text().splitlines()]
    want = [_strip(l) for l in (tmp_path / "single" / snap / "log.txt").read_text().splitlines()]
    assert got == want and len(got) == 1 + 1 + 450 + 2
    assert got[1] == "7 iterations per epoch" and got[2] == "iteration 1 : loss : %f, loss_ce: %f" % (1.0, 0.5)
    assert _files(tmp_path / "rank0") == _files(tmp_path / "single")


def test_trainer_rank_other_than_0_writes_and_validates_nothing(tmp_path):
    recipe = T.Recipe((), "single", None, T._LOG2, (("info/loss_ce", T._part("ce")),))
    args = argparse.Namespace(max_iterations=420, base_lr=0.01, num_classes=4, model="unet")
    lines, val = [], FakeValidator(None, None)
    FakeValidator.calls = []
    counter = iter(range(1, 10 ** 6))
    out = T.Trainer(args, recipe, torch.nn.Linear(2, 2), FakeStep(), lambda: ((next(counter),) for _ in range(5)), 5, val,
                    str(tmp_path), lines.append, device="cpu", rank=1).run()
    assert out == "Training Finished!" and next(counter) == 421
    assert lines == [] and FakeValidator.calls == [] and os.listdir(tmp_path) == []


# ---------------------------------------------------------------- the batch-size rule
def test_rank_batch():
    semi, s2l = "train_mean_teacher_2D.py", "train_s2l.py"
    assert T.rank_batch(SCRIPT, 24, 1) == 24 and T.rank_batch(semi, 12, 1) == 6 and T.rank_batch(semi, 13, 1) == 6
    assert T.rank_batch(SCRIPT, 128, 8) == 16 and T.rank_batch(s2l, 12, 4) == 3 and T.rank_batch(semi, 256, 8) == 16
    for script, bs, w in ((SCRIPT, 12, 8), (semi, 12, 4), (semi, 6, 2), (s2l, 12, 5)):
        with pytest.raises(ValueError, match=rf"--batch_size {bs} does not split over {w} ranks"):
            T.rank_batch(script, bs, w)


def test_indivisible_batch_raises_before_anything_is_built(tmp_path, monkeypatch):
    import torch.distributed as dist
    monkeypatch.setenv("WORLD_SIZE", "3")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.chdir(tmp_path)
    touched = []
    monkeypatch.setattr(T, "build", lambda *a, **k: touched.append("build"))
    monkeypatch.setattr(dist, "init_process_group", lambda *a, **k: touched.append("group"))
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a, **k: touched.append("device"))
    with pytest.raises(ValueError, match=r"--batch_size 8 does not split over 3 ranks"):
        T.train([SCRIPT, "--batch_size", "8"])
    with pytest.raises(ValueError, match=r"--batch_size 9 does not split over 3 ranks"):
        T.train(["train_deep_adversarial_network_2D.py", "--batch_size", "9"])
    assert touched == [] and os.listdir(tmp_path) == []


# ---------------------------------------------------------------- no torchrun environment: today's Namespace and loaders
class FakeStore:
    def __init__(self, n, scribbles=None):
        self.n, self.has4, self.scribbles = n, np.zeros(n, bool), scribbles
        self.names = [str(i) for i in range(n)]

    def __len__(self):
        return self.n


class FakeModel:
    def set_precision(self, p):
        self.precision = p


@pytest.mark.parametrize("script", ["train_weakly_supervised_segmentation_pCE_ours_proposed.py", "train_s2l.py",
                                    "train_uncertainty_aware_mean_teacher_2D.py"])
def test_no_torchrun_environment_gives_todays_namespace_and_loaders(script, monkeypatch):
    from wsl4mis_b200.ddp import env_world
    import wsl4mis_b200.networks.net_factory as NF
    for v in TORCHRUN_VARS:
        monkeypatch.delenv(v, raising=False)
    assert env_world() == (0, 0, 1)
    argv = ["--root_path", "synthetic:10", "--batch_size", "12"]
    name, args, precision = T.parse([script] + argv)
    assert str(args) == str(T.parser_for(script).parse_args(argv)) and precision == "bf16"
    monkeypatch.setattr(D.SliceStore, "from_arrays", classmethod(lambda cls, ims, labs, names=None, device=None, scribbles=None:
                                                                  FakeStore(len(ims), scribbles)))
    monkeypatch.setattr(NF, "net_factory", lambda **kw: FakeModel())
    seen = []
    monkeypatch.setitem(T.RECIPES, script, T.RECIPES[script]._replace(step=lambda a, m, w: seen.append(w) or FakeStep()))
    model, step, batches, n, refresh = T.build(name, args, precision)
    assert seen == [1] and model.precision == "bf16" and (refresh is not None) == (script == "train_s2l.py")
    if script == "train_uncertainty_aware_mean_teacher_2D.py":
        from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets as Semi
        n_l = len(Semi(base_dir="synthetic:10", labeled_type="labeled", fold=args.fold))
        assert n == -(-n_l // 6)                  # DataLoader(batch_size=batch_size // 2) over the labelled slices
    else:
        sets = D.BaseDataSets(base_dir="synthetic:10", split="train", fold=args.fold)
        assert n == -(-len(sets) // 12)


# ---------------------------------------------------------------- the loaders' partition and draws
@pytest.mark.parametrize("n,bs,world", [(37, 4, 2), (40, 5, 2), (23, 3, 4)])
def test_rank_loaders_cover_the_permutation_as_distributed_sampler(n, bs, world):
    from torch.utils.data.distributed import DistributedSampler
    for cls in (D.GpuLoader, D.S2LLoader):
        store = FakeStore(n, scribbles=object())
        per_rank = []
        for r in range(world):
            torch.manual_seed(11)
            ld = cls(store, bs, rank=r, world_size=world)
            per_rank.append([list(b) for epoch in range(2) for b in ld._batches()])
            assert len(per_rank[-1]) == 2 * len(ld) and all(len(b) <= bs for b in per_rank[-1])
        torch.manual_seed(11)
        for epoch in range(2):
            seed = int(torch.empty((), dtype=torch.int64).random_().item())
            g = torch.Generator()
            g.manual_seed(seed)
            order = torch.randperm(n, generator=g).tolist()
            for r in range(world):
                want = [order[i] for i in DistributedSampler(range(n), num_replicas=world, rank=r, shuffle=False)]
                got = [i for b in per_rank[r][epoch * len(per_rank[r]) // 2:(epoch + 1) * len(per_rank[r]) // 2] for i in b]
                assert got == want, (cls.__name__, epoch, r)
            assert set(i for r in range(world) for b in per_rank[r] for i in b) == set(range(n))


def test_rank_streams_differ_between_ranks_and_none_keeps_the_global_draws():
    draw = D.RandomGenerator.draw
    first = draw(True, D.rank_streams(2022, 0))               # a fresh pair of streams starts over
    s0, s1, s0b = D.rank_streams(2022, 0), D.rank_streams(2022, 1), D.rank_streams(2022, 0)
    d0, d1, d0b = ([draw(i % 3 == 0, s) for i in range(64)] for s in (s0, s1, s0b))
    assert d0 == d0b and d0 != d1 and first == d0[0]
    random.seed(5)
    np.random.seed(5)
    want = [draw(True) for _ in range(64)]
    random.seed(5)
    np.random.seed(5)
    assert [draw(True, None) for _ in range(64)] == want
    # the global streams are not consumed by rank streams
    random.seed(5)
    np.random.seed(5)
    [draw(True, s1) for _ in range(64)]
    assert [draw(True) for _ in range(64)] == want


def test_build_hands_each_rank_its_shard_and_its_own_streams(monkeypatch):
    import wsl4mis_b200.networks.net_factory as NF
    monkeypatch.setattr(D.SliceStore, "from_arrays", classmethod(lambda cls, ims, labs, names=None, device=None, scribbles=None:
                                                                  FakeStore(len(ims), scribbles)))
    monkeypatch.setattr(NF, "net_factory", lambda **kw: FakeModel())
    made = []
    orig = D.GpuLoader.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        made.append(self)
    monkeypatch.setattr(D.GpuLoader, "__init__", init)
    script = "train_deep_adversarial_network_2D.py"
    monkeypatch.setitem(T.RECIPES, script, T.RECIPES[script]._replace(step=lambda a, m, w: FakeStep()))
    name, args, precision = T.parse([script, "--root_path", "synthetic:10", "--batch_size", "24"])
    draws = []
    for r in range(2):
        made.clear()
        T.build(name, args, precision, rank=r, world_size=2)
        assert [(l.rank, l.world_size, l.batch_size) for l in made] == [(r, 2, 6), (r, 2, 6)]
        assert made[0].streams is made[1].streams          # one per-rank stream shared by both streams of the feed
        draws.append([D.RandomGenerator.draw(False, made[0].streams) for _ in range(32)])
    assert draws[0] != draws[1]
