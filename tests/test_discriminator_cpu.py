"""FCDiscriminator and dataset_semi on the host: the CPU oracle against the unmodified reference (tests/golden/fcdisc.npz), the
space-to-depth plan against F.conv2d(stride=2, padding=1) in fp64, the module's state_dict surface and the labelled / unlabelled split
of dataloaders.dataset_semi."""
import inspect
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dan_oracle as D


def _fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "fcdisc.npz"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_oracle_matches_reference_fixture(golden_dir, dtype, mode):
    z = _fixture(golden_dir)
    n, pseed, iseed, kseed, stride = (int(v) for v in z["seeds"])
    p = {k: v.to(dtype).requires_grad_(True) for k, v in D.synth_params(pseed, dtype=torch.float64).items()}
    mp, feat = (t.to(dtype).requires_grad_(True) for t in D.synth_inputs(iseed, n, dtype=torch.float64))
    logits = D.forward(p, mp, feat, mode == "train", D.chan_keep(kseed, n))
    F.cross_entropy(logits, torch.tensor([1, 0])).backward()
    ref = torch.from_numpy(z[mode + "/logits"]).double()
    assert (logits.detach().double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    for name, g in (("dmap", mp.grad), ("dfeat", feat.grad)):
        r = torch.from_numpy(z[f"{mode}/{name}"]).double()
        got = g[:, :, ::stride, ::stride].double()
        assert (got - r).abs().max().item() <= 2e-4 * r.abs().max().item(), name
    for k, v in p.items():
        for stat, fn in (("gnorm", lambda t: t.norm()), ("gabs", lambda t: t.abs().sum())):
            r = float(z[f"{mode}/{stat}/{k}"])
            assert abs(fn(v.grad.double()).item() - r) <= 2e-4 * r, (k, stat)


@pytest.mark.parametrize("N,C,Cout,H", [(2, 5, 16, 8), (1, 3, 7, 12), (3, 16, 32, 6), (2, 1, 4, 16)])
def test_space_to_depth_plan_equals_strided_conv(N, C, Cout, H):
    g = torch.Generator().manual_seed(N * 1000 + C * 10 + H)
    x = torch.randn(N, C, H, H + 2, dtype=torch.float64, generator=g)
    w = torch.randn(Cout, C, 4, 4, dtype=torch.float64, generator=g)
    b = torch.randn(Cout, dtype=torch.float64, generator=g)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, b, stride=2, padding=1)
    dy = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    ref.backward(dy)
    scale = ref.abs().max().item()
    assert (D.s2d_conv(x, w, b) - ref).abs().max().item() <= 1e-12 * scale
    assert (D.s2d_conv_input_grad(dy, w, C) - xr.grad).abs().max().item() <= 1e-12 * xr.grad.abs().max().item()
    assert (D.s2d_conv_weight_grad(x, dy) - wr.grad).abs().max().item() <= 1e-12 * wr.grad.abs().max().item()


def test_space_to_depth_packers_round_trip():
    x = torch.arange(2 * 3 * 4 * 6, dtype=torch.float64).reshape(2, 3, 4, 6)
    t = D.s2d(x, 16)
    assert t.shape == (2, 2, 3, 16) and not t[..., 12:].any()
    assert t[1, 1, 2, (1 * 2 + 0) * 3 + 2].item() == x[1, 2, 3, 4].item()        # T[n, Y, X, (a*2+b)*C + c] = x[n, c, 2Y+a, 2X+b]
    assert torch.equal(D.d2s(t, 3), x)
    w = torch.randn(5, 3, 4, 4, dtype=torch.float64)
    w3 = D.scatter(w, 16)
    assert int((w3 != 0).sum()) == w.numel() and torch.equal(D.gather(w3, 3), w)


def test_module_surface_matches_reference(golden_dir):
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    z = _fixture(golden_dir)
    torch.manual_seed(0)
    m = FCDiscriminator(4)
    sd = m.state_dict()
    assert list(sd.keys()) == [str(k) for k in z["keys"]] == list(D.param_shapes())
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(int(s) for s in z["shape/" + k]) == D.param_shapes()[k], k
        assert v.double().sum().item() == float(z["init_sum/" + k]), k            # the reference's seeded initialisation, bit for bit
        assert v.double().abs().sum().item() == float(z["init_abs/" + k]), k
    assert list(inspect.signature(FCDiscriminator).parameters) == ["num_classes", "ndf", "n_channel"]
    assert [p.dtype for p in m.parameters()] == [torch.float32] * 12
    m.eval()
    assert not m.dropout.training
    m.train()
    assert m.dropout.training


def test_module_rejects_unsupported_inputs():
    from wsl4mis_b200.networks.discriminator import FCDiscriminator
    m = FCDiscriminator(4)
    with pytest.raises(TypeError, match="CUDA"):
        m(torch.zeros(1, 4, 256, 256), torch.zeros(1, 1, 256, 256))
    with pytest.raises(ValueError):
        m.set_precision("fp16")
    with pytest.raises(ValueError):
        FCDiscriminator(4, ndf=24)


@pytest.mark.parametrize("fold", ["fold1", "fold2", "fold3", "fold4", "fold5"])
def test_dataset_semi_split(fold):
    from wsl4mis_b200.dataloaders.dataset import BaseDataSets as Base, fold_ids
    from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets
    lab = BaseDataSets(base_dir="synthetic:100", num=4, labeled_type="labeled", fold=fold, split="train")
    unl = BaseDataSets(base_dir="synthetic:100", num=4, labeled_type="unlabeled", fold=fold, split="train")
    train, test = fold_ids(fold)
    want_lab = [f"patient{10 * i:03d}" for i in range(1, 11) if f"patient{10 * i:03d}" in train]
    assert len(want_lab) == 8
    pl = sorted({c.split("_")[0] for c in lab.sample_list})
    pu = sorted({c.split("_")[0] for c in unl.sample_list})
    assert pl == want_lab
    assert pu == sorted(set(train) - set(want_lab))
    assert sorted(lab.sample_list + unl.sample_list) == sorted(Base("synthetic:100", "train", None, fold).sample_list)
    val = BaseDataSets(base_dir="synthetic:100", fold=fold, split="val")
    assert sorted(c.split("_")[0] for c in val.sample_list) == test


def test_dataset_semi_signature_and_samples():
    from wsl4mis_b200.dataloaders import dataset, dataset_semi
    from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets, RandomGenerator, TwoStreamBatchSampler
    assert list(inspect.signature(BaseDataSets).parameters) == ["base_dir", "num", "labeled_type", "split", "transform", "fold",
                                                                "sup_type"]
    assert RandomGenerator is dataset.RandomGenerator and TwoStreamBatchSampler is dataset.TwoStreamBatchSampler
    assert issubclass(BaseDataSets, dataset.BaseDataSets)
    a = BaseDataSets(base_dir="synthetic:40", num=4, labeled_type="labeled", fold="fold2", split="train")
    b = BaseDataSets(base_dir="synthetic:40", num=1000, labeled_type="labeled", fold="fold2", split="train")
    assert a.sample_list == b.sample_list                                   # num is ignored
    ds = BaseDataSets(base_dir="synthetic:40", labeled_type="labeled", fold="fold2", split="train", transform=RandomGenerator([64, 64]))
    s = ds[0]
    assert set(s) == {"image", "label", "idx"} and s["idx"] == ds.sample_list[0].split("_")[0] == "patient010"
    assert tuple(s["image"].shape) == (1, 64, 64) and tuple(s["label"].shape) == (64, 64)
    v = BaseDataSets(base_dir="synthetic:40", fold="fold2", split="val")[0]
    assert set(v) == {"image", "label", "idx"} and v["image"].ndim == 3 and v["idx"] == "patient021"
    assert dataset_semi.LABELED_IDS[0] == "patient010" and dataset_semi.LABELED_IDS[-1] == "patient100"
