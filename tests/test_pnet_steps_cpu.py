"""--model pnet in the trainer without a GPU: the two combinations no step runs (PNet2D in fp32 mode, PNet2D under the two-output
pCE_ours_proposed recipe) raise ValueError before any CUDA call, and the executor attributes the training steps read."""
import pytest
import torch

import wsl4mis_b200.train as TR

DMPLS = "train_weakly_supervised_segmentation_pCE_ours_proposed.py"


@pytest.fixture()
def no_cuda(monkeypatch):
    """any CUDA initialisation, network or data construction fails the test"""
    def forbidden(*a, **k):
        raise AssertionError("reached CUDA / the model / the data")
    monkeypatch.setattr(torch.cuda, "_lazy_init", forbidden)
    monkeypatch.setattr(torch.cuda, "init", forbidden)
    monkeypatch.setattr(TR, "build", forbidden)
    monkeypatch.setattr(TR, "_train_logged", forbidden)


def test_pnet_in_fp32_mode_is_rejected(no_cuda):
    with pytest.raises(ValueError, match="bf16 / fp16 / fp16x3") as e:
        TR.train(["train_weakly_supervised_pCE_2D.py", "--model", "pnet", "--precision", "fp32"])
    assert "--precision fp32" in str(e.value)


def test_pnet_under_the_two_output_recipe_is_rejected(no_cuda):
    with pytest.raises(ValueError, match="two outputs"):
        TR.train([DMPLS, "--model", "pnet"])
    with pytest.raises(ValueError, match="two outputs"):
        TR.parse([DMPLS, "--model", "pnet", "--precision", "fp16"])


@pytest.mark.parametrize("script", sorted(s for s in TR.RECIPES if s != DMPLS))
@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16x3"])
def test_pnet_is_accepted_by_every_other_recipe(script, precision):
    name, args, prec = TR.parse([script, "--model", "pnet", "--precision", precision])
    assert (name, args.model, prec) == (script, "pnet", precision)
    TR.check_model(script, args, prec)


def test_the_other_models_keep_their_combinations():
    """the check concerns PNet2D only: unet_cct under the two-output recipe and unet in fp32 mode parse as before"""
    assert TR.parse([DMPLS])[1].model == "unet_cct"
    assert TR.parse(["train_weakly_supervised_pCE_2D.py", "--precision", "fp32"])[2] == "fp32"


def test_executor_step_contract():
    """what the steps read of an executor: the outputs of forward(), the parameters a single-head step skips and the bucket
    prefix the data-parallel overlap all-reduces after backward (None: no overlap)"""
    from wsl4mis_b200.networks.pnet import PNet2D
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT, UNet_CCT_3H, UNet_DS
    ex = PNet2D(1, 4, 64, [1, 2, 4, 8, 16]).executor
    assert (ex.n_outputs, ex.aux_param_ids, ex.comm_split, ex.sync_bn) == (1, set(), None, None)
    with pytest.raises(NotImplementedError, match="PNet2D"):
        ex.sync_bn = (2, None)
    for cls, n in ((UNet, 1), (UNet_CCT, 2), (UNet_DS, 4), (UNet_CCT_3H, 3)):
        m = cls(1, 4)
        e = m.executor
        assert e.n_outputs == n
        assert e.comm_split == sum(q.numel() for q in m.encoder.parameters())
        assert e.aux_param_ids == ({id(q) for q in m.aux_decoder1.parameters()} if cls is UNet_CCT else set())
