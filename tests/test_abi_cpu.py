"""CPU-side checks of the C-ABI boundary: the library builds/loads and exports every symbol that
include/wsl4mis_b200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import subprocess

import pytest

from wsl4mis_b200 import _build, _lib


@pytest.fixture(scope="module")
def lib_path():
    if not os.path.exists(_lib.LIB_PATH):
        _build.build()
    return _lib.LIB_PATH


def test_header_parses_and_names_are_prefixed():
    protos = _lib.parse_header()
    assert len(protos) >= 25
    assert all(n.startswith("wsl_") for n in protos)
    for must in ("wsl_softmax_pce_fwd", "wsl_gatedcrf_fwd", "wsl_conv_tc", "wsl_bn_stats", "wsl_sgd_step"):
        assert must in protos


def test_library_exports_every_declared_symbol(lib_path):
    dll = ctypes.CDLL(lib_path)
    for name in _lib.parse_header():
        assert hasattr(dll, name), f"{name} declared in include/wsl4mis_b200.h but not exported"


def test_no_undeclared_exports(lib_path):
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if " T " in ln and ln.split()[-1].startswith("wsl_")}
    declared = set(_lib.parse_header())
    assert exported == declared, (exported - declared, declared - exported)


def test_abi_version_and_workspace(lib_path):
    dll = _lib.LIB.load()
    assert dll.wsl_abi_version() == 2
    assert dll.wsl_workspace_floats() >= 1 << 16


def test_product_path_has_no_oracle_import():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for dp, _, files in os.walk(os.path.join(root, "wsl4mis_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "wsl_oracle" not in src and "import oracle" not in src, f"{f} must not use the oracle"


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    fresh = _lib._Lib()
    with pytest.raises(RuntimeError, match="no CPU"):
        fresh.load()


def test_state_dict_layout_matches_oracle_key_order():
    import torch  # noqa
    import wsl_oracle as O
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT
    assert list(UNet(1, 4).state_dict().keys()) == list(O.unet_param_shapes(1, 4, ("decoder",)).keys())
    sd = UNet_CCT(1, 4).state_dict()
    shapes = O.unet_param_shapes(1, 4, ("main_decoder", "aux_decoder1"))
    assert list(sd.keys()) == list(shapes.keys())
    assert all(tuple(sd[k].shape) == tuple(shapes[k]) for k in sd)
    assert len(sd) == 202


def test_ramps():
    from wsl4mis_b200.utils import ramps
    assert ramps.sigmoid_rampup(0, 10) == pytest.approx(0.006737947, rel=1e-6)
    assert ramps.sigmoid_rampup(10, 10) == 1.0 and ramps.sigmoid_rampup(5, 0) == 1.0
    assert ramps.linear_rampup(5, 10) == 0.5 and ramps.cosine_rampdown(0, 10) == 1.0


def test_dropin_shim_exposes_the_reference_module_names():
    """`dropin/` ahead of the reference's code/ on PYTHONPATH gives the scripts' own import lines the H100 modules
    (train_weakly_supervised_pCE_GatedCRFLoss_2D.py:23-28)."""
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "utils" or k.startswith("utils.") or k == "networks" or k.startswith("networks.")}
    sys.path.insert(0, os.path.join(root, "dropin"))
    try:
        nf = importlib.import_module("networks.net_factory")
        un = importlib.import_module("networks.unet")
        lo = importlib.import_module("utils.losses")
        cr = importlib.import_module("utils.gate_crf_loss")
        ra = importlib.import_module("utils.ramps")
        assert callable(nf.net_factory)
        for name in ("ConvBlock", "DownBlock", "UpBlock", "Encoder", "Decoder", "UNet", "UNet_CCT", "UNet_DS", "UNet_CCT_3H",
                     "Decoder_DS", "Decoder_URDS", "Dropout", "FeatureDropout", "FeatureNoise"):
            assert hasattr(un, name), name
        for name in ("pDLoss", "DiceLoss", "MumfordShah_Loss", "entropy_loss", "softmax_mse_loss", "entropy_minmization",
                     "symmetric_mse_loss", "dice_loss"):
            assert hasattr(lo, name), name
        assert hasattr(cr, "ModelLossSemsegGatedCRF") and hasattr(ra, "sigmoid_rampup")
    finally:
        sys.path.remove(os.path.join(root, "dropin"))
        for k in [k for k in sys.modules if k == "utils" or k.startswith("utils.") or k == "networks" or k.startswith("networks.")]:
            sys.modules.pop(k)
        sys.modules.update(saved)


def test_unet_ds_state_dict_layout_matches_the_reference_order():
    """UNet_DS registers up1..up4, out_conv, out_conv_dp4..dp1 like networks/unet.py:138-168 (key order pinned through the
    oracle's shape table, itself checked against the reference module in oracle/make_golden.py:heads_golden)."""
    import torch
    from wsl4mis_b200.networks.unet import UNet_DS
    import wsl_oracle as O
    m = UNet_DS(1, 4)
    want = O.unet_param_shapes(1, 4, ("decoder",), ds=True)
    sd = m.state_dict()
    assert list(sd.keys()) == list(want.keys())
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in want.items())
    p = O.synth_params(1, 4, ("decoder",), 3, ds=True)
    m.load_state_dict(p)
    assert torch.equal(m.state_dict()["decoder.out_conv_dp4.weight"], p["decoder.out_conv_dp4.weight"])


def test_unet_cct_3h_and_urds_state_dict_layouts():
    """UNet_CCT_3H registers encoder, main_decoder, aux_decoder1, aux_decoder2 (unet.py:358-361); Decoder_URDS is a constructible
    parameter container with Decoder_DS's keys (unet.py:191-225)."""
    import wsl_oracle as O
    from wsl4mis_b200.networks.unet import UNet_CCT_3H, Decoder_URDS, Decoder_DS, _params
    sd = UNet_CCT_3H(1, 4).state_dict()
    want = O.unet_param_shapes(1, 4, ("main_decoder", "aux_decoder1", "aux_decoder2"))
    assert list(sd.keys()) == list(want.keys()) and all(tuple(sd[k].shape) == tuple(v) for k, v in want.items())
    assert list(Decoder_URDS(_params(1, 4)).state_dict().keys()) == list(Decoder_DS(_params(1, 4)).state_dict().keys())


def test_pnet_state_dict_layout():
    """PNet2D registers block{1..5}.{conv1,conv2,in1,in2}, catblock.conv{1,2}, out.conv{1,2} like networks/pnet.py:16-110"""
    import wsl_oracle as O
    from wsl4mis_b200.networks.pnet import PNet2D
    sd = PNet2D(1, 4, 64, [1, 2, 4, 8, 16]).state_dict()
    want = O.pnet_param_shapes(1, 4)
    assert list(sd.keys()) == list(want.keys()) and all(tuple(sd[k].shape) == tuple(v) for k, v in want.items())
