"""The test step's host side (wsl4mis_b200/test_2D.py) against test_2D_fully.py / test_2D_fully_sps.py: fold split, flags, the
checkpoint / prediction / original-image paths, the spacing order, and the synthetic stand-in's spacing stream."""
import argparse
import ast
import hashlib
import sys

import numpy as np
import pytest

import wsl4mis_b200.test_2D as T     # the module, not its names: pytest would collect test_single_volume
from wsl4mis_b200 import nifti
from wsl4mis_b200.dataloaders.dataset import synthetic_acdc, synthetic_spacing

import stage_test


def _staged_script(name):
    """the staged script's parser and get_fold_ids, executed from its source (its imports need h5py, SimpleITK, medpy)"""
    src = stage_test.read(name)
    if src is None:
        pytest.skip("reference test scripts not staged (run oracle/stage_test.py where the reference exists)")
    tree = ast.parse(src)
    keep = []
    for node in tree.body:
        src = ast.unparse(node)
        if src.startswith("parser") or (isinstance(node, ast.FunctionDef) and node.name == "get_fold_ids"):
            keep.append(node)
    ns = {"argparse": argparse}
    exec(compile(ast.Module(body=keep, type_ignores=[]), name, "exec"), ns)
    return ns


def _actions(p):
    return {a.dest: (a.option_strings, a.type, a.default, a.help) for a in p._actions if a.dest != "help"}


def test_fold_ids():
    for k in range(1, 6):
        train, test = T.get_fold_ids(f"fold{k}")
        assert test == ["patient{:0>3}".format(i) for i in range(20 * (k - 1) + 1, 20 * k + 1)]
        assert len(train) == 80 and not set(train) & set(test) and sorted(train + test) == ["patient{:0>3}".format(i) for i in range(1, 101)]
        assert train == sorted(train)
    assert T.get_fold_ids("fold6") == "ERROR KEY"


def test_flags_and_folds_match_the_staged_scripts():
    ref = _staged_script("test_2D_fully.py")
    assert _actions(T.parser) == _actions(ref["parser"])
    argv = ["--root_path", "/d/ACDC", "--exp", "ACDC/x", "--model", "unet_cct", "--fold", "fold2", "--num_classes", "4",
            "--sup_type", "label"]
    assert vars(T.parser.parse_args(argv)) == vars(ref["parser"].parse_args(argv))
    for f in ("fold1", "fold2", "fold3", "fold4", "fold5", "fold7"):
        assert T.get_fold_ids(f) == ref["get_fold_ids"](f)
    # the _sps script has the same flags; only the defaults of --exp and --model differ
    sps = _actions(_staged_script("test_2D_fully_sps.py")["parser"])
    ours = _actions(T.parser)
    assert sps.keys() == ours.keys()
    assert {k for k in ours if ours[k] != sps[k]} == {"exp", "model"}
    assert sps["model"][2] == "unet_cct"


def test_paths_follow_the_script(tmp_path, monkeypatch):
    F = T.parser.parse_args(["--exp", "ACDC/pCE", "--fold", "fold3", "--sup_type", "scribble", "--model", "unet_cct"])
    assert T.checkpoint_path(F) == "../model/ACDC/pCE_fold3/scribble/iter_60000.pth"
    assert T.predictions_dir(F) == "../model/ACDC/pCE_fold3/scribble/unet_cct_predictions/"
    # Inference removes and recreates the prediction directory before it builds the network
    work = tmp_path / "work"
    work.mkdir()
    monkeypatch.chdir(work)
    pred_dir = tmp_path / "model" / "ACDC" / "pCE_fold3" / "scribble" / "unet_cct_predictions"
    pred_dir.mkdir(parents=True)
    (pred_dir / "stale_pred.nii.gz").write_bytes(b"x")

    class Stop(Exception):
        pass

    def no_net(**kw):
        assert kw == {"net_type": "unet_cct", "in_chns": 1, "class_num": 4}
        raise Stop

    import wsl4mis_b200.networks.net_factory as NF
    monkeypatch.setattr(NF, "net_factory", no_net)
    F.root_path = "synthetic:3"
    with pytest.raises(Stop):
        T.Inference(F)
    assert pred_dir.is_dir() and not any(pred_dir.iterdir())


def test_original_image_is_read_relative_to_the_working_directory(tmp_path, monkeypatch):
    work = tmp_path / "work"
    work.mkdir()
    monkeypatch.chdir(work)
    with pytest.raises(FileNotFoundError) as e:
        T.original_path("patient001_frame01", str(tmp_path / "data" / "ACDC"))
    assert e.value.filename == "../data/ACDC_training/patient001_frame01.nii.gz"
    assert "../data/ACDC_training/patient001_frame01.nii.gz" in str(e.value)
    (tmp_path / "data" / "ACDC_training").mkdir(parents=True)
    nifti.write(str(tmp_path / "data" / "ACDC_training" / "patient001_frame01.nii.gz"), np.zeros((2, 3, 4)),
                nifti.header((2, 3, 4), (1.5, 1.25, 10.0)))
    path = T.original_path("patient001_frame01", "/elsewhere/ACDC")
    assert path == "../data/ACDC_training/patient001_frame01.nii.gz"
    assert T.metric_spacing(nifti.read(path).spacing) == (10.0, 1.5, 1.25)    # (z, x, y): rows take the x spacing


def test_h5_volumes_need_h5py(monkeypatch):
    monkeypatch.setitem(sys.modules, "h5py", None)
    with pytest.raises(ImportError, match="h5py is required to read the ACDC files; pass base_dir='synthetic'"):
        T._read_volume("/data/ACDC", "patient001_frame01.h5")


def test_synthetic_volumes_and_their_originals():
    root = "synthetic:30"
    files = T._volume_files(root)
    assert files == [f"patient{i:03d}_frame01.h5" for i in range(1, 31)]
    cases = synthetic_acdc(30)
    img, lab = T._read_volume(root, "patient007_frame01.h5")
    assert np.array_equal(img, cases["patient007"][0]) and np.array_equal(lab, cases["patient007"][1])
    path = T.original_path("patient007_frame01", root, img)
    org = nifti.read(path)
    assert org.spacing == tuple(float(np.float32(s)) for s in synthetic_spacing("patient007"))
    assert np.array_equal(org.array, img)
    assert T.original_path("patient007_frame01", root, img) == path          # written once


def test_synthetic_spacing_stream():
    sp = [synthetic_spacing(f"patient{i:03d}") for i in range(1, 101)]
    assert sp == [synthetic_spacing(f"patient{i:03d}_frame01") for i in range(1, 101)]       # deterministic, keyed by patient
    assert all(x in (1.25, 1.37, 1.5625) and y in (1.25, 1.37, 1.5625) and z in (5.0, 6.5, 10.0) for x, y, z in sp)
    assert len(set(sp)) > 10 and any(x != y for x, y, _ in sp)
    assert synthetic_spacing("patient001") == (1.5625, 1.25, 6.5)


def test_synthetic_acdc_is_unchanged():
    """the spacing stream draws nothing from synthetic_acdc's generator: its volumes are the same bytes as before"""
    c = synthetic_acdc(100)
    h = hashlib.sha256()
    for p in sorted(c):
        for a in c[p]:
            h.update(a.tobytes())
    assert h.hexdigest() == "c8e6015740394bd0bd6b91375a323565424b75f796c6e2b4d38c8dc4add289e1"
