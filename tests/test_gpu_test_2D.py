"""The GPU test step (wsl4mis_b200/test_2D.py) against the reference's per-slice loop (test_2D_fully.py:83-124) restated with scipy
zoom, batch-1 forwards and torch.softmax + argmax, and its metrics against the scipy restatement of medpy (_metric_oracle.py) at the
reference's spacing order; Inference end to end on a trained network; chunked inference against one batch."""
import gc
import os

import numpy as np
import pytest
import torch
from scipy.ndimage import zoom

import _metric_oracle as M

pytestmark = pytest.mark.gpu
DEV = "cuda"

if torch.cuda.is_available():
    import wsl4mis_b200.test_2D as T     # the module, not its names: pytest would collect test_single_volume
    from wsl4mis_b200 import nifti
    from wsl4mis_b200.dataloaders.dataset import GpuLoader, SliceStore, fold_ids, synthetic_acdc
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT

ROOT = "synthetic:100"
SHAPES = [(256, 216), (216, 256), (224, 154), (232, 256), (174, 208)]


@pytest.fixture(scope="module")
def trained():
    """state_dict of a UNet after 300 ce_dice steps (batch 12) on fold 1's training slices of synthetic:100: a network that
    predicts every class, as a trained checkpoint does"""
    cases = synthetic_acdc(100)
    train, _ = fold_ids("fold1")
    ims = [im for p in sorted(cases) if p in train for im in cases[p][0]]
    labs = [lb for p in sorted(cases) if p in train for lb in cases[p][1]]
    torch.manual_seed(0)
    net = UNet(1, 4).to(DEV)
    step = TrainStep(net, "ce_dice", graph=False)
    loader, done = GpuLoader(SliceStore.from_arrays(ims, labs, device=DEV), 12, drop_last=True), 0
    while done < 300:
        for batch in loader:
            step(batch["image"], batch["label"])
            done += 1
            if done == 300:
                break
    torch.cuda.synchronize()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    del net, step
    gc.collect()
    return sd


def _net(sd, cct, precision):
    """the trained UNet, or a UNet_CCT whose main decoder carries its decoder (aux decoder at its initialisation)"""
    torch.manual_seed(1)
    net = (UNet_CCT if cct else UNet)(1, 4)
    if cct:
        full = net.state_dict()
        full.update({k.replace("decoder.", "main_decoder.", 1) if k.startswith("decoder.") else k: v for k, v in sd.items()})
        sd = full
    net.load_state_dict(sd)
    return net.to(DEV).set_precision(precision).eval()


def _reference_loop(image, net):
    """test_2D_fully.py:89-102 (test_2D_fully_sps.py:97-100 for dual-head nets): label map and the top-2 logit margin behind
    every pixel"""
    S, x, y = image.shape
    prediction = np.zeros(image.shape, np.uint8)
    margin = np.zeros(image.shape, np.float32)
    for ind in range(S):
        sl = zoom(image[ind], (256 / x, 256 / y), order=0)
        inp = torch.from_numpy(sl).unsqueeze(0).unsqueeze(0).float().to(DEV)
        with torch.no_grad():
            out = net(inp)
            out = out[0] if isinstance(out, tuple) else out
            lab = torch.argmax(torch.softmax(out, dim=1), dim=1).squeeze(0).cpu().numpy()
            top2 = out[0].topk(2, dim=0).values
            mg = (top2[0] - top2[1]).cpu().numpy()
        prediction[ind] = zoom(lab, (x / 256, y / 256), order=0)
        margin[ind] = zoom(mg, (x / 256, y / 256), order=0)
    return prediction, margin


def _logit_error(image, net_a, net_b):
    """largest |logit difference| of the main heads of two networks on the 256x256 slices of `image`"""
    S, h, w = image.shape
    x = torch.from_numpy(np.stack([zoom(s, (256 / h, 256 / w), order=0) for s in image]))[:, None].to(DEV)
    with torch.no_grad():
        a, b = net_a(x), net_b(x)
    a, b = (a[0], b[0]) if isinstance(a, tuple) else (a, b)
    return (a - b).abs().max().item()


def _cases_of_every_shape():
    cases = synthetic_acdc(100)
    pick = {}
    for p in sorted(cases):
        pick.setdefault(cases[p][0].shape[1:], p)
    assert sorted(pick) == sorted(SHAPES)
    return [(pick[s], cases[pick[s]]) for s in SHAPES]


def _flags(**kw):
    F = T.parser.parse_args(["--root_path", ROOT])
    for k, v in kw.items():
        setattr(F, k, v)
    return F


def _check_metrics(got, pred, label, case):
    sp = T.metric_spacing(nifti.read(T.original_path(case, ROOT)).spacing)
    assert sp[1] != sp[0]                 # anisotropic: slice distance vs in-plane
    for k in range(1, 4):
        ref = (M.dc(pred == k, label == k), M.hd95(pred == k, label == k, sp), M.asd(pred == k, label == k, sp))
        for g, r in zip(got[k - 1], ref):
            assert abs(g - r) <= 1e-12 * abs(r), (case, k, got[k - 1], ref)


@pytest.mark.parametrize("cct", [False, True])
def test_volume_parity_with_the_reference_loop(trained, tmp_path, cct):
    """fp16x3 (fp32-accurate): the same label map as the per-slice loop.  bf16: the differing pixels are reported, those above a
    1e-3 fp16x3 top-2 margin too; bf16 storage moves logits by more than that (a few hundredths), so the map must be identical
    wherever the margin exceeds twice the measured largest logit difference, where no rounding can flip the argmax.  Metrics
    equal the scipy restatement of medpy on the map test_single_volume wrote."""
    ref_net = _net(trained, cct, "fp16x3")
    bf_net = _net(trained, cct, "bf16")
    F = _flags(model="unet_cct" if cct else "unet")
    report = []
    for pid, (image, label, _) in _cases_of_every_shape():
        case = f"{pid}_frame01"
        ref, margin = _reference_loop(image, ref_net)
        for precision, net in (("fp16x3", ref_net), ("bf16", bf_net)):
            out = tmp_path / precision
            out.mkdir(exist_ok=True)
            got = T.test_single_volume(case + ".h5", net, str(out) + "/", F)
            pred = nifti.read(str(out / f"{case}_pred.nii.gz")).array.astype(np.uint8)
            assert np.array_equal(pred, T.predict_volume(image, net).cpu().numpy())
            _check_metrics(got, pred, label, case)
            diff = pred != ref
            if precision == "fp16x3":
                assert not diff.any(), (case, int(diff.sum()))
            else:
                err = _logit_error(image, ref_net, bf_net)
                report.append((case, int(diff.sum()), int((diff & (margin > 1e-3)).sum()), pred.size, round(err, 4),
                               float(margin[diff].max()) if diff.any() else 0.0))
                assert not (diff & (margin > 2 * err)).any(), report[-1]
    print("bf16 vs the per-slice fp16x3 loop (case, differing pixels, of them with margin > 1e-3, pixels, max |logit diff|, "
          "largest margin at a differing pixel):", report)


def test_empty_class_raises_with_case_and_class(trained, tmp_path):
    sd = dict(trained)
    b = sd["decoder.out_conv.bias"].clone()
    b[3] = -1e4                            # class 3 never wins the argmax
    sd["decoder.out_conv.bias"] = b
    net = _net(sd, False, "bf16")
    with pytest.raises(RuntimeError) as e:
        T.test_single_volume("patient001_frame01.h5", net, str(tmp_path) + "/", _flags())
    msg = str(e.value)
    assert msg.startswith("The first supplied array does not contain any binary object.")
    assert "patient001_frame01" in msg and "class 3" in msg
    z = np.zeros((2, 8, 8), bool)
    o = z.copy()
    o[:, 2:5, 2:5] = True
    with pytest.raises(RuntimeError, match="^The first supplied array does not contain any binary object"):
        T.calculate_metric_percase(z, o, (5.0, 1.0, 1.0))
    with pytest.raises(RuntimeError, match="^The second supplied array does not contain any binary object"):
        T.calculate_metric_percase(o, z, (5.0, 1.0, 1.0))
    d, h, a = T.calculate_metric_percase(o, o, (5.0, 1.0, 1.0))
    assert (d, h, a) == (1.0, 0.0, 0.0)


def _save_checkpoint(sd, tmp_path, folds, exp="ACDC/e2e", sup="label"):
    for f in folds:
        d = tmp_path / "model" / f"{exp}_{f}" / sup
        d.mkdir(parents=True, exist_ok=True)
        torch.save(sd, str(d / "iter_60000.pth"))


def test_inference_end_to_end(trained, tmp_path, monkeypatch, capsys):
    _save_checkpoint(trained, tmp_path, ["fold1"])
    (tmp_path / "work").mkdir()
    monkeypatch.chdir(tmp_path / "work")
    F = T.parser.parse_args(["--root_path", ROOT, "--exp", "ACDC/e2e", "--fold", "fold1", "--sup_type", "label"])
    mean_dice = T.Inference(F)
    printed = capsys.readouterr().out
    assert "init weight from ../model/ACDC/e2e_fold1/label/iter_60000.pth" in printed
    # the same volumes, scored one by one with the checkpoint's network
    net = _net(torch.load("../model/ACDC/e2e_fold1/label/iter_60000.pth"), False, "bf16")
    cases = synthetic_acdc(100)
    names = [f"patient{i:03d}_frame01" for i in range(1, 21)]
    check = tmp_path / "check"
    check.mkdir()
    per_case = [T.test_single_volume(c + ".h5", net, str(check) + "/", F) for c in names]
    totals = [sum(np.asarray(m[k]) for m in per_case) / len(names) for k in range(3)]
    assert mean_dice == ((totals[0] + totals[1] + totals[2]) / 3)[0]
    assert 0.3 < mean_dice <= 1.0
    out = tmp_path / "model" / "ACDC" / "e2e_fold1" / "label" / "unet_predictions"
    assert sorted(os.listdir(out)) == sorted(f"{c}_{s}.nii.gz" for c in names for s in ("pred", "img", "gt"))
    for c in names:
        pid = c.split("_")[0]
        org = nifti.read(T.original_path(c, ROOT))
        pred = nifti.read(str(out / f"{c}_pred.nii.gz"))
        assert np.array_equal(pred.array, T.predict_volume(cases[pid][0], net).cpu().numpy().astype(np.float32))
        assert np.array_equal(nifti.read(str(out / f"{c}_img.nii.gz")).array, cases[pid][0])
        assert np.array_equal(nifti.read(str(out / f"{c}_gt.nii.gz")).array, cases[pid][1].astype(np.float32))
        for s in ("pred", "img", "gt"):
            h = nifti.read(str(out / f"{c}_{s}.nii.gz")).header
            assert all(h[k] == org.header[k] for k in nifti.GEOMETRY), (c, s)


@pytest.mark.parametrize("cct", [False, True])
def test_chunked_equals_one_batch(trained, cct):
    """The forward's per-pixel arithmetic does not depend on the batch size: the logits of a slice are the same bits in a
    batch of 1, of S and in a padded chunk of 16; so are the label maps for any chunk size."""
    net = _net(trained, cct, "bf16")
    pid, (image, _, _) = _cases_of_every_shape()[3]
    S, h, w = image.shape
    x = torch.from_numpy(np.stack([zoom(s, (256 / h, 256 / w), order=0) for s in image]))[:, None].to(DEV)
    with torch.no_grad():
        head = (lambda o: o[0] if isinstance(o, tuple) else o)
        whole = head(net(x)).clone()
        padded = head(net(torch.cat([x, torch.zeros(16 - S, 1, 256, 256, device=DEV)]))).clone()
        singles = torch.cat([head(net(x[i:i + 1])).clone() for i in range(S)])
    assert torch.equal(padded[:S], whole) and torch.equal(singles, whole)
    one = T.predict_volume(image, net, chunk=S)
    for chunk in (16, 4, 3, 1):
        assert torch.equal(T.predict_volume(image, net, chunk=chunk), one), chunk


def test_five_fold_pass_keeps_the_first_volumes_memory(trained, tmp_path, monkeypatch, capsys):
    _save_checkpoint(trained, tmp_path, [f"fold{k}" for k in range(1, 6)])
    (tmp_path / "work").mkdir()
    monkeypatch.chdir(tmp_path / "work")
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    seen = []
    inner = T.test_single_volume

    def counted(*a, **k):
        r = inner(*a, **k)
        torch.cuda.synchronize()
        seen.append(torch.cuda.max_memory_reserved())
        return r

    monkeypatch.setattr(T, "test_single_volume", counted)
    total = T.main(["--root_path", ROOT, "--exp", "ACDC/e2e", "--sup_type", "label"])
    capsys.readouterr()
    print(f"peak reserved after the first volume {seen[0] / 2**20:.1f} MiB, after {len(seen)} volumes "
          f"{torch.cuda.max_memory_reserved() / 2**20:.1f} MiB; mean Dice of the five folds {total:.4f}")
    assert len(seen) == 100
    assert torch.cuda.max_memory_reserved() == seen[0], [s / 2**20 for s in seen]
