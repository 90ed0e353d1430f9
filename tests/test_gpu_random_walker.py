"""pCE + Random Walker on the H100: the batched random-walker solver (wsl_random_walker via random_walker_labels) against the exact
fp64 CPU solve of oracle/rw_oracle.py, the random-walker drop-in dataset, the ce_dice TrainStep variant
(train_fully_supervised_2D.py / train_weakly_supervised_pCE_random_walker_2D.py:97-105) and both reference scripts unchanged."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import rw_oracle as R
import wsl_oracle as O
from _gpu_util import chan_masks, cosine, elem_masks_nchw, ENC_MASK_KEYS  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [(256, 216), (216, 256), (224, 154), (232, 256), (174, 208)]      # synthetic_acdc's slice shapes


def _structure(h, w, seed):
    """an ACDC-like slice (nested rings, noisy intensities in [0, 1]) and its dense labels"""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cy, cx = h * (0.4 + 0.2 * rs.rand()), w * (0.4 + 0.2 * rs.rand())
    r0 = min(h, w) * (0.11 + 0.03 * rs.rand())
    rr = np.sqrt((yy - cy) ** 2 + ((xx - cx) * (0.9 + 0.2 * rs.rand())) ** 2)
    lab = np.zeros((h, w), np.uint8)
    lab[rr < 2.2 * r0] = 1
    lab[rr < 1.6 * r0] = 2
    lab[rr < 1.0 * r0] = 3
    img = 0.15 + 0.2 * lab + 0.08 * rs.randn(h, w)
    img = ((img - img.min()) / (img.max() - img.min())).astype(np.float32)
    return img, lab


def _arcs(lab, seed):
    """thin one-pixel arcs, one per class, covering ~90 degrees of the class's median radius (the hard case: few seeds)"""
    rs = np.random.RandomState(seed)
    scr = np.full(lab.shape, 4, np.uint8)
    for c in range(4):
        ys, xs = np.nonzero(lab == c)
        cy, cx = ys.mean(), xs.mean()
        rr = np.sqrt((ys - cy) ** 2 + (xs - cx) ** 2)
        ang = np.arctan2(ys - cy, xs - cx)
        sel = (np.abs(rr - np.median(rr)) < 0.5) & (((ang - rs.rand() * 2 * np.pi) % (2 * np.pi)) < 1.6)
        scr[ys[sel], xs[sel]] = c
    return scr


def _dots(lab, seed, frac=0.03):
    rs = np.random.RandomState(seed)
    keep = rs.rand(*lab.shape) < frac
    return np.where(keep, lab, 4).astype(np.uint8)


def _cases():
    """>= 8 ragged slices: arcs on the five shapes and on 428x512, random dots on two shapes, a slice without class 2 scribbles and
    one without background scribbles (F17)"""
    ims, scrs, kinds = [], [], []
    for i, (h, w) in enumerate(SHAPES + [(428, 512)]):
        img, lab = _structure(h, w, 10 + i)
        ims.append(img)
        scrs.append(_arcs(lab, 20 + i))
        kinds.append("arcs")
    for i, (h, w) in enumerate(SHAPES[:2]):
        img, lab = _structure(h, w, 40 + i)
        ims.append(img)
        scrs.append(_dots(lab, 50 + i))
        kinds.append("dots")
    img, lab = _structure(*SHAPES[2], 60)
    s = _dots(lab, 61)
    s[s == 2] = 4
    ims.append(img); scrs.append(s); kinds.append("missing")
    img, lab = _structure(*SHAPES[3], 62)
    s = _arcs(lab, 63)
    s[s == 0] = 4
    ims.append(img); scrs.append(s); kinds.append("nobg")
    return ims, scrs, kinds


@pytest.fixture(scope="module")
def solved():
    from wsl4mis_b200.dataloaders import random_walker_labels
    ims, scrs, kinds = _cases()
    names = [f"{k}{i}" for i, k in enumerate(kinds)]
    labels, stats = random_walker_labels(ims, scrs, probs=True, names=names)
    ref = [R.random_walker(im, sc) for im, sc in zip(ims, scrs)]
    return ims, scrs, kinds, names, labels, stats, ref


def test_every_slice_matches_the_exact_solve(solved):
    ims, scrs, kinds, names, labels, stats, ref = solved
    assert len(ims) >= 8
    worst = 0.0
    for i, (k, lab, (rl, rp)) in enumerate(zip(kinds, labels, ref)):
        assert stats["resid"][i] <= 1e-7, (names[i], stats["resid"][i])
        err = np.abs(stats["probs"][i] - rp).max()
        worst = max(worst, err)
        assert err <= 1e-4, (names[i], err)
        srt = np.sort(rp, -1)
        clear = (srt[..., -1] - srt[..., -2]) > 1e-3
        assert np.array_equal(lab[clear], rl[clear]), (names[i], int((lab != rl)[clear].sum()))
        print(f"{names[i]} {lab.shape}: {stats['iters'][i]} iterations, residual {stats['resid'][i]:.2e}, max |p - p_exact| {err:.2e}, "
              f"{int((lab != rl).sum())} labels differ (all within a 1e-3 margin)")
    it = np.asarray(stats["iters"])
    arcs = [i for i, k in enumerate(kinds) if k == "arcs"]
    dots = [i for i, k in enumerate(kinds) if k == "dots"]
    print(f"worst probability error {worst:.2e}; iterations arcs {it[arcs].tolist()}, dots {it[dots].tolist()}")


def test_missing_class_and_missing_background(solved):
    ims, scrs, kinds, names, labels, stats, ref = solved
    i = kinds.index("missing")
    assert not labels[i].any() and not stats["probs"][i].any() and stats["iters"][i] == 0
    j = kinds.index("nobg")
    seeds = scrs[j] < 4
    assert np.array_equal(labels[j][seeds], scrs[j][seeds] - 1)      # F17: classes 1..3 come out as 0..2
    assert labels[j].max() == 2 and not stats["probs"][j][..., 3].any()


def test_bit_identical_across_runs_and_batch_composition(solved):
    from wsl4mis_b200.dataloaders import random_walker_labels
    ims, scrs, kinds, names, labels, stats, ref = solved
    again, st2 = random_walker_labels(ims, scrs, probs=True)
    for a, b, pa, pb in zip(labels, again, stats["probs"], st2["probs"]):
        assert np.array_equal(a, b) and np.array_equal(pa, pb)
    assert np.array_equal(stats["iters"], st2["iters"]) and np.array_equal(stats["resid"], st2["resid"])
    k = kinds.index("arcs") + 2
    alone, st3 = random_walker_labels([ims[k]], [scrs[k]], probs=True)
    assert np.array_equal(alone[0], labels[k]) and np.array_equal(st3["probs"][0], stats["probs"][k])
    assert st3["iters"][0] == stats["iters"][k]


def test_max_iter_raises_and_names_the_slice():
    from wsl4mis_b200.dataloaders import random_walker_labels
    ims, scrs, kinds = _cases()
    with pytest.raises(RuntimeError, match="slab0"):
        random_walker_labels(ims[:2], scrs[:2], max_iter=5, names=["slab0", "slab1"])


def test_slice_store_round_trip_trains_with_gpu_loader():
    from wsl4mis_b200.dataloaders import random_walker_labels
    from wsl4mis_b200.dataloaders.dataset import GpuLoader, SliceStore
    ims, scrs, kinds = _cases()
    store = SliceStore.from_arrays(ims[:4], [np.zeros_like(s) for s in scrs[:4]], device=DEV, scribbles=scrs[:4])
    rw, st = random_walker_labels(store)
    want, _ = random_walker_labels(ims[:4], scrs[:4])
    for i in range(4):
        h, w = ims[i].shape
        assert np.array_equal(rw.labels[rw.offs[i]: rw.offs[i] + h * w].view(h, w).cpu().numpy(), want[i])
    torch.manual_seed(0)
    batch = next(iter(GpuLoader(rw, 2, (64, 64))))
    assert batch["image"].shape == (2, 1, 64, 64) and int(batch["label"].max()) <= 3


def test_base_datasets_random_walker_uses_gpu_labels():
    from wsl4mis_b200.dataloaders import random_walker_labels
    from wsl4mis_b200.dataloaders.dataset import BaseDataSets
    db = BaseDataSets("synthetic:30", split="train", sup_type="random_walker")
    dense = BaseDataSets("synthetic:30", split="train", sup_type="label")
    scr = BaseDataSets("synthetic:30", split="train", sup_type="scribble")
    pairs = [scr._read(c) for c in scr.sample_list]
    want, _ = random_walker_labels([p[0] for p in pairs], [p[1] for p in pairs])
    n_diff = 0
    for i in range(len(db)):
        img, lab = db._read(db.sample_list[i])
        assert np.array_equal(img, pairs[i][0]) and np.array_equal(lab, want[i])
        n_diff += int((lab != dense._read(dense.sample_list[i])[1]).sum())
    assert n_diff > 0, "random-walker labels equal the dense ground truth: the pseudo labels were not used"
    s = db[0]
    assert set(s) == {"image", "label", "idx"}


# ---------------------------------------------------------------------------------------------------------------- ce_dice step
def test_ce_dice_step_matches_oracle():
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet
    n, hw = 4, 64
    torch.manual_seed(3)
    m = UNet(1, 4)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    em = elem_masks_nchw(5, n, hw, hw)
    m.dropout_masks = {i: e.permute(0, 2, 3, 1).contiguous().to(DEV) for i, e in enumerate(em)}
    image, label = O.synth_batch(n, hw, hw, seed=11, dense=True)
    label[:, :4] = 4                                         # a few ignored pixels: CE skips them, Dice counts them in no class
    step = TrainStep(m, "ce_dice", base_lr=0.01, graph=False)
    loss = step(image.to(DEV), label.to(DEV))
    torch.cuda.synchronize()
    O.QUANT = True
    try:
        ref_loss, grads = R.ce_dice_step(p, image, label, {k: e for k, e in zip(ENC_MASK_KEYS, em)})
    finally:
        O.QUANT = None
    assert abs(loss.item() - ref_loss.item()) < 0.02 * abs(ref_loss.item()) + 1e-4, (loss.item(), ref_loss.item())
    named = dict(m.named_parameters())
    worst = 1.0
    for k, g in grads.items():
        if k.endswith("bias") and (".0.bias" in k or ".4.bias" in k):
            continue                                         # zero-gradient biases in front of BatchNorm
        delta, ref_delta = named[k].detach().cpu() - p[k], -0.01 * (g + 1e-4 * p[k])
        c = cosine(delta, ref_delta)
        worst = min(worst, c)
        assert c > 0.9, (k, c)
    print(f"[ce_dice] loss {loss.item():.5f} (oracle {ref_loss.item():.5f}), worst update cosine {worst:.4f}")


def test_ce_dice_graph_replay_equals_eager():
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet
    n, hw = 4, 64
    img, lab = O.synth_batch(n, hw, hw, seed=5, dense=True)
    img, lab = img.to(DEV), lab.to(DEV)
    losses, finals = {}, {}
    for graph in (False, True):
        torch.manual_seed(7)
        step = TrainStep(UNet(1, 4).to(DEV), "ce_dice", graph=graph)
        losses[graph] = [step(img, lab).item() for _ in range(6)]
        torch.cuda.synchronize()
        finals[graph] = step.flat.clone()
        if graph:
            assert step._graphs[0] is not None
    assert np.allclose(losses[False], losses[True], rtol=2e-3), (losses[False], losses[True])
    assert cosine(finals[False], finals[True]) > 0.999999
    assert losses[True][-1] < losses[True][0]


def test_ce_dice_rejects_global_batch():
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.networks.unet import UNet
    step = TrainStep(UNet(1, 4).to(DEV), "ce_dice", graph=False)
    step.global_batch = True                                 # the flag world_size > 1 sets; the head refuses before any collective
    img, lab = O.synth_batch(2, 32, 32, seed=1, dense=True)
    with pytest.raises(NotImplementedError, match="ce_dice"):
        step(img.to(DEV), lab.to(DEV))


# ---------------------------------------------------------------------------------------------------------------- scripts
def _stage(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    try:
        import build_ref
        import stage_rw
        code = build_ref.extract(str(tmp_path))
        if code is None or not stage_rw.extract(code):
            pytest.skip("reference scripts not staged (run __graft_entry__.build() where the reference exists)")
    finally:
        sys.path.pop(0)
    return code


@pytest.mark.parametrize("script,sup_type", [("train_fully_supervised_2D.py", "label"),
                                             ("train_weakly_supervised_pCE_random_walker_2D.py", "random_walker")])
def test_reference_script_runs_unchanged(tmp_path, script, sup_type):
    code = _stage(tmp_path)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, os.path.join(ROOT, "tests", "harness")])
    r = subprocess.run([sys.executable, script, "--root_path", "synthetic:30", "--max_iterations", "6", "--batch_size", "4",
                        "--exp", "rw_test", "--fold", "fold1", "--sup_type", sup_type], cwd=code, env=env, capture_output=True,
                       text=True, timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    found = [(int(a), float(b)) for a, b in re.findall(r"iteration (\d+) : loss : ([-+0-9.eE]+)", out)]
    assert [i for i, _ in found] == list(range(1, 7)), out[-3000:]
    assert all(np.isfinite(l) and abs(l) < 1e4 for _, l in found), found
    assert os.path.exists(os.path.join(os.path.dirname(code), "model", "rw_test_fold1", sup_type, "log.txt"))


def test_random_walker_script_reads_gpu_labels(tmp_path):
    """the staged script's dataset is the drop-in BaseDataSets: with sup_type='random_walker' its training labels are the GPU pseudo
    labels, not the dense ground truth the reference's synthetic-free path would silently read"""
    code = _stage(tmp_path)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, os.path.join(ROOT, "tests", "harness")])
    probe = ("import numpy as np\nfrom dataloaders.dataset import BaseDataSets\n"
             "rw = BaseDataSets(base_dir='synthetic:30', split='train', fold='fold1', sup_type='random_walker')\n"
             "gt = BaseDataSets(base_dir='synthetic:30', split='train', fold='fold1', sup_type='label')\n"
             "import wsl4mis_b200.dataloaders.dataset as D\n"
             "assert type(rw) is D.BaseDataSets and len(rw._rw) == len(rw)\n"
             "d = sum(int((rw[i]['label'] != gt[i]['label']).sum()) for i in range(len(rw)))\n"
             "print('differing pixels', d)\nassert d > 0\n")
    r = subprocess.run([sys.executable, "-c", probe], cwd=code, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
