"""The native trainer on the GPU: the batched metrics and the ragged zoom bit-identical to their per-volume forms, the resident
validation set equal to val_2D.test_single_volume per volume, every recipe end to end, the trainer's arithmetic equal to a hand-written
loop over the same step, the logged validation numbers, and no host synchronisation between validation points."""
import gc
import os
import random
import re
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = "synthetic:100"
ACDC_SHAPES = [(256, 216), (216, 256), (224, 154), (232, 256), (174, 208), (512, 428), (154, 224), (256, 256)]

if torch.cuda.is_available():
    import wsl4mis_b200.train as TR
    import wsl4mis_b200.val_2D as V
    from wsl4mis_b200._lib import call
    from wsl4mis_b200.dataloaders.dataset import BaseDataSets, GpuLoader, SliceStore, fold_ids, synthetic_acdc
    from wsl4mis_b200.engine import TrainStep
    from wsl4mis_b200.metric import VolumeSet, surface_metrics_workspace_bytes
    from wsl4mis_b200.networks.net_factory import net_factory
    from wsl4mis_b200.networks.unet import UNet, UNet_CCT


# ---------------------------------------------------------------- kernels
def _labels(rs, shape, kind):
    lab = rs.randint(0, 4, size=shape).astype(np.uint8)
    if kind == "blobs":             # smooth regions, as label maps are
        lab = np.zeros(shape, np.uint8)
        zz, yy, xx = np.meshgrid(*[np.arange(s) for s in shape], indexing="ij")
        for c in (1, 2, 3):
            cz, cy, cx = (rs.rand(3) * np.array(shape)).astype(int)
            r = rs.randint(2, max(3, min(shape[1:]) // 3))
            lab[((yy - cy) ** 2 + (xx - cx) ** 2 + 4 * (zz - cz) ** 2) < r * r] = c
    return lab


def _per_volume(pred, gt, shape, spacing, classes):
    S, H, W = shape
    ws = torch.empty(surface_metrics_workspace_bytes(shape, classes), dtype=torch.uint8, device=DEV)
    out = torch.empty((classes - 1, 12), dtype=torch.float64, device=DEV)
    call("wsl_surface_metrics", pred, gt, 3, S, H, W, classes, *spacing, ws, out)
    return out.cpu()


@pytest.mark.parametrize("seed,nvol", [(0, 1), (1, 7), (2, 40)])
def test_batched_metrics_equal_per_volume_bitwise(seed, nvol):
    rs = np.random.RandomState(seed)
    shapes, spacings, preds, gts = [], [], [], []
    for v in range(nvol):
        shape = (21, 512, 428) if (v == 0 and nvol > 1) else (int(rs.randint(1, 12)), int(rs.randint(3, 90)), int(rs.randint(3, 90)))
        p, g = _labels(rs, shape, "blobs" if v % 2 else "noise"), _labels(rs, shape, "blobs")
        if v % 5 == 1:
            p[p == 2] = 0                       # class 2 empty in pred
        if v % 5 == 2:
            g[g == 3] = 0                       # class 3 empty in gt
        if v % 5 == 3:
            p[p == 1] = 0
            g[g == 1] = 0                       # class 1 empty in both
        sp = (1.0, 1.0, 1.0) if v % 3 == 0 else (float(rs.choice([5.0, 6.5, 10.0])), float(rs.choice([1.25, 1.37, 1.5625])),
                                                  float(rs.choice([1.25, 1.37, 1.5625])))
        shapes.append(shape), spacings.append(sp), preds.append(p), gts.append(g)
    vs = VolumeSet(shapes, 4, spacings, DEV)
    pred = torch.from_numpy(np.concatenate([p.ravel() for p in preds])).to(DEV)
    gt = torch.from_numpy(np.concatenate([g.ravel() for g in gts])).to(DEV)
    out = torch.empty((nvol, 3, 12), dtype=torch.float64, device=DEV)
    got = vs(pred, gt, out).cpu()
    for v in range(nvol):
        a, b = vs.offsets[v], vs.offsets[v + 1]
        ref = _per_volume(pred[a:b].contiguous(), gt[a:b].contiguous(), shapes[v], spacings[v], 4)
        assert torch.equal(got[v].view(torch.int64), ref.view(torch.int64)), (v, shapes[v], spacings[v])


def test_ragged_zoom_equals_per_slice_zoom_bitwise():
    rs = np.random.RandomState(3)
    shapes = ACDC_SHAPES
    imgs = [rs.rand(h, w).astype(np.float32) for h, w in shapes]
    offs = np.concatenate([[0], np.cumsum([h * w for h, w in shapes])[:-1]])
    table = torch.tensor([(int(o), h, w) for o, (h, w) in zip(offs, shapes)], dtype=torch.int64, device=DEV)
    flat = torch.from_numpy(np.concatenate([i.ravel() for i in imgs])).to(DEV)
    N, mhw = len(shapes), max(h * w for h, w in shapes)
    dense = torch.empty((N, 256, 256), dtype=torch.float32, device=DEV)
    call("wsl_zoom_nearest_ragged", flat, 0, table, N, mhw, 0, 256, 256, dense)
    lab = torch.from_numpy(rs.randint(0, 4, size=(N, 256, 256)).astype(np.uint8)).to(DEV)
    back = torch.empty(int(offs[-1]) + shapes[-1][0] * shapes[-1][1], dtype=torch.uint8, device=DEV)
    call("wsl_zoom_nearest_ragged", lab, 1, table, N, mhw, 1, 256, 256, back)
    for s, (h, w) in enumerate(shapes):
        ref = torch.empty((1, 256, 256), dtype=torch.float32, device=DEV)
        call("wsl_zoom_nearest", torch.from_numpy(imgs[s]).to(DEV), 0, 1, h, w, 256, 256, ref)
        assert torch.equal(dense[s].view(torch.int32), ref[0].view(torch.int32)), (h, w)
        refb = torch.empty((1, h, w), dtype=torch.uint8, device=DEV)
        call("wsl_zoom_nearest", lab[s].contiguous(), 1, 1, 256, 256, h, w, refb)
        assert torch.equal(back[int(offs[s]):int(offs[s]) + h * w].view(h, w), refb[0]), (h, w)


# ---------------------------------------------------------------- the resident validation set
@pytest.fixture(scope="module")
def trained():
    """state_dict of a UNet after 300 ce_dice steps (batch 12) on fold 1's training slices of synthetic:100"""
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
    torch.manual_seed(1)
    net = (UNet_CCT if cct else UNet)(1, 4)
    if cct:
        full = net.state_dict()
        full.update({k.replace("decoder.", "main_decoder.", 1) if k.startswith("decoder.") else k: v for k, v in sd.items()})
        sd = full
    net.load_state_dict(sd)
    return net.to(DEV).set_precision(precision).eval()


@pytest.mark.parametrize("cct", [False, True])
@pytest.mark.parametrize("precision", ["bf16", "fp16x3"])
def test_validation_set_equals_per_volume_loop(trained, cct, precision):
    net = _net(trained, cct, precision)
    vset = V.ValidationSet(ROOT, fold="fold1")
    got = vset.score(net, 4)
    db = BaseDataSets(base_dir=ROOT, fold="fold1", split="val")
    ref = []
    for i in range(len(db)):
        s = db[i]
        img, lab = torch.from_numpy(s["image"])[None], torch.from_numpy(s["label"])[None]
        ref.append((V.test_single_volume_cct if cct else V.test_single_volume)(img, lab, net, 4))
    assert len(got) == len(ref) == 20
    assert got == ref
    # each slice's logits: the same bits in the padded chunk as at batch S
    S, h, w = vset.shapes[0]
    with torch.no_grad():
        x = vset.x[:S].clone()
        out_s = net(x)
        out_c = net(vset.x[:vset.chunk])
    a = (out_s[0] if cct else out_s)[:S]
    b = (out_c[0] if cct else out_c)[:S]
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def test_prediction_against_empty_label_names_case_and_class(trained):
    net = _net(trained, False, "bf16")
    cases = synthetic_acdc(3)
    img, lab, _ = cases["patient002"]
    lab = lab.copy()
    lab[lab == 2] = 0
    vset = V.ValidationSet.from_arrays([cases["patient001"][0], img], [cases["patient001"][1], lab], ["patient001", "patient002"])
    with pytest.raises(RuntimeError, match=r"second supplied array.*case patient002, class 2"):
        vset.score(net, 4)


# ---------------------------------------------------------------- the trainer
def _argv(script, exp, iters, bs, extra=()):
    return [script, "--root_path", ROOT, "--exp", exp, "--fold", "fold1", "--max_iterations", str(iters), "--batch_size", str(bs),
            *extra]


@pytest.fixture()
def workdir(tmp_path, monkeypatch):
    work = tmp_path / "code"
    work.mkdir()
    monkeypatch.chdir(work)
    return tmp_path


def _keys(name):
    return list(net_factory(net_type=name, in_chns=1, class_num=4).state_dict().keys())


@pytest.mark.parametrize("script", sorted(TR.RECIPES) if torch.cuda.is_available() else [])
def test_every_recipe_runs(workdir, script):
    recipe = TR.RECIPES[script]
    bs = 4 if recipe.kind == "semi" else 2
    extra = ("--period_iter", "100") if recipe.kind == "s2l" else ()
    snap = TR.train(_argv(script, "T/r", 400, bs, extra))
    log = open(os.path.join(snap, "log.txt")).read().splitlines()
    msgs = [re.sub(r"^\[\d\d:\d\d:\d\d\.\d{3}\] ", "", l) for l in log]
    assert msgs[0].startswith("Namespace(") and msgs[1].endswith(" iterations per epoch")
    if recipe.log is not None:
        it = [m for m in msgs if m.startswith("iteration ") and " : loss : " in m]
        assert len(it) == 400 and [int(m.split()[1]) for m in it] == list(range(1, 401))
        pat = re.escape(recipe.log).replace("%d", r"\d+").replace("%f", r"-?(\d+\.\d{6}|nan|inf)")
        assert all(re.fullmatch(pat, m) for m in it), it[0]
    vals = [m for m in msgs if "mean_dice" in m]
    assert [int(m.split()[1]) for m in vals] == [200, 400]
    if recipe.kind == "s2l":
        assert msgs.count("update weight start") == 4 and msgs.count("update weight end") == 4
    files = os.listdir(snap)
    model = TR.parse(_argv(script, "T/r", 400, bs))[1].model
    assert f"{model}_best_model.pth" in files and any(re.fullmatch(r"iter_(200|400)_dice_[\d.]+\.pth", f) for f in files)
    sd = torch.load(os.path.join(snap, f"{model}_best_model.pth"))
    assert list(sd.keys()) == _keys(model)
    assert all(v.dtype == torch.float32 for k, v in sd.items() if "num_batches_tracked" not in k)
    net_factory(net_type=model, in_chns=1, class_num=4).load_state_dict(sd)


def test_3000_iterations_and_test_2D_reads_the_checkpoint(workdir):
    import wsl4mis_b200.test_2D as T2
    snap = TR.train(_argv("train_weakly_supervised_pCE_2D.py", "T/long", 3000, 4))
    msgs = open(os.path.join(snap, "log.txt")).read()
    assert "save model to ../model/T/long_fold1/scribble/iter_3000.pth" in msgs
    shutil.copy(os.path.join(snap, "iter_3000.pth"), os.path.join(snap, "iter_60000.pth"))
    F = T2.parser.parse_args(["--root_path", ROOT, "--exp", "T/long", "--fold", "fold1", "--sup_type", "scribble"])
    # the checkpoint loads and predicts; metrics may raise on an empty class, which is the script's behaviour too
    try:
        T2.Inference(F)
    except RuntimeError as e:
        assert "does not contain any binary object" in str(e)


def _flat_after(script, iters, use_trainer, workdir):
    argv = _argv(script, "T/eq", iters, 4)
    if use_trainer:
        snap = TR.train(argv)
        return snap
    name, args, precision = TR.parse(argv)
    model, step, batches, n, _ = TR.build(name, args, precision)
    it = 0
    for _ in range(args.max_iterations // n + 1):          # the INTEGRATION.md section 2 loop
        for inputs in batches():
            step(*inputs)
            it += 1
            if it >= args.max_iterations:
                break
        if it >= args.max_iterations:
            break
    torch.cuda.synchronize()
    return step.flat.clone()


@pytest.mark.parametrize("script", ["train_weakly_supervised_pCE_GatedCRFLoss_2D.py", "train_mean_teacher_2D.py"])
def test_trainer_adds_nothing_to_the_arithmetic(workdir, script, monkeypatch):
    holder = {}
    orig = TR.Trainer.run

    def run(self):
        out = orig(self)
        torch.cuda.synchronize()
        holder["flat"] = self.step.flat.clone()
        return out
    monkeypatch.setattr(TR.Trainer, "run", run)
    snap = _flat_after(script, 400, True, workdir)
    hand = _flat_after(script, 400, False, workdir)
    assert torch.equal(holder["flat"].view(torch.int32), hand.view(torch.int32))
    # the logged validation numbers are the real ones: val_2D's per-volume path on the saved best checkpoint
    msgs = open(os.path.join(snap, "log.txt")).read().splitlines()
    best_line = max((l for l in msgs if "mean_dice" in l), key=lambda l: float(l.split("mean_dice : ")[1].split()[0]))
    net = net_factory(net_type="unet", in_chns=1, class_num=4)
    net.load_state_dict(torch.load(os.path.join(snap, "unet_best_model.pth")))
    net.eval()
    db = BaseDataSets(base_dir=ROOT, fold="fold1", split="val")
    metric_list = 0.0
    for i in range(len(db)):
        s = db[i]
        metric_list += np.array(V.test_single_volume(torch.from_numpy(s["image"])[None], torch.from_numpy(s["label"])[None], net, 4))
    metric_list = metric_list / len(db)
    perf, hd = np.mean(metric_list, axis=0)[0], np.mean(metric_list, axis=0)[1]
    assert best_line.endswith("mean_dice : %f mean_hd95 : %f" % (perf, hd))


def test_no_host_sync_between_validation_points(workdir, monkeypatch):
    """iterations 1-300 capture every batch shape; 300-450 run under sync-debug 'error' across the validation at 400"""
    orig_add = TR._LogBuffer.add

    def add(self, iter_num, lr, values, host_values):
        orig_add(self, iter_num, lr, values, host_values)
        if iter_num == 300:
            torch.cuda.set_sync_debug_mode("error")
    monkeypatch.setattr(TR._LogBuffer, "add", add)
    try:
        snap = TR.train(_argv("train_weakly_supervised_pCE_GatedCRFLoss_2D.py", "T/sync", 450, 4))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    msgs = open(os.path.join(snap, "log.txt")).read()
    assert "iteration 400 : mean_dice" in msgs and "iteration 450 : loss" in msgs
