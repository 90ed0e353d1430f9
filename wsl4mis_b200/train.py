"""Train a reference recipe natively on the captured steps:

    python -m wsl4mis_b200.train train_weakly_supervised_pCE_GatedCRFLoss_2D.py --fold fold1 --exp ACDC/WeaklySeg_pCE_GatedCRFLoss

The command line is the script's own (``python -u train_X.py ARGS`` becomes ``python -m wsl4mis_b200.train train_X.py ARGS``), run
from the directory the scripts run in.  Each of the 16 scripts with a fused step has one entry in `RECIPES`: its argparse flags
(names, types, defaults and order, so ``str(args)`` is the script's Namespace), its step body, its loader and its per-iteration log
line.  The loop is the scripts' skeleton (train_weakly_supervised_pCE_2D.py:56-176): seeding, ``net_factory``, ``max_epoch =
max_iterations // len(loader) + 1`` (the labelled loader for the semi-supervised scripts), validation every 200 iterations with
best-model saves on a strict improvement, ``iter_{N}.pth`` every 3000, the stop at ``max_iterations``, and ``log.txt`` in the
scripts' logging format under ``../model/{exp}_{fold}/{sup_type}``.  ``--precision`` (bf16 | fp16 | fp16x3 | fp32, default bf16)
is the one flag the scripts lack; graph capture is always on.  ``--model pnet`` (PNet2D) runs every recipe but the two-output
``..._pCE_ours_proposed.py``, in bf16, fp16 or fp16x3 (`check_model`).

Several GPUs: ``torchrun --nproc_per_node W -m wsl4mis_b200.train train_X.py ARGS`` runs W ranks, batch-sharded data parallel
with per-rank BatchNorm statistics and loss normalisers (DESIGN §7).  ``--batch_size`` stays the script's global batch: each rank
takes batch_size / W (the two-stream scripts batch_size / 2 / W per stream), and its loaders walk their `shard` of every epoch's
permutation with augmentation draws from a stream of their own (`rank_streams`).  Rank 0 alone writes log.txt, TensorBoard scalars
and checkpoints, validates, and logs its own shard's loss parts; the other ranks go on to the next step and meet it at that step's
all-reduce.  With WORLD_SIZE unset or 1 nothing of this runs.

Between two validation points the loop does not wait on the device: each iteration's loss parts are copied, in stream order,
into a device buffer of up to 200 rows, and the buffer comes back in one device-to-host copy at each validation point, checkpoint
and at the end; its lines are then written in iteration order ahead of what follows them, so ``log.txt`` has the script's lines in
the script's order (only the timestamps are those of the flush).  Validation is ``val_2D.ValidationSet.score``: the validation
split stays on the device and is scored in one batched pass.
"""
import argparse
import logging
import os
import random
import sys
from collections import namedtuple
from itertools import cycle

import numpy as np
import torch

PRECISIONS = ("bf16", "fp16", "fp16x3", "fp32")
VAL_EVERY, SAVE_EVERY = 200, 3000

# argparse flags of the scripts, in their order: (name, type, default)
_WSS = (("root_path", str, "../data/ACDC"), ("exp", str, None), ("fold", str, "fold1"), ("sup_type", str, "scribble"),
        ("model", str, "unet"), ("num_classes", int, 4), ("max_iterations", int, 30000), ("batch_size", int, 24),
        ("deterministic", int, 1), ("base_lr", float, 0.01), ("patch_size", list, [256, 256]), ("seed", int, 2022))
_SEMI = (("root_path", str, "../data/ACDC"), ("exp", str, None), ("model", str, "unet"), ("fold", str, "fold2"),
         ("sup_type", str, "label"), ("max_iterations", int, 30000), ("batch_size", int, 12), ("deterministic", int, 1),
         ("base_lr", float, 0.01), ("patch_size", list, [256, 256]), ("seed", int, 2022), ("num_classes", int, 4),
         ("labeled_bs", int, 6), ("labeled_num", int, 4), ("ema_decay", float, 0.99), ("consistency_type", str, "mse"),
         ("consistency", float, 0.1), ("consistency_rampup", float, 200.0))


def _flags(base, extra=(), **defaults):
    """base flags with some defaults replaced, then `extra` flags appended"""
    out = [(n, t, defaults.get(n, d)) for n, t, d in base]
    assert set(defaults) <= {n for n, _, _ in base}
    return tuple(out) + tuple(extra)


# One recipe per script.  kind: 'single' (GpuLoader), 's2l' (S2LLoader + ensemble refresh), 'semi' (zip(cycle(labelled), unlabelled)).
# step: (args, model, world_size) -> step.  log: the per-iteration line (None: the script logs none), fed by iter_num, the loss and `cols`.
# cols: (TensorBoard tag, step -> 0-dim device tensor) of the values after the loss; host: (tag, step -> float) values from the host.
Recipe = namedtuple("Recipe", "flags kind step log cols host", defaults=((),))
_LOG2 = 'iteration %d : loss : %f, loss_ce: %f'
_LOG3 = 'iteration %d : loss : %f, loss_ce: %f, loss_dice: %f'


def _part(name, attr="loss_parts"):
    return lambda step: getattr(step, attr)[name]


def _train_step(variant):
    def make(args, model, world_size=1):
        from .engine import TrainStep
        step = TrainStep(model, variant, base_lr=args.base_lr, max_iterations=args.max_iterations, graph=True, world_size=world_size)
        if variant == "pce_variance":
            step.consistency, step.consistency_rampup = args.consistency, args.consistency_rampup
        return step
    return make


def _teacher_step(cls):
    def make(args, model, world_size=1):
        from . import engine
        from .networks.net_factory import net_factory
        ema = net_factory(net_type=args.model, in_chns=1, class_num=args.num_classes)     # create_model(ema=True)
        for p in ema.parameters():
            p.detach_()
        ema.set_precision(model.precision)
        return getattr(engine, cls)(model, ema, base_lr=args.base_lr, max_iterations=args.max_iterations,
                                    **({} if cls == "USTMStep" else dict(consistency=args.consistency,
                                                                          consistency_rampup=args.consistency_rampup)), graph=True,
                                    world_size=world_size)
    return make


def _em_step(args, model, world_size=1):
    from .engine import EntropyMinStep
    return EntropyMinStep(model, base_lr=args.base_lr, max_iterations=args.max_iterations, consistency=args.consistency,
                          consistency_rampup=args.consistency_rampup, graph=True, world_size=world_size)


def _dan_step(args, model, world_size=1):
    from .engine import DANStep
    from .networks.discriminator import FCDiscriminator
    disc = FCDiscriminator(num_classes=args.num_classes).cuda()
    return DANStep(model, disc, base_lr=args.base_lr, max_iterations=args.max_iterations, consistency=args.consistency,
                   consistency_rampup=args.consistency_rampup, graph=True, world_size=world_size)


def _s2l_step(args, model, world_size=1):
    from .engine import S2LStep
    return S2LStep(model, thr_iter=args.thr_iter, thr_conf=args.thr_conf, base_lr=args.base_lr, max_iterations=args.max_iterations,
                   graph=True, world_size=world_size)


_DMPLS = _train_step("dmpls")
_CE = (("info/loss_ce", _part("ce")),)
_SEMI_COLS = (("info/loss_ce", _part("loss_ce", "parts")), ("info/loss_dice", _part("loss_dice", "parts")),
              ("info/consistency_loss", _part("consistency", "parts")))
RECIPES = {
    "train_weakly_supervised_pCE_2D.py": Recipe(_flags(_WSS, exp="ACDC_pCE", base_lr=0.03), "single", _train_step("pce"), _LOG2, _CE),
    "train_weakly_supervised_pCE_GatedCRFLoss_2D.py": Recipe(
        _flags(_WSS, exp="ACDC_pCE_GatedCRFLoss", batch_size=6), "single", _train_step("pce_gatedcrf"), _LOG2,
        _CE + (("info/out_gatedcrf", _part("crf")),)),
    "train_weakly_supervised_pCE_MumfordShah_Loss_2D.py": Recipe(
        _flags(_WSS, exp="ACDC_pCE_MumfordShah_Loss", max_iterations=60000, batch_size=12), "single", _train_step("pce_ms"),
        'iteration %d : loss : %f, loss_ce: %f, loss_mumfordshah: %f', _CE + (("info/loss_mumfordshah", _part("ms")),)),
    "train_weakly_supervised_pCE_TV_2D.py": Recipe(
        _flags(_WSS, (("labeled_num", int, 50),), exp="ACDC_pCE_TV", seed=1337), "single", _train_step("pce_tv"), _LOG2,
        _CE + (("info/loss_tv", _part("tv")),)),
    "train_weakly_supervised_pCE_Entropy_Mini_2D.py": Recipe(
        _flags(_WSS, exp="ACDC_pCE_Entropy_Mini"), "single", _train_step("pce_entropy"), _LOG2, _CE),
    "train_weakly_supervised_pCE_Inter&Intra_Class_2D.py": Recipe(
        _flags(_WSS, (("consistency", float, 0.1), ("consistency_rampup", float, 200.0)), exp="ACDC_pCE_Inter&Intra_Class"),
        "single", _train_step("pce_variance"), _LOG2, _CE),
    "train_weakly_supervised_segmentation_pCE_ours_proposed.py": Recipe(
        _flags(_WSS, exp="ACDC/pCE_SPS", model="unet_cct", max_iterations=60000, batch_size=6), "single", _DMPLS,
        'iteration %d : loss : %f, loss_ce: %f, loss_pse_sup: %f, alpha: %f', _CE + (("info/loss_pse_sup", _part("pse_sup")),),
        (("info/alpha", lambda step: step.beta),)),
    "train_fully_supervised_2D.py": Recipe(
        _flags(_WSS, exp="ACDC", fold="fold5", sup_type="label", batch_size=16, base_lr=0.03), "single", _train_step("ce_dice"),
        _LOG2, _CE),
    "train_weakly_supervised_pCE_random_walker_2D.py": Recipe(
        _flags(_WSS, exp="ACDC/pCE_Random_Walker", sup_type="random_walker"), "single", _train_step("ce_dice"), _LOG2, _CE),
    "train_weakly_supervised_ustm_2D.py": Recipe(
        _flags(_WSS, exp="ACDC/pCE_Seg_USTM", max_iterations=60000, batch_size=12), "single", _teacher_step("USTMStep"), _LOG2,
        (("info/loss_ce", _part("ce", "parts")), ("info/consistency_loss", _part("consistency", "parts")))),
    "train_s2l.py": Recipe(
        _flags(_WSS, (("labeled_bs", int, 6), ("labeled_num", int, 4), ("ema_decay", float, 0.99), ("consistency", float, 0.1),
                      ("consistency_rampup", float, 200.0), ("period_iter", int, 100), ("thr_iter", int, 6000),
                      ("thr_conf", float, 0.8), ("alpha", float, 0.2)),
               exp="ACDC/pCE_scribble2label", max_iterations=60000, batch_size=12, seed=1337),
        "s2l", _s2l_step, None, _CE + (("info/loss_weight", _part("u")),)),
    "train_mean_teacher_2D.py": Recipe(_flags(_SEMI, exp="ACDC_Semi/Mean_Teacher"), "semi", _teacher_step("MeanTeacherStep"), _LOG3,
                                       _SEMI_COLS),
    "train_uncertainty_aware_mean_teacher_2D.py": Recipe(
        _flags(_SEMI, exp="ACDC_Semi/Uncertainty_Aware_Mean_Teacher"), "semi", _teacher_step("UAMTStep"), _LOG3, _SEMI_COLS),
    "train_entropy_minimization_2D.py": Recipe(_flags(_SEMI, exp="ACDC_Semi/Entropy_Minimization", fold="fold1"), "semi", _em_step,
                                               _LOG3, _SEMI_COLS),
    "train_deep_adversarial_network_2D.py": Recipe(_flags(_SEMI, exp="ACDC_Semi/DAN"), "semi", _dan_step, _LOG3, _SEMI_COLS),
    "train_partially_fully_supervised.py": Recipe(
        _flags(_SEMI, exp="ACDC_Semi/Entropy_Minimization", fold="fold1"), "semi", _train_step("ce_dice"), _LOG3,
        (("info/loss_ce", _part("ce")), ("info/loss_dice", _part("dice")))),
}
# the one script whose validation split ignores --fold (BaseDataSets(base_dir, split="val"): the default fold1)
VAL_FOLD_DEFAULT = {"train_weakly_supervised_pCE_Inter&Intra_Class_2D.py"}


def recipe_for(script):
    """the recipe of a script name or path; raises ValueError listing the supported names"""
    name = os.path.basename(script)
    if name not in RECIPES:
        raise ValueError(f"no native recipe for {script!r}; supported scripts: {', '.join(sorted(RECIPES))}")
    return RECIPES[name]


def parser_for(script):
    """the script's argparse parser: its flags with their names, types, defaults and order"""
    p = argparse.ArgumentParser()
    for name, ty, default in recipe_for(script).flags:
        p.add_argument("--" + name, type=ty, default=default)
    return p


def parse(argv):
    """[script, flags...] -> (script name, the script's Namespace, precision)"""
    if not argv:
        raise SystemExit("usage: python -m wsl4mis_b200.train <train_script.py> [--precision bf16|fp16|fp16x3|fp32] [the script's flags]")
    script = os.path.basename(argv[0])
    recipe_for(script)
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--precision", choices=PRECISIONS, default="bf16")
    opts, rest = pre.parse_known_args(argv[1:])
    args = parser_for(script).parse_args(rest)
    check_model(script, args, opts.precision)
    return script, args, opts.precision


PNET_PRECISIONS = ("bf16", "fp16", "fp16x3")       # PNet2D's dilated convolutions have no CUDA-core (fp32 mode) kernel


def check_model(script, args, precision):
    """raise ValueError for the --model / --precision combinations no step runs, before any data or network is built:
    PNet2D in fp32 mode, and PNet2D under the two-output recipe (pCE_ours_proposed unpacks ``outputs, outputs_aux1``)"""
    if args.model != "pnet":
        return
    if precision not in PNET_PRECISIONS:
        raise ValueError(f"--model pnet runs in {' / '.join(PNET_PRECISIONS)} (--precision {precision} is not available: PNet2D's "
                         f"dilated convolutions run on the tensor-core kernels only)")
    if recipe_for(script).step is _DMPLS:
        raise ValueError(f"{os.path.basename(script)} needs a network with two outputs (--model unet_cct): it unpacks "
                         f"'outputs, outputs_aux1 = model(volume_batch)', and PNet2D has one output")


def rank_batch(script, batch_size, world_size):
    """the per-rank batch of a recipe: batch_size / W (the two-stream recipes: batch_size / 2 / W per stream); raises ValueError
    when W > 1 does not divide it.  W = 1: the script's own batch_size (batch_size // 2 per stream)."""
    per_stream = recipe_for(script).kind == "semi"
    if world_size == 1:
        return batch_size // 2 if per_stream else batch_size
    div = 2 * world_size if per_stream else world_size
    if batch_size % div:
        raise ValueError(f"--batch_size {batch_size} does not split over {world_size} ranks: {os.path.basename(script)} needs a "
                         f"multiple of {div}" + (" (two streams of batch_size / 2, each split over the ranks)" if per_stream else ""))
    return batch_size // div


def snapshot_path(args):
    return "../model/{}_{}/{}".format(args.exp, args.fold, args.sup_type)


class _LogBuffer:
    """Per-iteration values kept on the device until a flush: row i = [loss, cols...] of one iteration, copied in stream order"""

    def __init__(self, ncols, device, rows=VAL_EVERY):
        self.dev = torch.device(device)
        self.buf = torch.zeros((rows, 1 + ncols), dtype=torch.float32, device=self.dev)
        self.host = torch.zeros(self.buf.shape, dtype=torch.float32, pin_memory=self.dev.type == "cuda")
        self.done = torch.cuda.Event() if self.dev.type == "cuda" else None
        self.pending = []          # (iter_num, lr, host values) of the rows not yet written

    def add(self, iter_num, lr, values, host_values):
        i = len(self.pending)
        assert i < self.buf.shape[0], "log buffer full: validation flushes it every 200 iterations"
        self.buf[i].copy_(torch.stack([v.reshape(()).float() for v in values]), non_blocking=True)
        self.pending.append((iter_num, lr, host_values))

    def flush(self):
        """-> [(iter_num, lr, [loss, cols...], host values)] in iteration order; one device-to-host copy"""
        n = len(self.pending)
        if not n:
            return []
        self.host[:n].copy_(self.buf[:n], non_blocking=True)
        if self.done is not None:
            self.done.record()
            self.done.synchronize()
        rows = [(it, lr, [float(v) for v in self.host[i].tolist()], hv) for i, (it, lr, hv) in enumerate(self.pending)]
        self.pending = []
        return rows


def _host_state(model):
    """model.state_dict() with every tensor copied to host memory: one wait on the device for the whole copy"""
    sd = model.state_dict()
    out = {k: v.detach().to("cpu", non_blocking=True) for k, v in sd.items()}
    if any(v.is_cuda for v in sd.values()):
        ev = torch.cuda.Event()
        ev.record()
        ev.synchronize()
    return out


class Trainer:
    """The scripts' loop around a step.  `batches()` yields one epoch of step inputs (a tuple per iteration); `validator` has
    ``score(model, classes)``; `log` takes one line; `writer` (optional) takes ``add_scalar(tag, value, step)``."""

    def __init__(self, args, recipe, model, step, batches, n_per_epoch, validator, snapshot, log, writer=None, refresh=None,
                 device=None, rank=0):
        """rank > 0: a data-parallel rank other than rank 0; it runs the steps (and the refresh) only, and never logs, validates or
        saves"""
        self.args, self.recipe, self.model, self.step = args, recipe, model, step
        self.main = int(rank) == 0
        self.batches, self.n_per_epoch, self.validator = batches, int(n_per_epoch), validator
        self.snapshot, self.log, self.writer, self.refresh = snapshot, log, writer, refresh
        dev = device if device is not None else next(model.parameters()).device
        self.buffer = _LogBuffer(len(recipe.cols), dev)

    def _write(self, rows):
        r = self.recipe
        for it, lr, vals, hv in rows:
            if self.writer is not None:
                self.writer.add_scalar("info/lr", lr, it)
                self.writer.add_scalar("info/total_loss", vals[0], it)
                for (tag, _), v in zip(r.cols, vals[1:]):
                    if tag != "info/loss_weight" or it > getattr(self.args, "thr_iter", 0):
                        self.writer.add_scalar(tag, v, it)
                for (tag, _), v in zip(r.host, hv):
                    self.writer.add_scalar(tag, v, it)
            if r.log is not None:
                self.log(r.log % tuple([it] + vals[:r.log.count("%f") - len(hv)] + list(hv)))

    def _flush(self):
        self._write(self.buffer.flush())

    def _save(self, paths):
        state = _host_state(self.model)
        for p in paths:
            torch.save(state, p)

    def _validate(self, iter_num, best):
        args = self.args
        metric_list = 0.0
        results = self.validator.score(self.model, args.num_classes)
        for metric_i in results:
            metric_list += np.array(metric_i)
        metric_list = metric_list / len(results)
        if self.writer is not None:
            for class_i in range(args.num_classes - 1):
                self.writer.add_scalar('info/val_{}_dice'.format(class_i + 1), metric_list[class_i, 0], iter_num)
                self.writer.add_scalar('info/val_{}_hd95'.format(class_i + 1), metric_list[class_i, 1], iter_num)
        performance = np.mean(metric_list, axis=0)[0]
        mean_hd95 = np.mean(metric_list, axis=0)[1]
        if self.writer is not None:
            self.writer.add_scalar('info/val_mean_dice', performance, iter_num)
            self.writer.add_scalar('info/val_mean_hd95', mean_hd95, iter_num)
        if performance > best:
            best = performance
            self._save([os.path.join(self.snapshot, 'iter_{}_dice_{}.pth'.format(iter_num, round(best, 4))),
                        os.path.join(self.snapshot, '{}_best_model.pth'.format(args.model))])
        self.log('iteration %d : mean_dice : %f mean_hd95 : %f' % (iter_num, performance, mean_hd95))
        self.model.train()
        return best

    def run(self):
        args, r, step, main = self.args, self.recipe, self.step, self.main
        if main:
            self.log("{} iterations per epoch".format(self.n_per_epoch))
        iter_num, best = 0, 0.0
        max_epoch = args.max_iterations // self.n_per_epoch + 1
        for _ in range(max_epoch):
            for inputs in self.batches():
                lr = args.base_lr * (1.0 - iter_num / args.max_iterations) ** 0.9
                loss = step(*inputs)
                iter_num += 1
                if main:
                    self.buffer.add(iter_num, lr, [loss] + [get(step) for _, get in r.cols], [get(step) for _, get in r.host])
                if main and iter_num > 0 and iter_num % VAL_EVERY == 0:
                    self._flush()
                    best = self._validate(iter_num, best)
                if main and iter_num % SAVE_EVERY == 0:
                    self._flush()
                    path = os.path.join(self.snapshot, 'iter_' + str(iter_num) + '.pth')
                    self._save([path])
                    self.log("save model to {}".format(path))
                if self.refresh is not None and iter_num > 0 and iter_num % args.period_iter == 0:
                    if main and r.log is not None:
                        self._flush()
                    if main:
                        self.log("update weight start")
                    self.refresh()          # every rank: the refresh is split over the ranks and gathered on all of them
                    if main:
                        self.log("update weight end")
                if iter_num >= args.max_iterations:
                    break
            if iter_num >= args.max_iterations:
                break
        if main:
            self._flush()
        return "Training Finished!"


def _summary_writer(path):
    """the scripts' SummaryWriter when torch.utils.tensorboard or tensorboardX imports, else None"""
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError:
        try:
            from tensorboardX import SummaryWriter
        except ImportError:
            return None
    return SummaryWriter(path)


def two_stream(loader_l, loader_u, labelled_only=False):
    """one epoch of the semi-supervised scripts' feed, zip(cycle(labelled), unlabelled): `cycle` keeps the labelled batches of its
    first pass and replays them until the unlabelled loader ends the epoch (DESIGN F19).  -> step inputs per iteration: (image_l,
    label_l, image_u), or (image_l, label_l) for the partially supervised script, which loads the unlabelled batch and never uses it"""
    for bl, bu in zip(cycle(loader_l), loader_u):
        yield (bl["image"], bl["label"]) if labelled_only else (bl["image"], bl["label"], bu["image"])


def build(script, args, precision, rank=0, world_size=1):
    """-> (model, step, batches, iterations per epoch, refresh or None): the recipe's network, step and loaders, seeded as the
    script seeds them (random / numpy / torch with --seed, then net_factory).  world_size > 1: rank `rank`'s step, and its loaders
    over its shard of each epoch at `rank_batch`, drawing their augmentation parameters from `rank_streams(--seed, rank)`."""
    from .dataloaders.dataset import BaseDataSets, BaseDataSets_s2l, GpuLoader, S2LLoader, rank_streams
    from .networks.net_factory import net_factory
    recipe = recipe_for(script)
    check_model(script, args, precision)
    bs = rank_batch(script, args.batch_size, world_size)
    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.cuda.manual_seed(args.seed)
    model = net_factory(net_type=args.model, in_chns=1, class_num=args.num_classes)
    if model is None:
        raise ValueError(f"net_factory does not build --model {args.model!r}")
    model.set_precision(precision)
    size = tuple(int(x) for x in args.patch_size)
    shard = dict(rank=rank, world_size=world_size, streams=rank_streams(args.seed, rank) if world_size > 1 else None)
    refresh = None
    if recipe.kind == "semi":
        from .dataloaders.dataset_semi import BaseDataSets as SemiSets
        store_l = SemiSets(base_dir=args.root_path, labeled_type="labeled", fold=args.fold, split="train").to_slice_store()
        store_u = SemiSets(base_dir=args.root_path, labeled_type="unlabeled", fold=args.fold, split="train").to_slice_store()
        loader_l, loader_u = GpuLoader(store_l, bs, size, **shard), GpuLoader(store_u, bs, size, **shard)
        step = recipe.step(args, model, world_size)
        labelled_only = script == "train_partially_fully_supervised.py"
        batches = lambda: two_stream(loader_l, loader_u, labelled_only)
        n = len(loader_l)
    elif recipe.kind == "s2l":
        store = BaseDataSets_s2l(base_dir=args.root_path, fold=args.fold).to_slice_store()
        loader = S2LLoader(store, bs, size, **shard)
        step = recipe.step(args, model, world_size)
        batches = lambda: ((b["image"], b["scribble"], b["weight"]) for b in loader)
        n = len(loader)
        refresh = lambda: step.refresh(store, alpha=args.alpha)
    else:
        store = BaseDataSets(base_dir=args.root_path, split="train", fold=args.fold, sup_type=args.sup_type).to_slice_store()
        loader = GpuLoader(store, bs, size, **shard)
        step = recipe.step(args, model, world_size)
        batches = lambda: ((b["image"], b["label"]) for b in loader)
        n = len(loader)
    return model, step, batches, n, refresh


def train(argv):
    """run one recipe from its command line ([script, flags...]); -> the snapshot directory.  Under torchrun (WORLD_SIZE > 1)
    each process is one rank on cuda:LOCAL_RANK, in an NCCL process group it creates and destroys (a caller that already holds
    one keeps it)."""
    import torch.distributed as dist
    from .ddp import env_world
    script, args, precision = parse(argv)
    rank, local_rank, world = env_world()
    rank_batch(script, args.batch_size, world)          # a batch that does not split raises before anything is built
    own_group = world > 1 and not dist.is_initialized()
    if own_group:
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        if rank == 0:
            return _train_logged(script, args, precision, world)
        model, step, batches, n, refresh = build(script, args, precision, rank, world)
        Trainer(args, recipe_for(script), model, step, batches, n, None, None, lambda msg: None, None, refresh, rank=rank).run()
        return snapshot_path(args)
    finally:
        if own_group:
            dist.destroy_process_group()


def _train_logged(script, args, precision, world=1):
    """rank 0 (or the one process): log.txt, TensorBoard, validation and checkpoints around the loop"""
    from .val_2D import ValidationSet
    snapshot = snapshot_path(args)
    os.makedirs(snapshot, exist_ok=True)
    logger = logging.getLogger("wsl4mis_b200.train")
    logger.setLevel(logging.INFO)
    logger.propagate = False
    fmt = logging.Formatter('[%(asctime)s.%(msecs)03d] %(message)s', datefmt='%H:%M:%S')
    handlers = [logging.FileHandler(snapshot + "/log.txt"), logging.StreamHandler(sys.stdout)]
    for h in handlers:
        h.setFormatter(fmt)
        logger.addHandler(h)
    writer = None
    try:
        logger.info(str(args))
        model, step, batches, n, refresh = build(script, args, precision, 0, world)
        val_fold = "fold1" if script in VAL_FOLD_DEFAULT else args.fold
        validator = ValidationSet(args.root_path, fold=val_fold)
        writer = _summary_writer(snapshot + '/log')
        Trainer(args, recipe_for(script), model, step, batches, n, validator, snapshot, logger.info, writer, refresh).run()
    finally:
        if writer is not None:
            writer.close()
        for h in handlers:
            logger.removeHandler(h)
            h.close()
    return snapshot


if __name__ == "__main__":
    train(sys.argv[1:])
