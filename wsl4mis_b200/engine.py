"""Fused per-step training body (the hot loop of every code/train_weakly_supervised_*.py script).

``TrainStep`` replays, with the reference's arithmetic and hyper-parameters, the step body of
  pce            train_weakly_supervised_pCE_2D.py:97-108
  pce_gatedcrf   train_weakly_supervised_pCE_GatedCRFLoss_2D.py:111-130
  pce_ms         train_weakly_supervised_pCE_MumfordShah_Loss_2D.py:98-110
  pce_tv         train_weakly_supervised_pCE_TV_2D.py:109-121
  dmpls          train_weakly_supervised_segmentation_pCE_ours_proposed.py:108-132
  pce_entropy    train_weakly_supervised_pCE_Entropy_Mini_2D.py:97-109
  pce_variance   train_weakly_supervised_pCE_Inter&Intra_Class_2D.py:112-125 (weight = consistency * sigmoid_rampup(it//150, 200))
  ce_dice        train_fully_supervised_2D.py:97-105 and train_weakly_supervised_pCE_random_walker_2D.py:97-104
                 (0.5 * (CE(ignore_index=4) + DiceLoss(softmax, label)) on dense or random-walker labels)
(``S2LStep`` below adds Scribble2Label, train_s2l.py:119-157, and its ensemble refresh :214-243; ``DANStep`` the adversarial
script, train_deep_adversarial_network_2D.py:126-184, with FCDiscriminator and a device Adam; ``UAMTStep``, ``MeanTeacherStep``
and ``EntropyMinStep`` the semi-supervised scripts train_uncertainty_aware_mean_teacher_2D.py, train_mean_teacher_2D.py and
train_entropy_minimization_2D.py.  train_partially_fully_supervised.py:121-142 needs no class of its own: its body is
0.5 * (CE + Dice) on the labelled batch, the unlabelled batch is loaded and never used, and on dense labels (no pixel is 4) the
CE's ignore_index=4 of ``ce_dice`` ignores nothing, so ``TrainStep(model, 'ce_dice')`` fed the labelled batches runs it) as ONE launch sequence: executor forward -> fused loss head (softmax+pCE, regulariser, combined backward into
dlogits) -> executor backward into a flat fp32 gradient bucket -> (NCCL all-reduce of that bucket when
world_size > 1) -> fused SGD(momentum 0.9, wd 1e-4) over the flat parameter buffer with the poly LR read from
device memory.  The whole sequence is CUDA-graph captured after the first call (graph=True).

For models returning two heads (unet_cct) under a single-head script (pce_gatedcrf, ...) the loss is applied to
``main_seg`` only, as SURVEY F7 prescribes; the untouched aux decoder then has no gradient and, like
torch.optim.SGD with ``grad is None``, is skipped by the optimiser.
"""
from __future__ import annotations

import math
import os
import random

import torch

from . import ddp
from . import _lib
from ._lib import call, workspace
from .utils import ramps

VARIANTS = ("pce", "pce_gatedcrf", "pce_ms", "pce_tv", "dmpls", "pce_entropy", "pce_variance", "ce_dice")


def _flatten(params, dev):
    """One fp32 buffer holding `params` back to back, each p.data re-pointed into it (views keep the nn.Parameter objects /
    state_dict intact) -> (buffer, {id(p): (offset, numel)})."""
    flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
    offsets, off = {}, 0
    for p in params:
        flat[off:off + p.numel()].copy_(p.data.reshape(-1))
        p.data = flat[off:off + p.numel()].view_as(p)
        offsets[id(p)] = (off, p.numel())
        off += p.numel()
    return flat, offsets


def _captured(fn):
    """fn() captured into a new CUDA graph -> (graph, what fn returned)"""
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def _ramp(consistency, iter_num, period, rampup):
    """the scripts' consistency weight consistency * sigmoid_rampup(iter_num // period, rampup)"""
    return consistency * ramps.sigmoid_rampup(iter_num // period, rampup)


def _masks(model):
    """the test hooks of `model` that fix its dropout: (dropout_masks, channel_keep), None where unset"""
    return getattr(model, "dropout_masks", None), getattr(model, "channel_keep", None)


def _aux_ids(model):
    """ids of the aux decoder's parameters on a two-decoder model (unet_cct): steps that read main_seg only (SURVEY F7) skip them"""
    return {id(q) for q in model.aux_decoder1.parameters()} if len(model.executor.dec) == 2 else set()


class _FlatSGDStep:
    """What every step class shares: the flat fp32 master parameters, the fused SGD over the trained `segments` of that buffer
    with the poly LR read from device memory, and the driver `_run` that executes the subclass's
    `_fwd_bwd(*inputs, **kw) -> (loss, flat gradient bucket)`, the all-reduce and `_finish` eagerly or as captured CUDA graphs.

    Graph mode keeps `input_sets` sets of static input buffers (``input_buffers(i)``).  With two, a caller can copy batch k+1
    from pinned host memory on a copy stream while the graph of batch k runs (bench.py's end-to-end leg does).  Tensors that are
    not one of those buffers are copied into set 0.  After two eager warm-up steps one graph is captured per input set, or per
    host key for a step that passes one (such a step keeps a single input set), and replayed from then on.

    Graphs and static buffers are kept per batch shape as well: the semi-supervised scripts' loaders keep their short last
    batches (no drop_last), so an epoch of ``zip(cycle(labelled), unlabelled)`` brings up to four shape combinations.  An input
    set's buffers, and the graphs keyed by its index or host key alone, have the shape of the first batch that set saw; every
    other shape gets its own buffers and graphs, keyed by (set index or host key, input shapes), after two eager warm-up steps at
    that shape (they allocate the executor's buffers for it)."""
    aliases = ()            # attributes _fwd_bwd sets that alias graph memory: kept per graph and restored on every replay
    input_sets = 2
    nccl_in_graph = False   # world_size > 1: capture the all-reduce in the step graph instead of issuing it between two graphs
    scratch = "step"        # executor buffer namespace of `_buf`
    ramps = ramps

    def __init__(self, model, base_lr, max_iterations, momentum, weight_decay, graph, world_size, process_group, skip):
        """skip: ids of the parameters the step does not train.  Like torch.optim.SGD with grad=None, the fused optimiser leaves
        them untouched: it walks the [offset, length] `segments` of the other parameters in the flat buffer."""
        self.model, self.ex = model, model.executor
        self.base_lr, self.max_iterations = float(base_lr), int(max_iterations)
        self.momentum, self.weight_decay = float(momentum), float(weight_decay)
        self.graph_enabled = bool(graph)
        self.world_size, self.pg = int(world_size), process_group
        self.iter_num = 0
        self.dev = next(model.parameters()).device
        self.flat, self.offsets = _flatten(self.ex.params, self.dev)
        if self.world_size > 1:
            ddp.broadcast_flat(self.flat, 0, self.pg)     # identical replicas (DDP does the same at construction)
        self.mom = torch.zeros_like(self.flat)
        self.segments = []
        for p in self.ex.params:
            if id(p) in skip:
                continue
            off, n = self.offsets[id(p)]
            if self.segments and self.segments[-1][0] + self.segments[-1][1] == off:
                self.segments[-1][1] += n
            else:
                self.segments.append([off, n])
        self.n_trained = self.segments[-1][0] + self.segments[-1][1]     # prefix that holds every trained parameter (the all-reduce payload)
        self.lr_dev = torch.full((1,), self.base_lr, dtype=torch.float32, device=self.dev)
        self.launches_per_step = 0
        self._warm, self._graphs, self._static = {}, {}, [None] * self.input_sets
        self._static_other = {}     # (input set, input shapes) -> buffers of the shapes an input set was not first called with

    def _buf(self, name, shape, dtype=torch.float32):
        """the step's scratch tensor `name` of this shape (one per name, shape and dtype, kept by the executor)"""
        return self.ex.buf(self.scratch, name, shape, dtype)

    def _ce_dice(self, logits, label, ignore, ns, scale=1.0, d=None, d16=None):
        """0.5 * (CE(ignore_index=`ignore`) + DiceLoss(softmax, label)) on dense labels -> (CE, Dice, loss), 0-dim device tensors;
        `scale` times the logit gradient goes to `d` (fp32 NCHW) or `d16` (bf16 NHWC-16), scratch to buffer namespace `ns`.  The
        Dice has no ignore mask (msum = NULL): a label-4 pixel is in no class but enters the Z sums, as one_hot(4) does."""
        N, C, H, W = logits.shape
        probs, gp = self.ex.buf(ns, "ce_dice.probs", (N, C, H, W), torch.float32), self.ex.buf(ns, "ce_dice.gprobs", (N, C, H, W), torch.float32)
        st, sums = self.ex.buf(ns, "ce_dice.stats", (2,), torch.float32), self.ex.buf(ns, "ce_dice.sums", (13,), torch.float32)
        call("wsl_softmax_pce_fwd", logits, label, probs, N, C, H, W, ignore, st, workspace("pce", self.dev))
        call("wsl_pdice_fwd", probs, label, None, 1.0, N, C, H, W, sums, workspace("pdice", self.dev))
        call("wsl_pdice_bwd", probs, label, None, 1.0, sums, N, C, H, W, 0.5, 0, gp)
        call("wsl_head_bwd", probs, label, st, None, 0.5 * scale, gp, 1.0 * scale, N, C, H, W, ignore, d, d16, self.ex.dt)
        return st[0], sums[0], 0.5 * (sums[0] + st[0])

    def _opt(self, g):
        for off, n in self.segments:
            call("wsl_sgd_step", self.flat[off:], g[off:], self.mom[off:], n, self.lr_dev, self.base_lr, self.momentum,
                 self.weight_decay, 1.0 / self.world_size)

    def _allreduce(self, g):
        """sum the trained prefix of the bucket over the ranks (the SGD kernel applies the 1/world mean)"""
        if self.world_size > 1:
            ddp.allreduce_flat(g[: self.n_trained], self.pg)

    def _finish(self, g, captured):
        """the update after the all-reduce.  captured: it runs inside a graph, so host values must reach it through device memory"""
        self._opt(g)

    def _step(self, inputs, kw, captured):
        loss, g = self._fwd_bwd(*inputs, **kw)
        self._allreduce(g)
        self._finish(g, captured)
        return loss, g

    def _advance_lr(self):
        # poly LR applied after the step with the pre-increment iteration (...pCE_2D.py:106-108)
        self.lr_dev.fill_(self.base_lr * (1.0 - self.iter_num / self.max_iterations) ** 0.9)
        self.iter_num += 1

    def _run(self, inputs, key=None, **kw):
        """One training step on `inputs` (the tensors `_fwd_bwd` reads; kw: its host arguments).  `key` names the host values a
        captured graph bakes in (USTM's rot90 count); without one, graphs are keyed by input set, and by the input shapes when they
        are not that set's first shapes.  Returns the loss (0-dim device tensor)."""
        shapes = tuple(tuple(x.shape) for x in inputs)
        if self.graph_enabled:
            s = 0
            for i, st in enumerate(self._static):
                if st is not None and st[0].data_ptr() == inputs[0].data_ptr():
                    s = i
            static = self.input_buffers(s, like=inputs)
            home = tuple(tuple(b.shape) for b in static) == shapes
            if not home:
                if (s, shapes) not in self._static_other:
                    self._static_other[(s, shapes)] = tuple(torch.empty_like(x) for x in inputs)
                static = self._static_other[(s, shapes)]
            for buf, x in zip(static, inputs):
                if buf.data_ptr() != x.data_ptr():
                    buf.copy_(x, non_blocking=True)
            inputs = static
        if not self.graph_enabled or self._warm.get(shapes, 0) < 2:    # graph mode: the eager warm-up allocates every buffer / tensor map
            c0 = _lib.COUNTERS["launch_calls"]
            loss, _ = self._step(inputs, kw, False)
            self.launches_per_step = _lib.COUNTERS["launch_calls"] - c0
            self._warm[shapes] = self._warm.get(shapes, 0) + 1
        else:
            k = s if key is None else key
            if not home:
                k = (k, shapes)
            if k not in self._graphs:
                self._graphs[k] = self._capture(inputs, kw) + (tuple(getattr(self, a) for a in self.aliases),)
            g1, g2, gloss, gg, kept = self._graphs[k]
            for a, v in zip(self.aliases, kept):
                setattr(self, a, v)
            g1.replay()
            if g2 is not None:                  # two-graph mode: the all-reduce is issued from the host between the graphs
                self._allreduce(gg)
                g2.replay()
            # the captured loss lives in graph-pool memory that the next replay overwrites: hand out a copy
            # (the aliased attributes, e.g. step.outputs, still point into the pool: read them before the next step)
            loss = gloss.clone()
        self._advance_lr()
        return loss

    def _capture(self, inputs, kw):
        """Capture the step -> (graph, second graph or None, loss, gradient bucket).  world_size 1: one graph.  world_size > 1
        with nccl_in_graph: ONE graph as well, with the all-reduces captured inside it (no host round trip and no second graph
        launch between backward and optimiser); otherwise, or if this NCCL / torch build refuses to capture the collective, two
        graphs (forward+backward | update) with the all-reduce issued from the host in between."""
        torch.cuda.synchronize()
        if self.world_size > 1 and self.nccl_in_graph:
            try:
                g1, (gloss, gg) = _captured(lambda: self._step(inputs, kw, True))
                self.comm_mode = "captured in the step graph (decoder slice overlapped with the encoder backward)" if self.overlap_comm else "captured in the step graph"
                return g1, None, gloss, gg
            except Exception as e:                   # pragma: no cover - depends on the NCCL build
                self.comm_mode = f"two graphs, host-issued all-reduce (capture failed: {type(e).__name__})"
                torch.cuda.synchronize()
                self.overlap_comm = False            # a host-issued collective cannot sit inside backward()
        if self.world_size == 1:
            g1, (gloss, gg) = _captured(lambda: self._step(inputs, kw, True))
            return g1, None, gloss, gg
        if not hasattr(self, "comm_mode"):
            self.comm_mode = "two graphs, host-issued all-reduce"
        g1, (gloss, gg) = _captured(lambda: self._fwd_bwd(*inputs, **kw))
        g2, _ = _captured(lambda: self._finish(gg, True))
        return g1, g2, gloss, gg

    def input_buffers(self, idx=0, like=None):
        """The device buffers read by the graphs of input set `idx` (0 .. input_sets - 1), one per tensor the step takes."""
        if self._static[idx] is None:
            src = like if like is not None else next((st for st in self._static if st is not None), None)
            assert src is not None, "call the step once (or pass like=) before asking for input buffers"
            self._static[idx] = tuple(torch.empty_like(t) for t in src)
        return self._static[idx]

    def static_inputs(self):
        return self._static[0]


class TrainStep(_FlatSGDStep):
    aliases = ("_outs", "loss_parts")

    def __init__(self, model, variant="pce_gatedcrf", base_lr=0.01, max_iterations=30000, momentum=0.9,
                 weight_decay=1e-4, graph=True, process_group=None, world_size=1, global_batch=False):
        """global_batch (world_size > 1): reproduce the SINGLE-PROCESS arithmetic of the reference at the global batch (SURVEY 8(e)):
        BatchNorm statistics over all ranks' pixels (forward and backward all-reduce 2C floats per layer), the pCE mean over the
        labelled pixels of the whole batch, Dice ratios of batch-wide sums.  Default off = stock DDP semantics (per-rank BatchNorm
        and loss normalisers), which is what the weak-scaling benchmark runs.  The collectives are issued from the host inside the
        step, so this mode runs eagerly (no CUDA graph)."""
        assert variant in VARIANTS
        # Parameters that receive gradients in this step body: everything the executor runs except (a) the aux decoder when
        # only main_seg enters the loss (SURVEY F7) and (b) deep-supervision heads (UNet_DS: the variants use output 0 only;
        # out_conv_dp4 never runs at all).
        skip = _aux_ids(model) if variant != "dmpls" else set()
        skip.update(id(q) for nm, q in model.named_parameters() if "out_conv_dp" in nm)
        skip.update(id(p) for p in model.executor.params if id(p) not in model.executor.used_param_ids)
        super().__init__(model, base_lr, max_iterations, momentum, weight_decay, graph, world_size, process_group, skip)
        self.variant = variant
        self.global_batch = bool(global_batch) and self.world_size > 1
        if self.global_batch:
            self.graph_enabled = False
            self.ex.sync_bn = (self.world_size, self.pg)
        dev = self.dev
        self.beta_dev = torch.tensor([0.5, 0.5], dtype=torch.float32, device=dev)
        self.cw_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        self.consistency, self.consistency_rampup = 0.1, 200.0
        if variant == "pce_variance":
            self.graph_enabled = False      # the ramp weight is a launch argument of the backward kernel
        self.beta = 0.5
        self.two_heads = len(self.ex.dec) == 2
        self.n_heads_trained = 2 if (variant == "dmpls") else 1
        if variant == "dmpls":
            assert self.two_heads, "dmpls needs a two-head model (unet_cct)"
        # the encoder's parameters come first in parameters(): [0, enc_end) is final only at the very end of backward(), the
        # decoder slice [enc_end, n_trained) ~2 ms earlier -- its all-reduce is issued from inside backward() on a side stream
        self.enc_end = sum(q.numel() for q in model.encoder.parameters())
        self.overlap_comm = self.world_size > 1 and os.environ.get("WSL4MIS_NO_COMM_OVERLAP", "0") != "1"
        self.nccl_in_graph = os.environ.get("WSL4MIS_NCCL_IN_GRAPH", "0") == "1"     # opt-in: capture the collectives in the step graph
        if self.graph_enabled and not self.nccl_in_graph:
            self.overlap_comm = False        # a host-issued collective cannot sit inside the captured backward
        self.loss_parts = {}

    # ------------------------------------------------------------------
    @staticmethod
    def _dlogits(ex, slot, name, N, C, H, W):
        """(fp32 NCHW buffer or None, bf16 NHWC-16 buffer or None, what backward() receives): in bf16 mode the head
        writes the out_conv gradient directly in the executor's layout (no conversion pass)."""
        if ex.dt != 1:
            d16 = ex.buf(slot, "head." + name + ".nhwc16", (N, H, W, 16))
            return None, d16, ("nhwc16", d16)
        d = ex.buf(slot, "head." + name, (N, C, H, W), torch.float32)
        return d, None, d

    def _head_bwd(self, h, probs, stats, label, ce_w, gp, reg_w, slot):
        """head h's logit gradient ce_w * d(pCE) + reg_w * gp (gp: the regulariser's probability gradient or None), written by
        wsl_head_bwd into a `_dlogits` buffer -> what backward() receives for that head"""
        N, C, H, W = probs[h].shape
        d, d16, dl = self._dlogits(self.ex, slot, f"dl{h}", N, C, H, W)
        call("wsl_head_bwd", probs[h], label, stats[h], None, ce_w, gp, reg_w, N, C, H, W, 4, d, d16, self.ex.dt)
        return dl

    def _head(self, logits_list, image, label, slot):
        """loss head: returns (loss tensor, [dlogits per decoder or None])."""
        ex = self.ex
        N, C, H, W = logits_list[0].shape
        dev = self.dev
        B = lambda name, shape, dt=torch.float32: ex.buf(slot, "head." + name, shape, dt)
        dl = [None] * len(logits_list)
        # the 16-bit layouts receive the logit gradient already multiplied by the executor's loss scale (1 unless fp16);
        # plain fp32 NCHW gradients are scaled by the executor itself
        S = ex.grad_scale_for(N, H, W) if ex.dt != 1 else 1.0
        if self.global_batch:
            S = S * self.world_size      # the pCE term is normalised by the global count: its rank contributions ADD, while the
            #                              optimiser averages the bucket (1/world) -- every per-rank-mean term is divided back below
        G = 1.0 / self.world_size if self.global_batch else 1.0       # factor for regularisers that are per-rank MEANS (CRF, entropy)
        v = self.variant
        if self.global_batch and v in ("pce_tv", "pce_variance"):
            raise NotImplementedError(f"global_batch semantics are not defined here for '{v}' (batch-slice TV / per-sample variance ramps)")
        if self.global_batch and v == "ce_dice":
            raise NotImplementedError("global_batch semantics are not defined here for 'ce_dice' (run it with per-rank normalisers)")
        if v == "ce_dice":
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            ce, dice, loss = self._ce_dice(logits_list[0], label, 4, slot, S, d, d16)
            self.loss_parts = {"ce": ce, "dice": dice}
            return loss, dl
        heads = range(self.n_heads_trained)
        probs, stats = [], []
        for h in heads:
            p = B(f"probs{h}", (N, C, H, W))
            st = B(f"stats{h}", (2,))
            call("wsl_softmax_pce_fwd", logits_list[h], label, p, N, C, H, W, 4, st, workspace("pce", dev))
            if self.global_batch:        # mean over the labelled pixels of the GLOBAL batch: all-reduce {sum of NLL, count}
                tot = torch.stack((st[0] * st[1], st[1]))
                ddp.allreduce_flat(tot, self.pg)
                st.copy_(torch.stack((tot[0] / tot[1], tot[1])))
            probs.append(p)
            stats.append(st)
        ce = stats[0][0]
        if v == "pce":
            loss = ce
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, None, 0.0 * S, slot)
        elif v == "pce_gatedcrf":
            gp = B("gprobs0", (N, C, H, W))
            out = B("crf", (2,))
            call("wsl_gatedcrf_fwd", probs[0], image, gp, N, C, H, W, 5, 6.0, 0.1, 1.0, out, workspace("crf", dev))
            loss = ce + 0.1 * out[0]
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, gp, 0.1 * S * G, slot)
            self.loss_parts = {"ce": ce, "crf": out[0]}
        elif v == "pce_ms":
            gp = B("gprobs0", (N, C, H, W))
            out = B("ms", (1,))
            cent = B("cent", (N * C,))
            call("wsl_mumford_shah_fwd", image, probs[0], N, C, H, W, out, cent, workspace("ms", dev))
            call("wsl_mumford_shah_bwd", image, probs[0], cent, N, C, H, W, 1e-6, 0, gp)
            loss = ce + 1e-6 * out[0]
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, gp, 1.0 * S, slot)
        elif v == "pce_tv":
            # tv_loss(outputs_soft[1:]) -- batch slice, sample 0 gets no TV term (SURVEY F12)
            gp = B("gprobs0", (N, C, H, W))
            gp.zero_()
            out = B("tv", (1,))
            if N > 1:
                call("wsl_tv_loss", probs[0][1:], (N - 1) * C, H, W, 1e-2, gp[1:], out, workspace("tv", dev))
                loss = ce + 1e-2 * out[0]
            else:
                loss = ce   # mean over an empty tensor is NaN in the reference; N=1 is never used with this script
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, gp, 1.0 * S, slot)
        elif v == "pce_entropy":
            gp = B("gprobs0", (N, C, H, W))
            out = B("ent", (1,))
            call("wsl_entropy_fwd", probs[0], N, C, H, W, out, workspace("ent", dev))
            call("wsl_entropy_bwd", probs[0], N, C, H, W, 0.1, 0, gp)
            loss = ce + 0.1 * out[0]
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, gp, 1.0 * S * G, slot)
        elif v == "pce_variance":
            w = _ramp(self.consistency, self.iter_num, 150, self.consistency_rampup)
            gp = B("gprobs0", (N, C, H, W))
            out = B("var", (3,))
            st = B("varstats", (N * C * 2 + N * 2,))
            call("wsl_class_variance_fwd", image, probs[0], N, C, H, W, out, st, workspace("var", dev))
            call("wsl_class_variance_bwd", image, probs[0], st, N, C, H, W, 1.0, 0, gp)
            # the ramp weight changes every 150 iterations: it multiplies on the device side so graphs stay valid
            self.cw_dev.fill_(w)
            loss = ce + self.cw_dev[0] * out[0]
            dl[0] = self._head_bwd(0, probs, stats, label, 1.0 * S, gp, float(w) * S, slot)
        else:  # dmpls
            pseudo = B("pseudo", (N, H, W), torch.uint8)
            call("wsl_mix_argmax", probs[0], probs[1], 0.0, 0.0, self.beta_dev, N, C, H, W, pseudo)   # beta from device memory
            loss = 0.5 * (stats[0][0] + stats[1][0])
            # pDLoss weighs every pixel by the batch-summed ignore mask (F14); with pseudo labels nothing is ignored, so the weight
            # is the batch size -- the GLOBAL one when the ranks reproduce the single-process arithmetic
            nb = float(N * self.world_size) if self.global_batch else float(N)
            for h in heads:
                sums = B(f"pd{h}", (13,))
                call("wsl_pdice_fwd", probs[h], pseudo, None, nb, N, C, H, W, sums, workspace("pdice", dev))
                if self.global_batch:    # Dice is a ratio of batch-wide sums (losses.py:209-217): all-reduce {I, Y, Z} per class first
                    ddp.allreduce_flat(sums[1:], self.pg)
                    i_, y_, z_ = sums[1:5].double(), sums[5:9].double(), sums[9:13].double()
                    sums[0:1].copy_((1.0 - (2.0 * i_ + 1e-5) / (z_ + y_ + 1e-5)).mean().float().reshape(1))
                gp = B(f"gprobs{h}", (N, C, H, W))
                call("wsl_pdice_bwd", probs[h], pseudo, None, nb, sums, N, C, H, W, 0.25, 0, gp)
                loss = loss + 0.25 * sums[0]
                dl[h] = self._head_bwd(h, probs, stats, label, 0.5 * S, gp, 1.0 * S, slot)
        return loss, dl

    def _fwd_bwd(self, image, label):
        ex = self.ex
        # single-head scripts on the two-head model never read the aux output: let its forward keep running on the
        # side stream underneath the loss head and the main backward (joined at the end of the backward)
        defer = self.two_heads and self.n_heads_trained == 1
        outs, slot = ex.forward(image, True, True, *_masks(self.model), defer_join=defer)
        loss, dl = self._head(outs, image, label, slot)
        ex.on_decoders_done = self._allreduce_decoders if self.overlap_comm else None
        try:
            gflat = ex.backward(slot, dl)
        finally:
            ex.on_decoders_done = None
        self._outs = outs
        return loss, gflat

    def _allreduce_decoders(self, gflat):
        """called by the executor between the decoder and encoder halves of backward(): sum the decoder slice of the bucket on the
        'comm' side stream while the encoder's BatchNorm-backward / dgrad / wgrad chain keeps the SMs busy"""
        if self.n_trained > self.enc_end:
            with self.ex.on_side("comm"):
                ddp.allreduce_flat(gflat[self.enc_end: self.n_trained], self.pg)

    def _allreduce(self, gflat):
        """the rest of the bucket after backward(): the encoder slice (or everything when the overlap is off)"""
        if self.overlap_comm:
            # SAME stream as the decoder slice: two collectives of one communicator on different streams may be scheduled in
            # different orders on different ranks (synchronous c10d collectives run on the caller's stream) and deadlock
            with self.ex.on_side("comm"):
                ddp.allreduce_flat(gflat[: self.enc_end], self.pg)
            self.ex.join_side("comm")
        else:
            super()._allreduce(gflat)

    # ------------------------------------------------------------------
    def __call__(self, image, label):
        """image: fp32 [N,1,H,W] CUDA, label: uint8 [N,H,W] CUDA.  Returns the loss (0-dim device tensor).
        Graph mode: ``input_buffers(0/1)`` are (image, label) pairs (see `_FlatSGDStep`)."""
        assert image.is_cuda and label.is_cuda and label.dtype == torch.uint8
        self.model.train()
        if self.variant == "dmpls":
            # beta = random.random() + 1e-10 from Python's host RNG, as the script (:117); handed to the kernels through
            # device memory so the captured graph sees a fresh value every replay
            self.beta = random.random() + 1e-10
            self.beta_dev.copy_(torch.tensor([self.beta, 1.0 - self.beta], dtype=torch.float32), non_blocking=False)
        return self._run((image, label))

    @property
    def outputs(self):
        return self._outs


class _NoisyTeacher:
    """The never-updated teacher of the UAMT, MT and USTM steps (SURVEY F8): no-grad training-mode passes on noisy inputs, and the
    softmax-MSE consistency against them (K13 kernels), masked by the uncertainty of T stochastic passes (T = 0: unmasked)."""

    def __init__(self, model, T, dev, world_size, pg):
        self.model, self.ex, self.T, self.dev = model, model.executor, int(T), dev
        if world_size > 1:          # replicas start identical; the teacher is broadcast once
            for q in list(model.parameters()) + list(model.buffers()):
                ddp.broadcast_flat(q.data, 0, pg)
        from .networks._engine import initial_rng_counter
        self.seed_dev = torch.full((1,), initial_rng_counter() ^ 0x5A5A5A5A, dtype=torch.int64, device=dev)

    def _noisy(self, x, reps, salt, given):
        """x repeated `reps` times + clamp(0.1 * randn, +-0.2); given (tests): that noise"""
        if given is not None:
            return (x.repeat(reps, 1, 1, 1) + given).contiguous()
        out = torch.empty((x.shape[0] * reps,) + tuple(x.shape[1:]), dtype=torch.float32, device=self.dev)
        call("wsl_add_clamped_noise", x, x.numel(), reps, 0.1, 0.2, 0xA5A5 + salt, self.seed_dev, out)
        return out

    def __call__(self, img, noises):
        """the passes on noisy copies of img: one at batch B -> ema_out, then T/2 on the twice-repeated batch whose logits fill
        mc [T*B, C, H, W] in order (None when T = 0).  noises (tests): the 1 + T/2 noise tensors; None draws them on the device"""
        self.seed_dev.add_(1)
        B, _, H, W = img.shape
        tmasks, tck = _masks(self.model)
        ema_out = self.ex.forward(self._noisy(img, 1, 0, None if noises is None else noises[0]), True, False, tmasks, tck)[0][0]
        if not self.T:
            return ema_out, None
        mc = self.ex.buf("teacher", "mc", (self.T * B, self.ex.n_class, H, W), torch.float32)
        for i in range(self.T // 2):
            tm2 = None if tmasks is None else {k: v.repeat(2, 1, 1, 1) for k, v in tmasks.items()}
            tck2 = None if tck is None else [c.repeat(2, 1) for c in tck]
            lg = self.ex.forward(self._noisy(img, 2, 1 + i, None if noises is None else noises[1 + i]), True, False, tm2, tck2)[0][0]
            mc[2 * B * i: 2 * B * (i + 1)].copy_(lg)
        return ema_out, mc

    def consistency(self, out, teacher, thr, w, mask, d):
        """the consistency of `out` against `teacher` = (ema_out, mc), uncertainty-masked by the threshold at `thr` into `mask` when
        given -> its value (0-dim device tensor); the weight at `w` times its gradient goes to d"""
        ema_out, mc = teacher
        B, C, H, W = out.shape
        cst = self.ex.buf("teacher", "cons", (3,), torch.float32)
        call("wsl_uamt_consistency_fwd", out, ema_out, mc, self.T, B, C, H, W, thr, 0.0, mask, cst, workspace("uamt", self.dev))
        call("wsl_uamt_consistency_bwd", out, ema_out, mask, cst, w, 0.0, B, C, H, W, d)
        return cst[2]


class _TwoBatchStep(_FlatSGDStep):
    """The body the semi-supervised scripts share, on a labelled and an unlabelled batch: training forwards of the student on the
    labelled then the unlabelled batch (BatchNorm running statistics updated in that order), the `_teacher` passes, 0.5 * (Dice + CE)
    on the labelled batch (dense labels, CE without ignore_index), the unlabelled term of `_unsupervised` weighted by ramp_dev[0],
    and the backward passes of the unlabelled then the labelled batch into one bucket; then SGD at the poly learning rate.
    Two-head models use main_seg on both sides and leave the aux decoder untrained (SURVEY F7).

    graph=True: one CUDA graph per batch shape after two eager warm-up steps at that shape (see `_FlatSGDStep`); the eager step
    issues hundreds of launches from Python and is host-bound.  The script's ramps stay host arithmetic, written to ramp_dev before
    every step.  world_size > 1: batch-sharded data parallel as `TrainStep` -- every rank runs the step on its shard, the bucket is
    all-reduced (sum) over NCCL and the fused SGD applies the 1/world mean (world_size > 1 with graph=True: forward+backward |
    host-issued all-reduce | SGD).  The replicas are broadcast from rank 0 at construction, a teacher once."""
    aliases = ("parts",)
    input_sets = 1
    teacher = None          # a _NoisyTeacher: its passes on the unlabelled batch run before the losses

    def __init__(self, model, base_lr, max_iterations, consistency, consistency_rampup, momentum, weight_decay, graph, world_size,
                 process_group):
        super().__init__(model, base_lr, max_iterations, momentum, weight_decay, graph, world_size, process_group, _aux_ids(model))
        self.consistency, self.consistency_rampup = float(consistency), float(consistency_rampup)
        self.ramp_dev = torch.zeros(3, dtype=torch.float32, device=self.dev)    # {consistency weight, the step's own host scalars}
        self.parts = {}

    def _ramps(self, thr=None):
        """the consistency weight consistency * sigmoid_rampup(iter_num // 300, consistency_rampup) of the current iteration
        (UAMT :183, MT :164-165, EM :139) and the uncertainty threshold `thr`, written to ramp_dev -> their `parts` entries"""
        cw = _ramp(self.consistency, self.iter_num, 300, self.consistency_rampup)
        self.ramp_dev[:2].copy_(torch.tensor([cw, 0.0 if thr is None else thr], dtype=torch.float32))
        return {"weight": cw, "threshold": thr}

    def __call__(self, image_l, label_l, image_u, noises=None):
        """image_l/image_u: fp32 [B,1,H,W]; label_l: uint8 [B,H,W] dense.  noises (tests): list of 1 + T/2 tensors holding the
        already-clamped noise of the teacher's inputs.  Returns the loss (0-dim device tensor)."""
        self.model.train()
        if self.teacher is not None:
            self.teacher.model.train()
        ramp_parts = self._ramps()
        assert noises is None or not self.graph_enabled, "graph mode draws the teacher noise on the device"
        loss = self._run((image_l, label_l, image_u), noises=noises)
        self.parts = dict(self.parts, **ramp_parts)
        return loss

    def _softmax(self, logits, out):
        """softmax over the class axis into `out` (the pCE kernel without labels)"""
        N, C, H, W = logits.shape
        call("wsl_softmax_pce_fwd", logits, None, out, N, C, H, W, 255, self._buf("softmax.stats", (2,)), workspace("pce", self.dev))

    def _parts(self, ce, dice, supervised, term, extra):
        return {"supervised": supervised, "consistency": term, **extra}

    def _fwd_bwd(self, image_l, label_l, image_u, noises=None):
        """forward passes, losses and both backward passes; returns (loss, flat gradient bucket)"""
        ex = self.ex
        masks = _masks(self.model)
        outs_l, slot_l = ex.forward(image_l.contiguous(), True, True, *masks)
        outs_u, slot_u = ex.forward(image_u.contiguous(), True, True, *masks)
        teacher = None if self.teacher is None else self.teacher(image_u, noises)
        dl_l = self._buf("dl_l", tuple(outs_l[0].shape))
        ce, dice, supervised = self._ce_dice(outs_l[0], label_l, 255, self.scratch, d=dl_l)
        term, dl_u, extra = self._unsupervised(outs_u[0], teacher)
        loss = supervised + self.ramp_dev[0] * term
        self.parts = self._parts(ce, dice, supervised, term, extra)
        rest = [None] * (len(ex.dec) - 1)
        ex.backward(slot_u, [dl_u] + rest, zero_grads=True)
        return loss, ex.backward(slot_l, [dl_l] + rest, zero_grads=False)


class UAMTStep(_TwoBatchStep):
    """Per-step body of train_uncertainty_aware_mean_teacher_2D.py:138-197 (BASELINE config 5) on the fused kernels.

    Teacher (`ema_model`, never updated by the reference): one no-grad forward on the noisy unlabelled inputs and T/2 = 4 no-grad
    forwards on the twice-repeated noisy batch (T = 8 stochastic passes).  The unlabelled term is the uncertainty-masked
    softmax-MSE consistency (:181-189), weighted by w(t) = consistency * sigmoid_rampup(iter_num // 300, consistency_rampup) (:183),
    with the threshold of :186.  graph=True needs noises=None."""

    def __init__(self, model, ema_model, base_lr=0.01, max_iterations=30000, consistency=0.1, consistency_rampup=200.0,
                 momentum=0.9, weight_decay=1e-4, T=8, process_group=None, world_size=1, graph=False):
        super().__init__(model, base_lr, max_iterations, consistency, consistency_rampup, momentum, weight_decay, graph, world_size,
                         process_group)
        self.ema_model = ema_model
        self.teacher = _NoisyTeacher(ema_model, T, self.dev, self.world_size, self.pg)

    def _ramps(self):
        thr = (0.75 + 0.25 * ramps.sigmoid_rampup(self.iter_num, self.max_iterations)) * math.log(2)       # :186
        return super()._ramps(thr if self.teacher.T else None)

    def _unsupervised(self, out_u, teacher):
        """the consistency term -> (its value, w * its logit gradient, {"mask": the uncertainty mask or None})"""
        B, C, H, W = out_u.shape
        mask = self._buf("mask", (B, H, W), torch.uint8) if self.teacher.T else None
        dl_u = self._buf("dl_u", (B, C, H, W))
        cons = self.teacher.consistency(out_u, teacher, self.ramp_dev[1:2], self.ramp_dev[0:1], mask, dl_u)
        return cons, dl_u, {"mask": mask}


class MeanTeacherStep(UAMTStep):
    """Per-step body of train_mean_teacher_2D.py:138-180 on the fused kernels: `UAMTStep` with T = 0, no uncertainty estimate.

    Teacher (`ema_model`): one training-mode no-grad forward on unlabelled + clamp(0.1 * randn, +-0.2) (:147-149, :157-159).  The
    unlabelled term is torch.mean((softmax(student_u) - softmax(teacher))^2) (:169-170, the consistency kernels' T = 0 mode),
    weighted by w(t) = consistency * sigmoid_rampup(iter_num // 300, consistency_rampup) (:73-75, :164-165).  As written in the
    script, the teacher is never updated and never put in eval mode (update_ema_variables is defined but not called, SURVEY F8)."""

    def __init__(self, model, ema_model, base_lr=0.01, max_iterations=30000, consistency=0.1, consistency_rampup=200.0,
                 momentum=0.9, weight_decay=1e-4, world_size=1, process_group=None, graph=False, global_batch=False):
        if global_batch:
            raise NotImplementedError("global_batch semantics are not defined for the mean-teacher step (run it with per-rank normalisers)")
        super().__init__(model, ema_model, base_lr=base_lr, max_iterations=max_iterations, consistency=consistency,
                         consistency_rampup=consistency_rampup, momentum=momentum, weight_decay=weight_decay, T=0,
                         process_group=process_group, world_size=world_size, graph=graph)


class EntropyMinStep(_TwoBatchStep):
    """Per-step body of train_entropy_minimization_2D.py:121-150 on the fused kernels, with no teacher.

    The unlabelled term is losses.entropy_loss(softmax(student_u), C=4) (:141, utils/losses.py:30-36), weighted by
    w(t) = consistency * sigmoid_rampup(iter_num // 300, consistency_rampup) (:139)."""

    def __init__(self, model, base_lr=0.01, max_iterations=30000, consistency=0.1, consistency_rampup=200.0, momentum=0.9,
                 weight_decay=1e-4, world_size=1, process_group=None, graph=False, global_batch=False):
        if global_batch:
            raise NotImplementedError("global_batch semantics are not defined for the entropy-minimisation step (run it with per-rank normalisers)")
        super().__init__(model, base_lr, max_iterations, consistency, consistency_rampup, momentum, weight_decay, graph, world_size,
                         process_group)

    def _unsupervised(self, out_u, teacher):
        B, C, H, W = out_u.shape
        probs, ent = self._buf("probs_u", (B, C, H, W)), self._buf("ent", (1,))
        self._softmax(out_u, probs)
        call("wsl_entropy_fwd", probs, B, C, H, W, ent, workspace("ent", self.dev))
        gp, dl_u = self._buf("gprobs_u", (B, C, H, W)), self._buf("dl_u", (B, C, H, W))
        call("wsl_entropy_bwd", probs, B, C, H, W, 1.0, 0, gp)
        # the ramp weight scales the probability gradient from device memory, so one captured graph serves every iteration
        # (wsl_entropy_bwd takes its scale as a launch argument, and wsl_head_bwd's grad_out scales the CE term only)
        gp.mul_(self.ramp_dev[0])
        call("wsl_head_bwd", probs, None, None, None, 0.0, gp, 1.0, B, C, H, W, 255, dl_u, None, self.ex.dt)
        return ent[0], dl_u, {"mask": None}


class USTMStep(_FlatSGDStep):
    """Per-step body of train_weakly_supervised_ustm_2D.py:113-170: pCE on scribbles + uncertainty-aware self-ensembling with a
    random rot90 transform (Python host RNG, :123) and the EMA teacher update the script really performs (:163).  The teacher's
    passes and the consistency are `UAMTStep`'s, on the rotated batch.

    graph=True: the rot90 count is a kernel ARGUMENT, so one CUDA graph is captured per count (at most four, each on the first
    step that draws it after two eager warm-up steps); threshold, consistency weight and the EMA factor reach the captured
    kernels through `ramp_dev`."""
    aliases = ("parts",)
    input_sets = 1          # graphs are keyed by the rot90 count alone

    def __init__(self, model, ema_model, base_lr=0.01, max_iterations=60000, ema_decay=0.99, *, consistency=0.1,
                 consistency_rampup=200.0, momentum=0.9, weight_decay=1e-4, T=8, process_group=None, world_size=1, graph=False):
        """The keywords after ema_decay are `UAMTStep`'s; consistency and consistency_rampup are accepted and unused (the script's
        weight ramp is fixed, :145)."""
        super().__init__(model, base_lr, max_iterations, momentum, weight_decay, graph, world_size, process_group, _aux_ids(model))
        self.ema_model = ema_model
        self.teacher = _NoisyTeacher(ema_model, T, self.dev, self.world_size, self.pg)
        self.ema_decay = float(ema_decay)
        self.tflat, _ = _flatten(self.teacher.ex.params, self.dev)
        self.ramp_dev = torch.zeros(3, dtype=torch.float32, device=self.dev)     # {threshold, weight, 1 - EMA alpha}

    def _ramps(self):
        cw = _ramp(1.0, self.iter_num, 1000, 60)                                 # :145
        thr = (0.75 + 0.25 * ramps.sigmoid_rampup(self.iter_num, self.max_iterations)) * math.log(2)     # :148
        alpha = min(1 - 1 / (self.iter_num + 1), self.ema_decay)         # :63, global_step = iter_num before the increment
        self.ramp_dev.copy_(torch.tensor([thr, cw, 1.0 - alpha], dtype=torch.float32))
        return thr, cw, alpha

    def _finish(self, g, captured):
        """SGD on the student, then the EMA teacher update (:163): eager with the host alpha, captured with the factor from ramp_dev"""
        self._opt(g)
        n = min(self.tflat.numel(), self.flat.numel())
        if captured:
            self.tflat[:n].lerp_(self.flat[:n], self.ramp_dev[2])        # t + (1 - alpha) * (s - t)
        else:
            call("wsl_ema_update", self.tflat, self.flat, n, float(self._alpha))

    def __call__(self, image, label, noises=None, rot_times=None):
        self.model.train()
        self.ema_model.train()
        assert image.shape[2] == image.shape[3], "rot90 consistency needs square inputs"
        self.rot_times = random.randrange(0, 4) if rot_times is None else int(rot_times)
        thr, cw, self._alpha = self._ramps()
        assert noises is None or not self.graph_enabled, "graph mode draws the teacher noise on the device"
        loss = self._run((image, label), key=self.rot_times, noises=noises)
        self.parts = dict(self.parts, weight=cw, threshold=thr)
        return loss

    def _fwd_bwd(self, image, label, noises=None):
        ex, dev, k = self.ex, self.dev, self.rot_times
        outs, slot = ex.forward(image.contiguous(), True, True, *_masks(self.model))
        out = outs[0]
        B, C, H, W = out.shape
        rimg = self._buf("rimg", (B, 1, H, W))
        call("wsl_rot90", image.contiguous(), B, H, k, 0, rimg)
        teacher = self.teacher(rimg, noises)
        # pCE (ignore_index 4)
        probs, st = self._buf("probs", (B, C, H, W)), self._buf("stats", (2,))
        call("wsl_softmax_pce_fwd", out, label, probs, B, C, H, W, 4, st, workspace("pce", dev))
        d = self._buf("dl", (B, C, H, W))
        call("wsl_head_bwd", probs, label, st, None, 1.0, None, 0.0, B, C, H, W, 4, d, None, self.ex.dt)
        # consistency on the rotated student logits; threshold (:148) / weight (:145) from ramp_dev
        rout, dr, mask = self._buf("rout", (B, C, H, W)), self._buf("dr", (B, C, H, W)), self._buf("mask", (B, H, W), torch.uint8)
        call("wsl_rot90", out, B * C, H, k, 0, rout)
        cons = self.teacher.consistency(rout, teacher, self.ramp_dev[0:1], self.ramp_dev[1:2], mask, dr)
        call("wsl_rot90", dr, B * C, H, (4 - k) % 4, 1, d)              # rotate the gradient back and add it to the pCE part
        loss = st[0] + self.ramp_dev[1] * cons
        self.parts = {"ce": st[0], "consistency": cons, "mask": mask}
        g = ex.backward(slot, [d] + [None] * (len(ex.dec) - 1))
        return loss, g


class S2LStep(TrainStep):
    """Per-step body of train_s2l.py:119-157 (Scribble2Label) on the fused kernels, plus its ensemble refresh (:214-243).

    Step: pCE on the scribbles (ignore_index 4); from iteration `thr_iter` on (pre-increment counter, :125) plus 0.5 * CE on the
    u-labels derived from the augmented prediction memory (`weight`, [B,H,W,4]) where scribble == 4 and weight > thr_conf.  Both
    terms, their u-label map and the combined logit gradient come from two kernels; thr_conf and the before/after-thr_iter switch
    live in device memory (`ctrl`), so graph=True captures one graph that serves the whole run.  SGD / poly LR as TrainStep.

    Only single-output models run this script (softmax(model(img)), :228); multi-GPU Scribble2Label is not supported."""

    def __init__(self, model, thr_iter=6000, thr_conf=0.8, base_lr=0.01, max_iterations=60000, momentum=0.9, weight_decay=1e-4,
                 graph=True, world_size=1, **kw):
        if int(world_size) != 1:
            raise NotImplementedError("Scribble2Label runs on one GPU (world_size must be 1)")
        ex = model.executor
        if len(ex.dec) != 1 or any(ex.ds_heads) or not hasattr(ex, "enc_blocks"):
            raise ValueError("Scribble2Label needs a single-output U-Net (train_s2l.py:228 takes softmax(model(img)))")
        super().__init__(model, "pce", base_lr=base_lr, max_iterations=max_iterations, momentum=momentum, weight_decay=weight_decay,
                         graph=graph, **kw)
        self.thr_iter, self.thr_conf = int(thr_iter), float(thr_conf)
        self.ctrl = torch.tensor([self.thr_conf, 0.0], dtype=torch.float32, device=self.dev)    # {thr_conf, w_u}
        self._w_u = 0.0
        self._weight = None

    def _fwd_bwd(self, image, label, weight):
        self._weight = weight.contiguous()          # read by _head
        return super()._fwd_bwd(image, label)

    def _head(self, logits_list, image, label, slot):
        ex = self.ex
        N, C, H, W = logits_list[0].shape
        S = ex.grad_scale_for(N, H, W) if ex.dt != 1 else 1.0
        probs = ex.buf(slot, "head.probs0", (N, C, H, W), torch.float32)
        ulab = ex.buf(slot, "head.ulab", (N, H, W), torch.uint8)
        st = ex.buf(slot, "head.s2l", (5,), torch.float32)
        call("wsl_s2l_fwd", logits_list[0], label, self._weight, self.ctrl, N, C, H, W, probs, ulab, st, workspace("s2l", self.dev))
        d, d16, dl0 = self._dlogits(ex, slot, "dl0", N, C, H, W)
        call("wsl_s2l_head_bwd", probs, label, ulab, st, self.ctrl, S, N, C, H, W, d, d16, ex.dt)
        self.loss_parts = {"ce": st[0], "u": st[2], "u_labels": ulab}
        return st[4], [dl0]

    def __call__(self, image, scribble, weight):
        """image fp32 [N,1,H,W], scribble uint8 [N,H,W] (4 = unlabelled), weight fp32 [N,H,W,4] (S2LLoader's batch).  Returns the
        loss (0-dim device tensor): NaN after thr_iter when no unlabelled pixel clears thr_conf, as the reference.
        Graph mode: ``input_buffers(0/1)`` are (image, scribble, weight) triples."""
        assert image.is_cuda and scribble.is_cuda and scribble.dtype == torch.uint8
        assert weight.is_cuda and weight.dtype == torch.float32 and tuple(weight.shape) == (image.shape[0],) + tuple(image.shape[2:]) + (4,)
        w_u = 0.5 if self.iter_num >= self.thr_iter else 0.0
        if w_u != self._w_u:
            self.ctrl[1].fill_(w_u)
            self._w_u = w_u
        self.model.train()
        return self._run((image, scribble, weight))

    @torch.no_grad()
    def refresh(self, store, alpha=0.2, chunk=64, size=256, masks=None):
        """Ensemble refresh of train_s2l.py:221-243 into ``store.weight_live``: for every training slice in dataset order,
        zoom(order 0) to size x size, softmax(model(img)) in TRAIN mode at batch 1 (BatchNorm on that slice's own statistics,
        running statistics updated once per slice, dropout on), zoom back (order 0) and w = alpha*p + (1-alpha)*w.

        Here `chunk` slices run as ONE per-sample-BatchNorm forward (exactly what `chunk` batch-1 training forwards compute, the
        running statistics updated in slice order across chunks); one kernel then does softmax at the back-zoom source pixel
        and the EMA.  masks (tests): dropout keep masks {encoder block: uint8 [len(store), h, w, C]} for the whole pass."""
        assert store.weight_live is not None, "the store has no prediction memory (SliceStore.from_arrays(..., scribbles=))"
        self.model.train()
        n, dev = len(store), store.images.device
        a, b = float(alpha), float(1.0 - alpha)
        for s in range(0, n, int(chunk)):
            idx = list(range(s, min(n, s + int(chunk))))
            B = len(idx)
            tab = store.table(idx, [(0, 0, 0, 0, 0)] * B)          # mode 0: zoom(order 0) only (:223-224)
            img = torch.empty(B, 1, size, size, dtype=torch.float32, device=dev)
            lab = torch.empty(B, size, size, dtype=torch.uint8, device=dev)
            call("wsl_augment_batch", store.images, store.labels, tab, B, size, size, img, lab)
            mk = None if masks is None else {k: v[s: s + B] for k, v in masks.items()}
            outs, _ = self.ex.forward(img, True, False, mk, None, bn_per_sample=True)
            max_hw = int(max(int(store.shapes[i, 0]) * int(store.shapes[i, 1]) for i in idx))
            call("wsl_s2l_refresh", outs[0], tab, B, size, max_hw, a, b, store.weight_live)


class DANStep(_TwoBatchStep):
    """Per-step body of train_deep_adversarial_network_2D.py:126-184 (adversarial semi-supervised training with FCDiscriminator).

    Phase 1 (`_fwd_bwd`, :138-160; student in training mode, D in eval mode): the two-batch body of `_TwoBatchStep` with the
    unlabelled term w(t) * CE(D(softmax(out_u), image_u), DAN_target[:B_u]), w(t) = consistency * sigmoid_rampup(iter_num // 150,
    rampup).  That term reaches the student through D's map gradient and the softmax Jacobian; D's own parameter gradients, which
    the script discards (:176), are not computed.  Then SGD (momentum 0.9, weight decay 1e-4) at the poly learning rate.
    Phase 2 (`_finish`, :162-178; student in eval mode, D in training mode with fresh Dropout2d masks): no-grad eval forwards of both
    halves on the updated weights, D on cat(softmax_l, softmax_u) against [1]*B_l + [0]*B_u, and one Adam step of D
    (`wsl_adam_step`, torch's multi-tensor arithmetic) over D's parameters, which live in one flat buffer (`dflat`).

    D's operands are packed once per iteration, at the top of the step, into the executor's resident buffers; both phases read them
    (D's weights change only in the Adam step at the end), and a `load_state_dict` between steps is picked up.  graph=True captures
    the whole iteration as one CUDA graph per batch shape after two eager warm-up steps at that shape: the first batch, a full one
    with B_u == B_l, and after it an epoch's shorter last batches; the ramp weight and Adam's t-dependent scalars are written to `ramp_dev` before every step.  The modules' train() / eval() flags are not touched: each pass runs in the script's mode.
    Test hooks: `model.dropout_masks` (phase 1) and `disc.channel_keep` (phase 2, [B_l + B_u, C] masks) as for the modules."""
    scratch = "dan"

    def __init__(self, model, disc, base_lr=0.01, max_iterations=30000, consistency=0.1, consistency_rampup=200.0, disc_lr=1e-4,
                 betas=(0.9, 0.99), graph=True, world_size=1):
        if int(world_size) != 1:
            raise NotImplementedError("DANStep runs on one GPU (world_size must be 1): the adversarial script has no multi-GPU form")
        ex = model.executor
        if len(getattr(ex, "dec", ())) != 1 or any(getattr(ex, "ds_heads", ())):
            raise ValueError("DANStep needs a single-output segmentation network: the script takes torch.softmax(model(x), dim=1) "
                             "(train_deep_adversarial_network_2D.py:143-144), which fails on a tuple of outputs")
        super().__init__(model, base_lr, max_iterations, consistency, consistency_rampup, 0.9, 1e-4, graph, 1, None)
        self.disc, self.dex = disc, disc.executor
        if next(disc.parameters()).device != self.dev:
            raise ValueError(f"DANStep: the discriminator is on {next(disc.parameters()).device}, the model on {self.dev}")
        self.dflat, self.doffsets = _flatten(list(disc.parameters()), self.dev)
        self.dgrad = torch.zeros_like(self.dflat)
        self.exp_avg, self.exp_avg_sq = torch.zeros_like(self.dflat), torch.zeros_like(self.dflat)
        self.adam_t = 0
        self.disc_lr, self.betas, self.eps = float(disc_lr), (float(betas[0]), float(betas[1])), 1e-8

    def __call__(self, image_l, label_l, image_u):
        """image_l / image_u: fp32 [B_l,1,256,256] / [B_u,1,256,256]; label_l: uint8 [B_l,256,256] dense.  Returns the phase-1 loss
        (0-dim device tensor); `parts` holds loss_ce, loss_dice, consistency (the adversarial CE), weight and disc_loss."""
        from .networks.discriminator import HW
        for name, t in (("image_l", image_l), ("image_u", image_u)):
            if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 4 and tuple(t.shape[1:]) == (self.disc.n_channel, HW, HW)):
                raise ValueError(f"DANStep: {name} must be a CUDA fp32 [N, {self.disc.n_channel}, {HW}, {HW}] tensor (got "
                                 f"{tuple(t.shape)} {t.dtype}); FCDiscriminator's kernels take the scripts' 256 x 256 patches")
        if not (label_l.is_cuda and label_l.dtype == torch.uint8 and tuple(label_l.shape) == (image_l.shape[0], HW, HW)):
            raise ValueError(f"DANStep: label_l must be a CUDA uint8 [{image_l.shape[0]}, {HW}, {HW}] tensor (got {tuple(label_l.shape)})")
        if self.graph_enabled and not self._warm and image_u.shape[0] != image_l.shape[0]:
            raise ValueError(f"DANStep(graph=True) takes its first batch as the full batch and needs B_u == B_l there (got "
                             f"{image_u.shape[0]} and {image_l.shape[0]}); an epoch's shorter last batches may follow, each captured "
                             f"in its own graph")
        cw = _ramp(self.consistency, self.iter_num, 150, self.consistency_rampup)     # :151-152
        t = self.adam_t + 1
        b1, b2 = self.betas
        step_size, bc2_sqrt = self.disc_lr / (1 - b1 ** t), (1 - b2 ** t) ** 0.5          # as torch's Adam computes them (doubles)
        self.ramp_dev.copy_(torch.tensor([cw, step_size, bc2_sqrt], dtype=torch.float32))
        loss = self._run((image_l, label_l, image_u))
        self.adam_t = t
        self.parts = dict(self.parts, weight=cw)
        return loss

    def _fwd_bwd(self, image_l, label_l, image_u):
        """phase 1 -> (loss, student gradient bucket)"""
        self._inputs = (image_l, image_u)
        self._dpacks = self.dex.pack_resident(self.dev)
        return super()._fwd_bwd(image_l, label_l, image_u)

    def _unsupervised(self, out_u, teacher):
        """the adversarial term (:151-157): D in eval mode on softmax(out_u); its gradient w.r.t. the map only"""
        B, Bu = self._inputs[0].shape[0], out_u.shape[0]
        _, C, H, W = out_u.shape
        pu = self._buf("probs_u", (Bu, C, H, W))
        self._softmax(out_u, pu)
        logits, rec = self.dex.forward(pu, self._inputs[1].contiguous(), False, True, True, None, packs=self._dpacks)
        adv, dlg = self._buf("adv", (1,)), self._buf("dlogits_u", (Bu, 2))
        call("wsl_disc_ce", logits, Bu, min(B, Bu), self.ramp_dev[0:1], 0.0, adv, dlg)
        dmap, _, _ = self.dex.backward(rec, dlg, True, False, param_grads=False)
        dl_u = self._buf("dl_u", (Bu, C, H, W))
        call("wsl_head_bwd", pu, None, None, None, 0.0, dmap, 1.0, Bu, C, H, W, 255, dl_u, None, self.ex.dt)
        return adv[0], dl_u, {}

    def _parts(self, ce, dice, supervised, term, extra):
        return {"loss_ce": ce, "loss_dice": dice, "consistency": term}

    def _finish(self, g, captured):
        """student SGD (:158-160), then phase 2 (:162-178) and D's Adam step; host scalars come from ramp_dev in both modes"""
        self._opt(g)
        ex, dex = self.ex, self.dex
        image_l, image_u = self._inputs
        B, _, H, W = image_l.shape
        N = B + image_u.shape[0]
        maps, imgs = self._buf("maps", (N, ex.n_class, H, W)), self._buf("imgs", (N, 1, H, W))
        self._softmax(ex.forward(image_l.contiguous(), False, False)[0][0], maps[:B])
        self._softmax(ex.forward(image_u.contiguous(), False, False)[0][0], maps[B:])
        imgs[:B].copy_(image_l)
        imgs[B:].copy_(image_u)
        logits, rec = dex.forward(maps, imgs, True, True, False, getattr(self.disc, "channel_keep", None), packs=self._dpacks)
        dloss, dlg = self._buf("disc_loss", (1,)), self._buf("dlogits_d", (N, 2))
        call("wsl_disc_ce", logits, N, B, None, 1.0, dloss, dlg)
        dex.backward(rec, dlg, False, False, bucket=(self.dgrad, self.doffsets))
        b1, b2 = self.betas
        call("wsl_adam_step", self.dflat, self.dgrad, self.exp_avg, self.exp_avg_sq, self.dflat.numel(), self.ramp_dev[1:3], 0.0, 0.0,
             b1, b2, self.eps)
        self.parts["disc_loss"] = dloss[0]
