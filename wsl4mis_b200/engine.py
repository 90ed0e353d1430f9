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
(``S2LStep`` below adds Scribble2Label, train_s2l.py:119-157, and its ensemble refresh :214-243) as ONE launch sequence: executor forward -> fused loss head (softmax+pCE, regulariser, combined backward into
dlogits) -> executor backward into a flat fp32 gradient bucket -> (NCCL all-reduce of that bucket when
world_size > 1) -> fused SGD(momentum 0.9, wd 1e-4) over the flat parameter buffer with the poly LR read from
device memory.  The whole sequence is CUDA-graph captured after the first call (graph=True).

For models returning two heads (unet_cct) under a single-head script (pce_gatedcrf, ...) the loss is applied to
``main_seg`` only, as SURVEY F7 prescribes; the untouched aux decoder then has no gradient and, like
torch.optim.SGD with ``grad is None``, is skipped by the optimiser.
"""
from __future__ import annotations

import os
import random

import torch

from . import ddp
from . import _lib
from ._lib import call, workspace

VARIANTS = ("pce", "pce_gatedcrf", "pce_ms", "pce_tv", "dmpls", "pce_entropy", "pce_variance", "ce_dice")


class TrainStep:
    def __init__(self, model, variant="pce_gatedcrf", base_lr=0.01, max_iterations=30000, momentum=0.9,
                 weight_decay=1e-4, graph=True, process_group=None, world_size=1, global_batch=False):
        """global_batch (world_size > 1): reproduce the SINGLE-PROCESS arithmetic of the reference at the global batch (SURVEY 8(e)):
        BatchNorm statistics over all ranks' pixels (forward and backward all-reduce 2C floats per layer), the pCE mean over the
        labelled pixels of the whole batch, Dice ratios of batch-wide sums.  Default off = stock DDP semantics (per-rank BatchNorm
        and loss normalisers), which is what the weak-scaling benchmark runs.  The collectives are issued from the host inside the
        step, so this mode runs eagerly (no CUDA graph)."""
        assert variant in VARIANTS
        self.model, self.variant = model, variant
        self.ex = model.executor
        self.base_lr, self.max_iterations = float(base_lr), int(max_iterations)
        self.momentum, self.weight_decay = float(momentum), float(weight_decay)
        self.graph_enabled = bool(graph)
        self.world_size = int(world_size)
        self.pg = process_group
        self.global_batch = bool(global_batch) and self.world_size > 1
        if self.global_batch:
            self.graph_enabled = False
            self.ex.sync_bn = (self.world_size, self.pg)
        self.iter_num = 0
        self._graphs = [None, None]
        self._warm = 0
        self._static = [None, None]
        dev = next(model.parameters()).device
        self.dev = dev
        # flat fp32 master parameters (views keep the nn.Parameter objects / state_dict intact)
        params = self.ex.params
        n = sum(p.numel() for p in params)
        self.flat = torch.empty(n, dtype=torch.float32, device=dev)
        off = 0
        self.offsets = {}
        for p in params:
            self.flat[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + p.numel()].view_as(p)
            self.offsets[id(p)] = (off, p.numel())
            off += p.numel()
        if self.world_size > 1:
            ddp.broadcast_flat(self.flat, 0, self.pg)     # identical replicas (DDP does the same at construction)
        self.mom = torch.zeros_like(self.flat)
        self.lr_dev = torch.full((1,), self.base_lr, dtype=torch.float32, device=dev)
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
        # Parameters that receive gradients in this step body: everything the executor runs except (a) the aux decoder when
        # only main_seg enters the loss (SURVEY F7) and (b) deep-supervision heads (UNet_DS: the variants use output 0 only;
        # out_conv_dp4 never runs at all).  Like torch.optim.SGD with grad=None, the fused optimiser leaves those untouched:
        # it walks the contiguous segments of trained parameters in the flat buffer.
        skip = set()
        if self.two_heads and self.n_heads_trained == 1:
            skip.update(id(q) for q in self.model.aux_decoder1.parameters())
        skip.update(id(q) for nm, q in model.named_parameters() if "out_conv_dp" in nm)
        self.segments = []
        for p in params:
            if id(p) in skip or id(p) not in self.ex.used_param_ids:
                continue
            off_p, n_p = self.offsets[id(p)]
            if self.segments and self.segments[-1][0] + self.segments[-1][1] == off_p:
                self.segments[-1][1] += n_p
            else:
                self.segments.append([off_p, n_p])
        self.n_trained = self.segments[-1][0] + self.segments[-1][1]     # prefix that holds every trained parameter (the all-reduce payload)
        # the encoder's parameters come first in parameters(): [0, enc_end) is final only at the very end of backward(), the
        # decoder slice [enc_end, n_trained) ~2 ms earlier -- its all-reduce is issued from inside backward() on a side stream
        self.enc_end = sum(q.numel() for q in model.encoder.parameters())
        self.overlap_comm = self.world_size > 1 and os.environ.get("WSL4MIS_NO_COMM_OVERLAP", "0") != "1"
        self.nccl_in_graph = os.environ.get("WSL4MIS_NCCL_IN_GRAPH", "0") == "1"     # opt-in: capture the collectives in the step graph
        if self.graph_enabled and not self.nccl_in_graph:
            self.overlap_comm = False        # a host-issued collective cannot sit inside the captured backward
        self.loss_parts = {}
        self.launches_per_step = 0

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
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, None, 0.0 * S, N, C, H, W, 4, d, d16, self.ex.dt)
        elif v == "pce_gatedcrf":
            gp = B("gprobs0", (N, C, H, W))
            out = B("crf", (2,))
            call("wsl_gatedcrf_fwd", probs[0], image, gp, N, C, H, W, 5, 6.0, 0.1, 1.0, out, workspace("crf", dev))
            loss = ce + 0.1 * out[0]
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, gp, 0.1 * S * G, N, C, H, W, 4, d, d16, self.ex.dt)
            self.loss_parts = {"ce": ce, "crf": out[0]}
        elif v == "pce_ms":
            gp = B("gprobs0", (N, C, H, W))
            out = B("ms", (1,))
            cent = B("cent", (N * C,))
            call("wsl_mumford_shah_fwd", image, probs[0], N, C, H, W, out, cent, workspace("ms", dev))
            call("wsl_mumford_shah_bwd", image, probs[0], cent, N, C, H, W, 1e-6, 0, gp)
            loss = ce + 1e-6 * out[0]
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, gp, 1.0 * S, N, C, H, W, 4, d, d16, self.ex.dt)
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
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, gp, 1.0 * S, N, C, H, W, 4, d, d16, self.ex.dt)
        elif v == "pce_entropy":
            gp = B("gprobs0", (N, C, H, W))
            out = B("ent", (1,))
            call("wsl_entropy_fwd", probs[0], N, C, H, W, out, workspace("ent", dev))
            call("wsl_entropy_bwd", probs[0], N, C, H, W, 0.1, 0, gp)
            loss = ce + 0.1 * out[0]
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, gp, 1.0 * S * G, N, C, H, W, 4, d, d16, self.ex.dt)
        elif v == "pce_variance":
            from .utils import ramps
            w = self.consistency * ramps.sigmoid_rampup(self.iter_num // 150, self.consistency_rampup)
            gp = B("gprobs0", (N, C, H, W))
            out = B("var", (3,))
            st = B("varstats", (N * C * 2 + N * 2,))
            call("wsl_class_variance_fwd", image, probs[0], N, C, H, W, out, st, workspace("var", dev))
            call("wsl_class_variance_bwd", image, probs[0], st, N, C, H, W, 1.0, 0, gp)
            # the ramp weight changes every 150 iterations: it multiplies on the device side so graphs stay valid
            self.cw_dev.fill_(w)
            loss = ce + self.cw_dev[0] * out[0]
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 1.0 * S, gp, float(w) * S, N, C, H, W, 4, d, d16, self.ex.dt)
        elif v == "ce_dice":
            # DiceLoss(4)(softmax, label) has no ignore mask and no F14 weighting: pDLoss kernels with msum = NULL, mconst = 1
            # (a label-4 pixel is in no class but its probabilities still enter the Z sums, as one_hot(4) does in the reference)
            sums = B("dice0", (13,))
            call("wsl_pdice_fwd", probs[0], label, None, 1.0, N, C, H, W, sums, workspace("pdice", dev))
            gp = B("gprobs0", (N, C, H, W))
            call("wsl_pdice_bwd", probs[0], label, None, 1.0, sums, N, C, H, W, 0.5, 0, gp)
            loss = 0.5 * (ce + sums[0])
            d, d16, dl[0] = self._dlogits(ex, slot, "dl0", N, C, H, W)
            call("wsl_head_bwd", probs[0], label, stats[0], None, 0.5 * S, gp, 1.0 * S, N, C, H, W, 4, d, d16, self.ex.dt)
            self.loss_parts = {"ce": ce, "dice": sums[0]}
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
                d, d16, dl[h] = self._dlogits(ex, slot, f"dl{h}", N, C, H, W)
                call("wsl_head_bwd", probs[h], label, stats[h], None, 0.5 * S, gp, 1.0 * S, N, C, H, W, 4, d, d16, self.ex.dt)
        return loss, dl

    def _fwd_bwd(self, image, label):
        ex = self.ex
        c0 = _lib.COUNTERS["launch_calls"]
        # single-head scripts on the two-head model never read the aux output: let its forward keep running on the
        # side stream underneath the loss head and the main backward (joined at the end of the backward)
        defer = self.two_heads and self.n_heads_trained == 1
        outs, slot = ex.forward(image, True, True, getattr(self.model, "dropout_masks", None),
                                getattr(self.model, "channel_keep", None), defer_join=defer)
        loss, dl = self._head(outs, image, label, slot)
        ex.on_decoders_done = self._allreduce_decoders if self.overlap_comm else None
        try:
            gflat = ex.backward(slot, dl)
        finally:
            ex.on_decoders_done = None
        self._outs = outs
        self.launches_per_step = _lib.COUNTERS["launch_calls"] - c0 + 1     # + the SGD kernel (also inside the graph)
        return loss, gflat

    def _opt(self, gflat):
        for off, n in self.segments:
            call("wsl_sgd_step", self.flat[off:], gflat[off:], self.mom[off:], n, self.lr_dev, self.base_lr, self.momentum,
                 self.weight_decay, 1.0 / self.world_size)

    def _allreduce_decoders(self, gflat):
        """called by the executor between the decoder and encoder halves of backward(): sum the decoder slice of the bucket on the
        'comm' side stream while the encoder's BatchNorm-backward / dgrad / wgrad chain keeps the SMs busy"""
        if self.n_trained > self.enc_end:
            with self.ex.on_side("comm"):
                ddp.allreduce_flat(gflat[self.enc_end: self.n_trained], self.pg)

    def _allreduce(self, gflat):
        """the rest of the bucket after backward(): the encoder slice (or everything when the overlap is off)"""
        if self.world_size > 1:
            if self.overlap_comm:
                # SAME stream as the decoder slice: two collectives of one communicator on different streams may be scheduled in
                # different orders on different ranks (synchronous c10d collectives run on the caller's stream) and deadlock
                with self.ex.on_side("comm"):
                    ddp.allreduce_flat(gflat[: self.enc_end], self.pg)
                self.ex.join_side("comm")
            else:
                ddp.allreduce_flat(gflat[: self.n_trained], self.pg)

    # ------------------------------------------------------------------
    def __call__(self, image, label):
        """image: fp32 [N,1,H,W] CUDA, label: uint8 [N,H,W] CUDA.  Returns the loss (0-dim device tensor).

        Graph mode keeps TWO sets of static input buffers (``input_buffers(0/1)``) with one captured graph each, so a
        caller can copy batch k+1 from pinned host memory on a copy stream while the graph of batch k runs
        (bench.py's end-to-end leg does).  Tensors that are not one of those buffers are copied into set 0."""
        assert image.is_cuda and label.is_cuda and label.dtype == torch.uint8
        self.model.train()
        if self.variant == "dmpls":
            # beta = random.random() + 1e-10 from Python's host RNG, as the script (:117); handed to the kernels through
            # device memory so the captured graph sees a fresh value every replay
            self.beta = random.random() + 1e-10
            self.beta_dev.copy_(torch.tensor([self.beta, 1.0 - self.beta], dtype=torch.float32), non_blocking=False)
        if not self.graph_enabled:
            loss, g = self._fwd_bwd(image, label)
            self._allreduce(g)
            self._opt(g)
        else:
            idx = 0
            for i, st in enumerate(self._static):
                if st is not None and st[0].data_ptr() == image.data_ptr():
                    idx = i
            simg, slab = self.input_buffers(idx, like=(image, label))
            assert simg.shape == image.shape, "graph mode needs a fixed batch shape"
            if simg.data_ptr() != image.data_ptr():
                simg.copy_(image, non_blocking=True)
            if slab.data_ptr() != label.data_ptr():
                slab.copy_(label, non_blocking=True)
            if self._warm < 2:                      # eager warm-up allocates every buffer / tensor map
                loss, g = self._fwd_bwd(simg, slab)
                self._allreduce(g)
                self._opt(g)
                self._warm += 1
            else:
                if self._graphs[idx] is None:
                    self._graphs[idx] = self._capture(simg, slab)
                g1, g2, gloss, gg, self._outs, self.loss_parts = self._graphs[idx]
                g1.replay()
                if g2 is not None:                  # two-graph fallback: NCCL issued from the host between the graphs
                    self._allreduce(gg)
                    g2.replay()
                # the captured loss lives in graph-pool memory that the next replay overwrites: hand out a copy
                # (step.outputs / step.loss_parts still alias the pool: read them before the next step)
                loss = gloss.clone()
        # poly LR applied after the step with the pre-increment iteration (...pCE_2D.py:106-108)
        lr_ = self.base_lr * (1.0 - self.iter_num / self.max_iterations) ** 0.9
        self.lr_dev.fill_(lr_)
        self.iter_num += 1
        return loss

    def _capture(self, simg, slab):
        """Capture the step.  world_size 1: one graph.  world_size > 1: ONE graph as well, with the NCCL all-reduces captured
        inside it (decoder slice on a side branch under the encoder's backward, encoder slice + SGD at the end) -- no host round
        trip and no second graph launch between backward and optimiser; if this NCCL / torch build refuses to capture the
        collective, fall back to two graphs with the all-reduce issued from the host in between."""
        torch.cuda.synchronize()
        if self.world_size > 1 and self.nccl_in_graph:
            try:
                g1 = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g1):
                    gloss, gg = self._fwd_bwd(simg, slab)
                    self._allreduce(gg)
                    self._opt(gg)
                self.comm_mode = "captured in the step graph (decoder slice overlapped with the encoder backward)" if self.overlap_comm else "captured in the step graph"
                return (g1, None, gloss, gg, self._outs, dict(self.loss_parts))
            except Exception as e:                   # pragma: no cover - depends on the NCCL build
                self.comm_mode = f"two graphs, host-issued all-reduce (capture failed: {type(e).__name__})"
                torch.cuda.synchronize()
                self.overlap_comm = False            # a host-issued collective cannot sit inside backward()
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            gloss, gg = self._fwd_bwd(simg, slab)
            if self.world_size == 1:
                self._opt(gg)
        g2 = None
        if self.world_size > 1:
            if not hasattr(self, "comm_mode"):
                self.comm_mode = "two graphs, host-issued all-reduce"
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                self._opt(gg)
        return (g1, g2, gloss, gg, self._outs, dict(self.loss_parts))

    def input_buffers(self, idx=0, like=None):
        """(image, label) device buffers read by captured graph `idx` (0 or 1)."""
        if self._static[idx] is None:
            src = like if like is not None else self._static[1 - idx]
            assert src is not None, "call the step once (or pass like=) before asking for input buffers"
            self._static[idx] = (torch.empty_like(src[0]), torch.empty_like(src[1]))
        return self._static[idx]

    def static_inputs(self):
        return self._static[0]

    @property
    def outputs(self):
        return self._outs


class UAMTStep:
    """Per-step body of train_uncertainty_aware_mean_teacher_2D.py:138-197 (BASELINE config 5) on the fused kernels.

    Batch = labelled half + unlabelled half.  Student: two training forwards with gradient (labelled, unlabelled);
    teacher (`ema_model`, never updated and never put in eval mode by the reference, SURVEY F8): one no-grad forward on the
    noisy unlabelled inputs and T/2 = 4 no-grad forwards on the twice-repeated noisy batch (T = 8 stochastic passes).
    Loss = 0.5*(Dice + CE) on the labelled half + w(t) * uncertainty-masked softmax-MSE consistency (K13 kernels).
    Two-head models (unet_cct) use main_seg on both sides (SURVEY F7)."""

    def __init__(self, model, ema_model, base_lr=0.01, max_iterations=30000, consistency=0.1, consistency_rampup=200.0,
                 momentum=0.9, weight_decay=1e-4, T=8, process_group=None, world_size=1, graph=False):
        """world_size > 1: batch-sharded data parallel -- every rank runs the step on its shard, the flat gradient bucket is
        all-reduced (sum) over NCCL and the fused SGD applies the 1/world mean, as `TrainStep` does.  The student replicas are
        broadcast from rank 0 at construction; the teacher is never updated by the reference (SURVEY F8) and is broadcast once.

        graph=True: after two eager warm-up steps the whole body (two student forwards, 1 + T/2 teacher forwards, losses, two
        backwards, SGD) is captured in ONE CUDA graph (world_size > 1: forward+backward | host-issued all-reduce | SGD, as
        `TrainStep`) -- the eager step issues ~900 launches from Python and is host-bound.  The ramps of the script (consistency
        weight :183, uncertainty threshold :186, poly LR :194) stay host arithmetic: they are written to a 2-float device buffer
        before every replay and read by the kernels through their *_ptr arguments.  Needs a fixed batch shape and noises=None."""
        from .utils import ramps
        self.world_size, self.pg = int(world_size), process_group
        self.ramps = ramps
        self.model, self.ema_model = model, ema_model
        self.ex, self.ex_t = model.executor, ema_model.executor
        self.base_lr, self.max_iterations = float(base_lr), int(max_iterations)
        self.consistency, self.consistency_rampup = float(consistency), float(consistency_rampup)
        self.momentum, self.weight_decay, self.T = float(momentum), float(weight_decay), int(T)
        self.iter_num = 0
        dev = next(model.parameters()).device
        self.dev = dev
        params = self.ex.params
        n = sum(p.numel() for p in params)
        self.flat = torch.empty(n, dtype=torch.float32, device=dev)
        off = 0
        for p in params:
            self.flat[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()
        first_aux = next(model.aux_decoder1.parameters()) if len(self.ex.dec) == 2 else None
        self.n_trained = n if first_aux is None else sum(p.numel() for p in params[: [id(q) for q in params].index(id(first_aux))])
        if self.world_size > 1:
            ddp.broadcast_flat(self.flat, 0, self.pg)
            for q in list(ema_model.parameters()) + list(ema_model.buffers()):
                ddp.broadcast_flat(q.data, 0, self.pg)
        self.mom = torch.zeros_like(self.flat)
        self.lr_dev = torch.full((1,), self.base_lr, dtype=torch.float32, device=dev)
        from .networks._engine import initial_rng_counter
        self.seed_dev = torch.full((1,), initial_rng_counter() ^ 0x5A5A5A5A, dtype=torch.int64, device=dev)
        self.ramp_dev = torch.zeros(2, dtype=torch.float32, device=dev)            # {uncertainty threshold, consistency weight}
        self.graph_enabled = bool(graph)
        self._warm, self._graph, self._static = 0, None, None
        self.launches_per_step = 0

    def _noisy(self, x, reps, salt, given):
        if given is not None:
            return (x.repeat(reps, 1, 1, 1) + given).contiguous()
        out = torch.empty((x.shape[0] * reps,) + tuple(x.shape[1:]), dtype=torch.float32, device=self.dev)
        call("wsl_add_clamped_noise", x, x.numel(), reps, 0.1, 0.2, 0xA5A5 + salt, self.seed_dev, out)
        return out

    def _ramps(self):
        """host arithmetic of :183 and :186 for the current iteration -> (threshold, weight), also written to ramp_dev"""
        import math
        cw = self.consistency * self.ramps.sigmoid_rampup(self.iter_num // 300, self.consistency_rampup)
        thr = (0.75 + 0.25 * self.ramps.sigmoid_rampup(self.iter_num, self.max_iterations)) * math.log(2)
        self.ramp_dev.copy_(torch.tensor([thr, cw], dtype=torch.float32))
        return thr, cw

    def _opt(self, g):
        call("wsl_sgd_step", self.flat, g, self.mom, self.n_trained, self.lr_dev, self.base_lr, self.momentum, self.weight_decay,
             1.0 / self.world_size)

    def __call__(self, image_l, label_l, image_u, noises=None):
        """image_l/image_u: fp32 [B,1,H,W]; label_l: uint8 [B,H,W] dense.  noises (tests): list of 1 + T/2 tensors holding
        the already-clamped noise of :147-149 and :167-169.  Returns the loss (0-dim device tensor)."""
        self.model.train()
        self.ema_model.train()
        thr, cw = self._ramps()
        if not self.graph_enabled:
            loss, g = self._body(image_l, label_l, image_u, noises)
            if self.world_size > 1:
                ddp.allreduce_flat(g[: self.n_trained], self.pg)
            self._opt(g)
        else:
            assert noises is None, "graph mode draws the teacher noise on the device"
            if self._static is None:
                self._static = (torch.empty_like(image_l), torch.empty_like(label_l), torch.empty_like(image_u))
            sl, sb, su = self._static
            assert sl.shape == image_l.shape and su.shape == image_u.shape, "graph mode needs a fixed batch shape"
            sl.copy_(image_l, non_blocking=True)
            sb.copy_(label_l, non_blocking=True)
            su.copy_(image_u, non_blocking=True)
            if self._warm < 2:                      # eager warm-up allocates every buffer / tensor map / workspace
                c0 = _lib.COUNTERS["launch_calls"]
                loss, g = self._body(sl, sb, su, None)
                if self.world_size > 1:
                    ddp.allreduce_flat(g[: self.n_trained], self.pg)
                self._opt(g)
                self.launches_per_step = _lib.COUNTERS["launch_calls"] - c0
                self._warm += 1
            else:
                if self._graph is None:
                    torch.cuda.synchronize()
                    g1, g2 = torch.cuda.CUDAGraph(), None
                    with torch.cuda.graph(g1):
                        gloss, gg = self._body(sl, sb, su, None)
                        if self.world_size == 1:
                            self._opt(gg)
                    if self.world_size > 1:
                        g2 = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(g2):
                            self._opt(gg)
                    self._graph = (g1, g2, gloss, gg, dict(self.parts))
                    self.comm_mode = "two graphs, host-issued all-reduce"
                g1, g2, gloss, gg, self.parts = self._graph
                g1.replay()
                if g2 is not None:
                    ddp.allreduce_flat(gg[: self.n_trained], self.pg)
                    g2.replay()
                loss = gloss.clone()                # the captured loss lives in graph-pool memory
        self.parts = dict(self.parts, weight=cw, threshold=thr)
        lr_ = self.base_lr * (1.0 - self.iter_num / self.max_iterations) ** 0.9
        self.lr_dev.fill_(lr_)
        self.iter_num += 1
        return loss

    def _body(self, image_l, label_l, image_u, noises):
        """forward passes, losses and both backward passes; returns (loss, flat gradient bucket)"""
        ex, ex_t, dev = self.ex, self.ex_t, self.dev
        B, _, H, W = image_u.shape
        C, T = 4, self.T
        self.seed_dev.add_(1)
        masks, ck = getattr(self.model, "dropout_masks", None), getattr(self.model, "channel_keep", None)
        tmasks, tck = getattr(self.ema_model, "dropout_masks", None), getattr(self.ema_model, "channel_keep", None)
        outs_l, slot_l = ex.forward(image_l.contiguous(), True, True, masks, ck)
        outs_u, slot_u = ex.forward(image_u.contiguous(), True, True, masks, ck)
        out_l, out_u = outs_l[0], outs_u[0]
        ema_out = ex_t.forward(self._noisy(image_u, 1, 0, None if noises is None else noises[0]), True, False, tmasks, tck)[0][0]
        mc = ex.buf("uamt", "mc", (T * B, C, H, W), torch.float32)
        for i in range(T // 2):
            tm2 = None if tmasks is None else {k: v.repeat(2, 1, 1, 1) for k, v in tmasks.items()}
            tck2 = None if tck is None else [c.repeat(2, 1) for c in tck]
            lg = ex_t.forward(self._noisy(image_u, 2, 1 + i, None if noises is None else noises[1 + i]), True, False, tm2, tck2)[0][0]
            mc[2 * B * i: 2 * B * (i + 1)].copy_(lg)
        Bf = lambda name, shape, dt=torch.float32: ex.buf("uamt", name, shape, dt)
        # ---- supervised half: 0.5 * (Dice + CE), CE without ignore_index (:127,:178-180) ----
        probs, st = Bf("probs_l", (B, C, H, W)), Bf("stats_l", (2,))
        call("wsl_softmax_pce_fwd", out_l, label_l, probs, B, C, H, W, 255, st, workspace("pce", dev))
        sums = Bf("dice", (13,))
        call("wsl_pdice_fwd", probs, label_l, None, 1.0, B, C, H, W, sums, workspace("pdice", dev))
        gp = Bf("gprobs_l", (B, C, H, W))
        call("wsl_pdice_bwd", probs, label_l, None, 1.0, sums, B, C, H, W, 0.5, 0, gp)
        dl_l = Bf("dl_l", (B, C, H, W))
        call("wsl_head_bwd", probs, label_l, st, None, 0.5, gp, 1.0, B, C, H, W, 255, dl_l, None, self.ex.dt)
        # ---- consistency half (:181-189) ----
        # threshold (:186) and weight (:183) come from ramp_dev (written by _ramps() before the body / the graph replay)
        mask, cst = Bf("mask", (B, H, W), torch.uint8), Bf("cons", (3,))
        call("wsl_uamt_consistency_fwd", out_u, ema_out, mc, T, B, C, H, W, self.ramp_dev[0:1], 0.0, mask, cst, workspace("uamt", dev))
        dl_u = Bf("dl_u", (B, C, H, W))
        call("wsl_uamt_consistency_bwd", out_u, ema_out, mask, cst, self.ramp_dev[1:2], 0.0, B, C, H, W, dl_u)
        loss = 0.5 * (sums[0] + st[0]) + self.ramp_dev[1] * cst[2]
        self.parts = {"supervised": 0.5 * (sums[0] + st[0]), "consistency": cst[2], "mask": mask}
        # ---- two backward passes through the shared student weights, gradients accumulated in the flat bucket ----
        nd = len(ex.dec)
        ex.backward(slot_u, [dl_u] + [None] * (nd - 1), zero_grads=True)
        g = ex.backward(slot_l, [dl_l] + [None] * (nd - 1), zero_grads=False)
        return loss, g


class USTMStep(UAMTStep):
    """Per-step body of train_weakly_supervised_ustm_2D.py:113-170: pCE on scribbles + uncertainty-aware self-ensembling with a
    random rot90 transform (Python host RNG, :123) and the EMA teacher update the script really performs (:163).

    graph=True: the rot90 count is a kernel ARGUMENT, so one CUDA graph is captured per count (at most four, each on the first
    step that draws it after two eager warm-up steps); threshold, consistency weight and the EMA factor reach the captured
    kernels through `ramp_dev`."""

    def __init__(self, model, ema_model, base_lr=0.01, max_iterations=60000, ema_decay=0.99, **kw):
        super().__init__(model, ema_model, base_lr=base_lr, max_iterations=max_iterations, **kw)
        self.ema_decay = float(ema_decay)
        tparams = self.ex_t.params
        n = sum(p.numel() for p in tparams)
        self.tflat = torch.empty(n, dtype=torch.float32, device=self.dev)
        off = 0
        for p in tparams:
            self.tflat[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.tflat[off:off + p.numel()].view_as(p)
            off += p.numel()
        self.ramp_dev = torch.zeros(3, dtype=torch.float32, device=self.dev)     # {threshold, weight, 1 - EMA alpha}
        self._graphs = {}

    def _ramps(self):
        import math
        cw = 1.0 * self.ramps.sigmoid_rampup(self.iter_num // 1000, 60)                                      # :145
        thr = (0.75 + 0.25 * self.ramps.sigmoid_rampup(self.iter_num, self.max_iterations)) * math.log(2)     # :148
        alpha = min(1 - 1 / (self.iter_num + 1), self.ema_decay)         # :63, global_step = iter_num before the increment
        self.ramp_dev.copy_(torch.tensor([thr, cw, 1.0 - alpha], dtype=torch.float32))
        return thr, cw, alpha

    def _finish(self, g, alpha):
        """SGD on the student, then the EMA teacher update (:163).  alpha=None (captured): the factor is read from ramp_dev"""
        self._opt(g)
        n = min(self.tflat.numel(), self.flat.numel())
        if alpha is None:
            self.tflat[:n].lerp_(self.flat[:n], self.ramp_dev[2])        # t + (1 - alpha) * (s - t)
        else:
            call("wsl_ema_update", self.tflat, self.flat, n, float(alpha))

    def __call__(self, image, label, noises=None, rot_times=None):
        self.model.train()
        self.ema_model.train()
        assert image.shape[2] == image.shape[3], "rot90 consistency needs square inputs"
        k = random.randrange(0, 4) if rot_times is None else int(rot_times)
        self.rot_times = k
        thr, cw, alpha = self._ramps()
        if not self.graph_enabled:
            loss, g = self._body(image, label, noises, k)
            if self.world_size > 1:
                ddp.allreduce_flat(g[: self.n_trained], self.pg)
            self._finish(g, alpha)
        else:
            assert noises is None, "graph mode draws the teacher noise on the device"
            if self._static is None:
                self._static = (torch.empty_like(image), torch.empty_like(label))
            si, sl = self._static
            assert si.shape == image.shape, "graph mode needs a fixed batch shape"
            si.copy_(image, non_blocking=True)
            sl.copy_(label, non_blocking=True)
            if self._warm < 2:
                c0 = _lib.COUNTERS["launch_calls"]
                loss, g = self._body(si, sl, None, k)
                if self.world_size > 1:
                    ddp.allreduce_flat(g[: self.n_trained], self.pg)
                self._finish(g, alpha)
                self.launches_per_step = _lib.COUNTERS["launch_calls"] - c0
                self._warm += 1
            else:
                if k not in self._graphs:
                    torch.cuda.synchronize()
                    g1, g2 = torch.cuda.CUDAGraph(), None
                    with torch.cuda.graph(g1):
                        gloss, gg = self._body(si, sl, None, k)
                        if self.world_size == 1:
                            self._finish(gg, None)
                    if self.world_size > 1:
                        g2 = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(g2):
                            self._finish(gg, None)
                    self._graphs[k] = (g1, g2, gloss, gg, dict(self.parts))
                    self.comm_mode = "two graphs per rot90 count, host-issued all-reduce"
                g1, g2, gloss, gg, self.parts = self._graphs[k]
                g1.replay()
                if g2 is not None:
                    ddp.allreduce_flat(gg[: self.n_trained], self.pg)
                    g2.replay()
                loss = gloss.clone()
        self.parts = dict(self.parts, weight=cw, threshold=thr)
        lr_ = self.base_lr * (1.0 - self.iter_num / self.max_iterations) ** 0.9
        self.lr_dev.fill_(lr_)
        self.iter_num += 1
        return loss

    def _body(self, image, label, noises, k):
        ex, ex_t, dev = self.ex, self.ex_t, self.dev
        B, _, H, W = image.shape
        C, T = 4, self.T
        self.seed_dev.add_(1)
        masks, ck = getattr(self.model, "dropout_masks", None), getattr(self.model, "channel_keep", None)
        tmasks, tck = getattr(self.ema_model, "dropout_masks", None), getattr(self.ema_model, "channel_keep", None)
        outs, slot = ex.forward(image.contiguous(), True, True, masks, ck)
        out = outs[0]
        Bf = lambda name, shape, dt=torch.float32: ex.buf("ustm", name, shape, dt)
        rimg = Bf("rimg", (B, 1, H, W))
        call("wsl_rot90", image.contiguous(), B, H, k, 0, rimg)
        ema_out = ex_t.forward(self._noisy(rimg, 1, 0, None if noises is None else noises[0]), True, False, tmasks, tck)[0][0]
        mc = Bf("mc", (T * B, C, H, W))
        for i in range(T // 2):
            tm2 = None if tmasks is None else {kk: v.repeat(2, 1, 1, 1) for kk, v in tmasks.items()}
            tck2 = None if tck is None else [c.repeat(2, 1) for c in tck]
            lg = ex_t.forward(self._noisy(rimg, 2, 1 + i, None if noises is None else noises[1 + i]), True, False, tm2, tck2)[0][0]
            mc[2 * B * i: 2 * B * (i + 1)].copy_(lg)
        # pCE (ignore_index 4)
        probs, st = Bf("probs", (B, C, H, W)), Bf("stats", (2,))
        call("wsl_softmax_pce_fwd", out, label, probs, B, C, H, W, 4, st, workspace("pce", dev))
        d = Bf("dl", (B, C, H, W))
        call("wsl_head_bwd", probs, label, st, None, 1.0, None, 0.0, B, C, H, W, 4, d, None, self.ex.dt)
        # consistency on the rotated student logits; threshold (:148) / weight (:145) from ramp_dev
        rout = Bf("rout", (B, C, H, W))
        call("wsl_rot90", out, B * C, H, k, 0, rout)
        mask, cst = Bf("mask", (B, H, W), torch.uint8), Bf("cons", (3,))
        call("wsl_uamt_consistency_fwd", rout, ema_out, mc, T, B, C, H, W, self.ramp_dev[0:1], 0.0, mask, cst, workspace("uamt", dev))
        dr = Bf("dr", (B, C, H, W))
        call("wsl_uamt_consistency_bwd", rout, ema_out, mask, cst, self.ramp_dev[1:2], 0.0, B, C, H, W, dr)
        call("wsl_rot90", dr, B * C, H, (4 - k) % 4, 1, d)              # rotate the gradient back and add it to the pCE part
        loss = st[0] + self.ramp_dev[1] * cst[2]
        self.parts = {"ce": st[0], "consistency": cst[2], "mask": mask}
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
        self._wstatic = None

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
        loss (0-dim device tensor): NaN after thr_iter when no unlabelled pixel clears thr_conf, as the reference."""
        assert weight.is_cuda and weight.dtype == torch.float32 and tuple(weight.shape) == (image.shape[0],) + tuple(image.shape[2:]) + (4,)
        w_u = 0.5 if self.iter_num >= self.thr_iter else 0.0
        if w_u != self._w_u:
            self.ctrl[1].fill_(w_u)
            self._w_u = w_u
        if self.graph_enabled:
            if self._wstatic is None:
                self._wstatic = torch.empty_like(weight)
            assert self._wstatic.shape == weight.shape, "graph mode needs a fixed batch shape"
            if self._wstatic.data_ptr() != weight.data_ptr():
                self._wstatic.copy_(weight, non_blocking=True)
            self._weight = self._wstatic
        else:
            self._weight = weight.contiguous()
        return super().__call__(image, scribble)

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
