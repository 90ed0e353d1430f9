"""Planned executor for the 2D U-Net family on the wsl4mis_b200 kernels.

The reference builds its network out of per-layer nn.Modules and lets autograd walk them
(networks/unet.py:13-135,286-346).  Here the nn.Modules are only *parameter containers* (same names,
shapes and init order, so state_dicts interchange); the arithmetic is a fixed launch sequence over
preallocated channels-last bf16 buffers:

  forward   conv (wgmma implicit GEMM, or CUDA-core direct for Cin=1 / tiny maps) -> BN statistics ->
            BN-affine + LeakyReLU + dropout (+ fused 2x2 max-pool)      [x2 per ConvBlock]
            decoder: conv1x1 -> bilinear x2 -> two-source conv (concat never materialised)
  backward  BN backward (fused with LeakyReLU/dropout/max-pool routing and the skip/aux/pool gradient sum)
            -> weight gradient -> data gradient, in reverse order, gradients written into ONE flat fp32 buffer
            (the DDP bucket).

All launches go to torch's current stream, never allocate or synchronise, and are CUDA-graph capturable.
"""
from __future__ import annotations

import contextlib
import ctypes
import os
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from .. import _lib
from .._lib import LIB, call, workspace

BF16 = torch.bfloat16
LRELU_SLOPE = 0.01

# execution modes: storage type of activations / activation gradients and the convolution kernels they run on
#   bf16    (dtype code 0) wgmma on bf16 operands -- the throughput mode (BASELINE config 2 names bf16)
#   fp16    (dtype code 2) the same kernels on fp16 operands (11-bit mantissa, identical MMA rate); gradients travel
#           multiplied by a power-of-two loss scale so that they stay inside fp16's range
#   fp16x3  (dtype code 1) fp32 storage; every convolution on the tensor cores with fp16 hi/lo split operands
#           (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, fp32 accumulation): the tensor-core mode that meets the fp32 reference
#   fp32    (dtype code 1) fp32 storage, CUDA-core direct convolutions: the arithmetic cross-check of everything else
PRECISIONS = {"bf16": 0, "fp16": 2, "fp16x3": 1, "fp32": 1}


def _ceil16(c):
    return (c + 15) // 16 * 16


def initial_rng_counter():
    """Start value of the device-side dropout / noise counter: a hash of torch's seed (the scripts call
    torch.manual_seed(args.seed), train_weakly_supervised_pCE_2D.py:187-190) and of the data-parallel rank, so that different
    --seed runs draw different masks and the ranks of one job draw different masks on their shards (ADVICE r1)."""
    rank = 0
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            rank = dist.get_rank()
        else:
            rank = int(os.environ.get("RANK", "0"))
    except Exception:
        rank = 0
    z = (torch.initial_seed() * 0x9E3779B97F4A7C15 + (rank + 1) * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF
    z ^= z >> 31
    return int(z & 0x3FFFFFFFFFFF)           # 46 bits: room for ~10^13 increments inside int64


class ConvLayer:
    """One nn.Conv2d (+ optional following BatchNorm2d/LeakyReLU/Dropout) and its packed operands."""

    def __init__(self, name, conv: nn.Conv2d, bn: Optional[nn.BatchNorm2d], drop_p: float, src_channels: Sequence[int]):
        self.name, self.conv, self.bn, self.drop_p = name, conv, bn, float(drop_p)
        self.ks = conv.kernel_size[0]
        self.dil = conv.dilation[0]          # PNet2D's blocks: 1, 2, 4, 8, 16 (networks/pnet.py:25-28); 1 everywhere in the U-Nets
        self.srcC = list(src_channels)
        self.Cin, self.Cout = conv.in_channels, conv.out_channels
        assert sum(self.srcC) == self.Cin
        self.CinP, self.CoutP = _ceil16(self.Cin), _ceil16(self.Cout)
        self.T = self.ks * self.ks
        self._packs = None

    def packs(self, dev):
        if self._packs is None or self._packs["wf"].device != dev:
            T, CinP, CoutP = self.T, self.CinP, self.CoutP
            pk = {
                "wf": torch.zeros(T * CinP * CoutP, dtype=torch.float32, device=dev),
                "bf": torch.zeros(T * CinP * CoutP, dtype=BF16, device=dev),
                "wd": [], "bd": [],
                "bias": torch.zeros(CoutP, dtype=torch.float32, device=dev),
            }
            for c in self.srcC:
                sp = _ceil16(c)
                pk["wd"].append(torch.zeros(T * CoutP * sp, dtype=torch.float32, device=dev))
                pk["bd"].append(torch.zeros(T * CoutP * sp, dtype=BF16, device=dev))
            if self.bn is not None:
                C = self.Cout
                pk["ss"] = torch.zeros(2 * C, dtype=torch.float32, device=dev)
            self._packs = pk
        return self._packs

    def pack(self, dev, dtype16=0):
        pk = self.packs(dev)
        w = self.conv.weight
        beg = 0
        for i, c in enumerate(self.srcC):
            call("wsl_pack_conv_weights", w, self.Cout, self.Cin, self.ks, self.CoutP, self.CinP, beg, c,
                 pk["wf"] if i == 0 else None, pk["wd"][i], pk["bf"] if i == 0 else None, pk["bd"][i], dtype16)
            beg += c
        if self.Cout == self.CoutP:
            pk["bias"] = self.conv.bias.detach()
        else:
            pk["bias"][: self.Cout].copy_(self.conv.bias.detach())


class UNetExecutor:
    """Forward/backward launch sequences for Encoder + k Decoders (k=1: UNet, k=2: UNet_CCT)."""

    MAX_SLOTS = 4

    def __init__(self, model: nn.Module, encoder: nn.Module, decoders: List[nn.Module], aux_dropout: Sequence[bool],
                 precision: str = "bf16", runs=None):
        """decoders: the decoder modules that own parameters; aux_dropout[i]: decoder i sees channel-dropped features.
        runs (optional): the decoder passes of one forward as (decoder index, feature transform) with transform in
        {None, "chan_drop", "feat_noise"} -- UNet_CCT_3H runs aux_decoder1 twice (unet.py:367-370) and never runs aux_decoder2."""
        assert precision in PRECISIONS
        if runs is None:
            runs = [(i, "chan_drop" if a else None) for i, a in enumerate(aux_dropout)]
        self.runs = list(runs)
        self.aux = [t for _, t in self.runs]           # feature transform of every decoder pass
        self.layers: List[ConvLayer] = []
        ft = encoder.ft_chns
        self.ft = ft
        self.in_chns = encoder.in_chns

        def block(name, seq, srcC):
            l1 = ConvLayer(f"{name}.0", seq[0], seq[1], seq[3].p, srcC)
            l2 = ConvLayer(f"{name}.4", seq[4], seq[5], 0.0, [seq[4].in_channels])
            self.layers += [l1, l2]
            return (l1, l2)

        self.enc_blocks = [block("encoder.in_conv.conv_conv", encoder.in_conv.conv_conv, [self.in_chns])]
        for i in range(1, 5):
            cb = getattr(encoder, f"down{i}").maxpool_conv[1]
            self.enc_blocks.append(block(f"encoder.down{i}", cb.conv_conv, [ft[i - 1]]))
        self.dec = []
        self.ds_heads = []
        built = {}
        for didx, _ in self.runs:
            if didx in built:                  # a second pass through the same decoder shares its layers (and their gradients)
                self.dec.append(built[didx][0])
                self.ds_heads.append(built[didx][1])
                continue
            d = decoders[didx]
            ups = []
            for j in range(1, 5):
                ub = getattr(d, f"up{j}")
                c1 = ConvLayer(f"up{j}.conv1x1", ub.conv1x1, None, 0.0, [ub.conv1x1.in_channels])
                self.layers.append(c1)
                c2 = ub.conv1x1.out_channels
                ups.append((c1, block(f"up{j}.conv", ub.conv.conv_conv, [c2, c2])))
            oc = ConvLayer("out_conv", d.out_conv, None, 0.0, [d.out_conv.in_channels])
            self.layers.append(oc)
            self.dec.append((ups, oc))
            # deep-supervision heads of Decoder_DS (unet.py:159-168): a 3x3 class head on the output of up1 / up2 / up3
            # (index j = 0, 1, 2 <-> out_conv_dp3 / dp2 / dp1); out_conv_dp4 owns parameters but never runs
            heads = {}
            if hasattr(d, "out_conv_dp3"):
                for j, lvl in enumerate((3, 2, 1)):
                    hc = getattr(d, f"out_conv_dp{lvl}")
                    heads[j] = ConvLayer(f"out_conv_dp{lvl}", hc, None, 0.0, [hc.in_channels])
                    self.layers.append(heads[j])
            self.ds_heads.append(heads)
            built[didx] = (self.dec[-1], heads)
        self.n_class = decoders[0].out_conv.out_channels
        self._init_runtime(model, precision)
        # what the training steps (engine.py) read of an executor; PNetExecutor defines the same three
        self.n_outputs = len(self.dec) + 3 * sum(1 for heads in self.ds_heads if heads)      # tensors forward() returns
        # parameters a step that reads main_seg only leaves untrained (SURVEY F7): the aux decoder of unet_cct
        self.aux_param_ids = {id(q) for q in model.aux_decoder1.parameters()} if len(self.dec) == 2 else set()
        # the encoder's parameters come first in parameters(): a data-parallel step all-reduces the decoder slice of the bucket
        # from inside backward() (on_decoders_done) and this prefix after it; None would turn that overlap off
        self.comm_split = sum(q.numel() for q in encoder.parameters())

    def _init_runtime(self, model, precision):
        """state shared by every planned network (the U-Net family here, PNet2D in _pnet_engine.py): precision, parameter
        bookkeeping, buffers, side streams"""
        self.model = model
        self.precision = precision
        self.dt = PRECISIONS[precision]
        self.act_dtype = {0: BF16, 1: torch.float32, 2: torch.float16}[self.dt]
        self.split_tc = precision == "fp16x3"
        # power-of-two factor carried by every activation gradient (set per backward from the batch shape; 1 = off)
        self.scaled_grads = precision == "fp16"        # fp16x3 scales every staged operand by its own power of two instead
        self.params = [p for p in model.parameters()]
        used = set()
        for L in self.layers:
            used.update(id(t) for t in (L.conv.weight, L.conv.bias))
            if L.bn is not None:
                used.update(id(t) for t in (L.bn.weight, L.bn.bias))
        self.used_param_ids = used        # parameters no launch touches (Decoder_DS.out_conv_dp4) get no gradient, like autograd
        self._gflat = None
        self._gviews = None
        self._bufs: Dict = {}
        self._live: List[int] = []
        self._seed_host = 0x5EED
        self.use_tc = True               # False: every convolution on the CUDA-core direct kernels (a reference for the wgmma ones)
        self.on_decoders_done = None     # optional callback(gflat) between the decoder and encoder halves of backward()
        # Synchronised BatchNorm over data-parallel ranks (SURVEY 8(e)(2)): (world_size, process_group) or None.  Statistics of the
        # GLOBAL batch: forward all-reduces {sum, sum of squares} per layer, backward {sum dz, sum dz*xhat}; 2C floats each.
        self.sync_bn = None
        self.multi_stream = True         # False: every launch on the current stream (per-kernel timing, single-chain networks)
        self._sides = {}                 # named side streams
        self._side_stack = []            # names of the side streams we are currently issuing on (innermost last)
        self._side_dirty = set()
        self._stat_bufs = {}
        self._stat_rows = ctypes.c_int(0)
        self._accumulate = False
        self._bn_per_sample = False      # forward(..., bn_per_sample=True) is running
        self.stats = {"launches": 0}

    # ---------------------------------------------------------------- buffers
    def buf(self, slot, name, shape, dtype=None):
        dtype = self.act_dtype if dtype is None else dtype
        key = (slot, name, tuple(shape), dtype)
        t = self._bufs.get(key)
        if t is None:
            t = torch.empty(shape, dtype=dtype, device=self.dev)
            self._bufs[key] = t
        return t

    def grads(self):
        """Flat fp32 gradient bucket + per-parameter views (in model.parameters() order)."""
        if self._gflat is None or self._gflat.device != self.dev:
            n = sum(p.numel() for p in self.params)
            self._gflat = torch.zeros(n, dtype=torch.float32, device=self.dev)
            self._gviews, off = {}, 0
            for p in self.params:
                self._gviews[id(p)] = self._gflat[off:off + p.numel()].view_as(p)
                off += p.numel()
        return self._gflat, self._gviews

    def gview(self, p):
        return self.grads()[1][id(p)]

    def _ws(self, tag):
        return workspace(tag + ("" if not self._side_stack else "." + self._side_stack[-1]), self.dev)

    def _wgrad_partials(self):
        """per-stream workspace for the split-K partial tiles of the deterministic weight gradient: the kernels launch about two CTAs
        per SM with at most 3 x 64 x 128 floats (96 KB) each, about 25 MB of the 32 MB on a 132-SM H100"""
        key = ("wgp", self._side_stack[-1] if self._side_stack else "main")
        t = self._bufs.get(key)
        if t is None or t.device != self.dev:
            t = self._bufs[key] = torch.empty(8 * 1024 * 1024, dtype=torch.float32, device=self.dev)
        return t

    def _stat_scratch(self):
        """per-stream scratch for the conv-epilogue BatchNorm partial rows"""
        key = self._side_stack[-1] if self._side_stack else "main"
        if key not in self._stat_bufs or self._stat_bufs[key].device != self.dev:
            self._stat_bufs[key] = torch.zeros(592 * 2 * 256 + 64, dtype=torch.float32, device=self.dev)   # + ticket word
        return self._stat_bufs[key]

    # ---------------------------------------------------------------- two-stream scheduling
    # Independent work is issued on a side stream so that HBM-bound elementwise kernels of one chain overlap the
    # tensor-core kernels of the other: (a) the aux decoder's forward runs beside the main decoder's, (b) every
    # weight-gradient kernel runs beside the data-gradient -> BatchNorm-backward chain.  Inside a captured CUDA
    # graph the fork/join events become graph edges.
    def _side_stream(self, name="side"):
        st = self._sides.get(name)
        if st is None or st.device != self.dev:
            st = self._sides[name] = torch.cuda.Stream(device=self.dev)
        return st

    @contextlib.contextmanager
    def on_side(self, name="side"):
        """Issue the enclosed launches on the named side stream, ordered after everything issued so far on the CURRENT stream
        (which may itself be a side stream: weight gradients of the aux-decoder chain fork from that chain)."""
        if not self.multi_stream:
            yield
            return
        side = self._side_stream(name)
        ev = torch.cuda.Event()
        ev.record()
        side.wait_event(ev)
        self._side_stack.append(name)
        try:
            with torch.cuda.stream(side):
                yield
        finally:
            self._side_stack.pop()
            self._side_dirty.add(name)

    def join_side(self, name=None):
        """Make the current stream wait for the named side stream (default: all of them)."""
        if not self.multi_stream:
            return
        for nm in ([name] if name is not None else sorted(self._side_dirty)):
            if nm in self._side_dirty:
                ev = torch.cuda.Event()
                ev.record(self._side_stream(nm))
                torch.cuda.current_stream().wait_event(ev)
                self._side_dirty.discard(nm)

    # ---------------------------------------------------------------- primitive launches
    def _tag(self, kind, L, N, H, W, cin, cout):
        """Label the next C-ABI call for bench.py's per-kernel table: algorithmic FLOPs and ideal bytes."""
        if _lib.PROFILE is not None:
            flops = 2.0 * cin * cout * L.T * H * W * N
            if kind == "wgrad":
                byts = 2.0 * (cin + cout) * H * W * N
            else:
                byts = 2.0 * (cin + cout) * H * W * N
            _lib.PROFILE.meta = (kind, L.name, flops, byts)

    def _tag_bytes(self, kind, L, byts):
        """Label a bandwidth-bound launch with its algorithmic bytes (bench.py prints GB/s for it)."""
        if _lib.PROFILE is not None:
            _lib.PROFILE.meta = (kind, L.name, 0.0, float(byts))

    def _untag(self):
        if _lib.PROFILE is not None:
            _lib.PROFILE.meta = None

    def _tc2_ok(self, layer_cin_list, H, W):
        """persistent / resident-weight / halo-view kernels: 8 x 16 pixel tiles"""
        return (self.dt != 1 and self.use_tc and all(c % 16 == 0 for c in layer_cin_list) and W % 8 == 0 and H % 16 == 0)

    def _tc_ok(self, layer_cin_list, H, W):
        return (self.dt != 1 and self.use_tc and all(c % 16 == 0 for c in layer_cin_list) and W % 16 == 0 and H % 8 == 0)

    def _split_ok(self, layer_cin_list, H, W):
        """fp16 hi/lo split convolutions (fp16x3 mode): the per-tap wgmma kernel's 16 x 8 pixel tiles"""
        return self.split_tc and self.use_tc and all(c % 16 == 0 for c in layer_cin_list) and W % 16 == 0 and H % 8 == 0

    def _staged(self, name, srcs, chans, P):
        """fp32 NHWC source(s) -> fp16 [P][2*C] (hi | lo) staging buffer of the split convolutions"""
        C = sum(chans)
        key = ("stage", name, P, C, self._side_stack[-1] if self._side_stack else "main")
        t = self._bufs.get(key)
        if t is None:
            t = self._bufs[key] = (torch.empty((P, 2 * C), dtype=torch.float16, device=self.dev),
                                   torch.zeros(3, dtype=torch.float32, device=self.dev))     # {2^k, 2^-k, scratch}
        call("wsl_split_f32", srcs[0], chans[0], srcs[1] if len(srcs) > 1 else None, chans[1] if len(chans) > 1 else 0, P, t[0], t[1])
        return t[0], t[1][1:]

    def conv_fwd(self, L: ConvLayer, srcs, out, out_mode, N, H, W, cout_store, src_f32=False, bn_out=None, srcC_override=None):
        """bn_out = (save, ss) buffers: when the convolution runs on conv_first or the persistent wgmma kernel the complete
        training-mode BatchNorm statistics of its output are produced by the kernel itself (partial rows in the epilogue,
        finalised by bn_finalize).  Returns True when that happened."""
        pk = L.packs(self.dev)
        srcC = list(srcC_override) if srcC_override is not None else L.srcC     # (a materialised concat enters as ONE source)
        rows = False
        s0 = srcs[0]
        s1 = srcs[1] if len(srcs) > 1 else None
        c0 = srcC[0]
        c1 = srcC[1] if len(srcC) > 1 else 0
        self._tag("fwd", L, N, H, W, L.Cin, L.Cout)
        f32 = 1 if (src_f32 or self.dt == 1) else self.dt  # dtype code of the sources
        if out_mode == 0 and self.dt != 0:
            out_mode = 2 if self.dt == 1 else 3            # fp32 / fp16 NHWC activations
        first = src_f32 and L.Cin == 1 and L.Cout == 16 and L.ks == 3 and out_mode in (0, 2, 3)
        if not first:
            self.join_side("pack")        # packed operands are produced on a side stream at the start of forward()
        if first:
            rows = bn_out is not None
            sb = self._stat_scratch() if rows else None
            call("wsl_conv_first", s0, L.conv.weight, L.conv.bias, out, self.dt, N, H, W, L.Cout, sb,
                 ctypes.addressof(self._stat_rows) if rows else None)
        elif not src_f32 and self._split_ok(srcC, H, W):
            st, inv = self._staged("x", srcs, srcC, N * H * W)
            call("wsl_conv_tc_split", st, L.Cin, inv, pk["f3"], pk["bias"], out, out_mode, N, H, W, L.CoutP, cout_store, L.ks, L.dil)
        elif not src_f32 and L.dil != 1:
            assert self._tc_ok(srcC, H, W), "dilated convolutions run on the per-tap wgmma kernel (W % 16 == 0, H % 8 == 0, 16-bit or fp16x3 mode)"
            call("wsl_conv_tc_dil", s0, c0, s1, c1, pk["bf"], pk["bias"], out, 0 if out_mode == 3 else out_mode, N, H, W, L.CoutP,
                 cout_store, L.ks, self.dt, L.dil)
        elif not src_f32 and self._tc2_ok(srcC, H, W):
            rows = bn_out is not None and out_mode in (0, 3)
            sb = self._stat_scratch() if rows else None
            call("wsl_conv_tc2", s0, c0, s1, c1, pk["bf"], pk["bias"], out, 0 if out_mode == 3 else out_mode, N, H, W, L.CoutP,
                 cout_store, L.ks, self.dt, sb, ctypes.addressof(self._stat_rows) if rows else None)
        elif not src_f32 and self._tc_ok(srcC, H, W):
            call("wsl_conv_tc", s0, c0, s1, c1, pk["bf"], pk["bias"], out, 0 if out_mode == 3 else out_mode, N, H, W, L.CoutP,
                 cout_store, L.ks, self.dt)
        else:
            call("wsl_conv_direct", s0, c0, s1, c1, f32, pk["wf"], pk["bias"], out, out_mode, N, H, W,
                 L.CinP, L.CoutP, cout_store, L.ks)
        self._untag()                              # the finalize launch is not a convolution: keep it out of the conv roofline rows
        if rows:
            self._finalize_stats(L, sb, self._stat_rows.value, N * H * W, bn_out[0], bn_out[1])
        return rows

    def conv_dgrad(self, L: ConvLayer, i, dy, out, N, H, W):
        pk = L.packs(self.dev)
        ci = L.srcC[i]
        sp = _ceil16(ci)
        self._tag("dgrad", L, N, H, W, ci, L.Cout)
        if self._split_ok([L.CoutP], H, W):
            st, inv = self._staged("dy", [dy], [L.CoutP], N * H * W)
            call("wsl_conv_tc_split", st, L.CoutP, inv, pk["d3"][i], None, out, 2, N, H, W, sp, ci, L.ks, L.dil)
        elif L.dil != 1:
            assert self._tc_ok([L.CoutP], H, W), "dilated data gradient: per-tap wgmma kernel only"
            call("wsl_conv_tc_dil", dy, L.CoutP, None, 0, pk["bd"][i], None, out, 0, N, H, W, sp, ci, L.ks, self.dt, L.dil)
        elif self._tc2_ok([L.CoutP], H, W):
            call("wsl_conv_tc2", dy, L.CoutP, None, 0, pk["bd"][i], None, out, 0, N, H, W, sp, ci, L.ks, self.dt, None, None)
        elif self._tc_ok([L.CoutP], H, W):
            call("wsl_conv_tc", dy, L.CoutP, None, 0, pk["bd"][i], None, out, 0, N, H, W, sp, ci, L.ks, self.dt)
        else:
            call("wsl_conv_direct", dy, L.CoutP, None, 0, self.dt, pk["wd"][i], None, out, {0: 0, 1: 2, 2: 3}[self.dt], N, H, W, L.CoutP, sp, ci, L.ks)
        self._untag()

    def conv_wgrad(self, L: ConvLayer, srcs, dy, N, H, W, src_f32=False, srcC_override=None):
        self.last_backward_param_ids.update((id(L.conv.weight), id(L.conv.bias)))
        srcC = list(srcC_override) if srcC_override is not None else L.srcC
        s0 = srcs[0]
        s1 = srcs[1] if len(srcs) > 1 else None
        c0 = srcC[0]
        c1 = srcC[1] if len(srcC) > 1 else 0
        self._tag("wgrad", L, N, H, W, L.Cin, L.Cout)
        fits = L.CoutP <= 64 or L.CoutP % 64 == 0        # the dY boxes of wsl_wgrad_tc and wsl_wgrad_tc_split: one per 64 filters
        tc = not src_f32 and self._tc_ok(srcC, H, W) and fits
        split = not src_f32 and self._split_ok(srcC, H, W) and fits
        if src_f32 and L.Cin == 1 and L.Cout == 16 and L.ks == 3 and L.bn is not None:
            call("wsl_wgrad_first", s0, dy, self.dt, self.gview(L.conv.weight), N, H, W, L.Cout)
        elif split:
            sx, ix = self._staged("x", srcs, srcC, N * H * W)
            sg, ig = self._staged("dy", [dy], [L.CoutP], N * H * W)
            call("wsl_wgrad_tc_split", sx, L.Cin, ix, sg, L.CoutP, ig, self.gview(L.conv.weight), N, H, W, L.Cout, L.ks, L.dil)
            tc = True
        elif L.dil != 1 and not src_f32:
            assert tc, "dilated weight gradient: per-tap wgmma kernel only"
            pw = self._wgrad_partials()
            call("wsl_wgrad_tc_dil", s0, c0, s1, c1, dy, L.CoutP, self.gview(L.conv.weight), N, H, W, L.Cout, L.ks, self.dt, L.dil, pw,
                 pw.numel())
        elif tc and L.ks == 3 and self._tc2_ok(srcC, H, W) and (L.CoutP <= 64 or L.CoutP % 128 == 0):
            pw = self._wgrad_partials()
            call("wsl_wgrad_tc3", s0, c0, s1, c1, dy, L.CoutP, self.gview(L.conv.weight), N, H, W, L.Cout, L.ks, self.dt, pw, pw.numel())
        elif tc:
            pw = self._wgrad_partials()
            call("wsl_wgrad_tc", s0, c0, s1, c1, dy, L.CoutP, self.gview(L.conv.weight), N, H, W, L.Cout, L.ks, self.dt, pw, pw.numel())
        else:
            call("wsl_wgrad_direct", s0, c0, s1, c1, 1 if (src_f32 or self.dt == 1) else self.dt, dy, self.dt, L.CoutP,
                 self.gview(L.conv.weight), self.gview(L.conv.bias) if L.bn is None else None, N, H, W, L.Cout, L.ks)
        self._untag()
        # Bias gradient.  A conv bias that feeds training-mode BatchNorm has an exactly-zero gradient (BN removes the
        # per-channel mean); the reference holds ~1e-8 rounding noise there.  We leave the zero-filled bucket as is.
        if tc and L.bn is None:
            call("wsl_channel_sum", dy, self.dt, N * H * W, L.CoutP, L.Cout, self.gview(L.conv.bias), self._ws("csum"))

    def bn_bufs(self, L, slot, tag):
        C = L.Cout
        return (self.buf(slot, tag + ".save", (2 * C,), torch.float32), self.buf(slot, tag + ".ss", (2 * C,), torch.float32))

    def bn_fwd(self, L: ConvLayer, y, act, N, H, W, training, slot, tag, mask=None, pooled=None, pool_idx=None, stats_done=False):
        bn = L.bn
        C = L.Cout
        pk = L.packs(self.dev)
        save = self.buf(slot, tag + ".save", (2 * C,), torch.float32)
        ss = self.buf(slot, tag + ".ss", (2 * C,), torch.float32)
        if training and self._bn_per_sample:
            # every image normalised by its own statistics (B batch-1 training forwards); {scale, shift} per image
            save = self.buf(slot, tag + ".save_ps", (N, 2 * C), torch.float32)
            ss = self.buf(slot, tag + ".ss_ps", (N, 2 * C), torch.float32)
            call("wsl_bn_stats_ps", y, self.dt, N, H * W, C, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                 bn.num_batches_tracked, float(bn.momentum), float(bn.eps), save, ss, self._ws("bn_ps"))
            p = L.drop_p
            self._tag_bytes("bn_act", L, N * H * W * C * (4 if self.dt == 1 else 2) * (2.25 if pooled is not None else 2.0))
            call("wsl_bn_act_fwd_ps", y, self.dt, ss, N, H, W, C, LRELU_SLOPE, p, mask, self._layer_seed(L),
                 self.seed_dev if mask is None and p > 0 else None, act, pooled, pool_idx)
            self._untag()
            return save, ss
        if training and stats_done:
            pass                       # save / ss come from the convolution epilogue's partial rows (bn_finalize)
        elif training and self.sync_bn is not None:
            raw = self.buf(slot, tag + ".raw", (2 * C,), torch.float32)
            call("wsl_bn_stats", y, self.dt, N * H * W, C, bn.weight, bn.bias, None, None, None, float(bn.momentum), float(bn.eps),
                 save, ss, self._ws("bn"), raw)
            from .. import ddp
            ddp.allreduce_flat(raw, self.sync_bn[1])
            call("wsl_bn_finalize", raw, 1, N * H * W * self.sync_bn[0], C, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                 bn.num_batches_tracked, float(bn.momentum), float(bn.eps), save, ss)
        elif training:
            call("wsl_bn_stats", y, self.dt, N * H * W, C, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                 bn.num_batches_tracked, float(bn.momentum), float(bn.eps), save, ss, self._ws("bn"), None)
        else:
            call("wsl_bn_eval_prepare", bn.weight, bn.bias, bn.running_mean, bn.running_var, float(bn.eps), C, ss)
        p = L.drop_p if training else 0.0
        seed = self._layer_seed(L)
        esz = 4 if self.dt == 1 else 2
        self._tag_bytes("bn_act", L, N * H * W * C * esz * (2.25 if pooled is not None else 2.0))
        call("wsl_bn_act_fwd", y, self.dt, ss, N, H, W, C, LRELU_SLOPE, p, mask, seed, self.seed_dev if mask is None and p > 0 else None,
             act, pooled, pool_idx)
        self._untag()
        return save, ss

    def bn_bwd(self, L: ConvLayer, y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, dy, N, H, W, slot, tag):
        bn = L.bn
        self.last_backward_param_ids.update((id(bn.weight), id(bn.bias)))
        C = L.Cout
        coef = self.buf(slot, tag + ".coef", (2 * C,), torch.float32)
        p = L.drop_p
        esz = 4 if self.dt == 1 else 2
        nsrc = (g0 is not None) + (g1 is not None) + 0.25 * (gpool is not None)
        self._tag_bytes("bn_bwd", L, N * H * W * C * esz * (2 * (1 + nsrc) + 1))      # reduce: y + sources; apply: again + dY
        args = (y, self.dt, ss, save, g0, g1, cs1, gpool, pool_idx, mask, self._layer_seed(L),
                self.seed_dev if mask is None and p > 0 else None, p, LRELU_SLOPE, N, H, W, C, self.gview(bn.weight),
                self.gview(bn.bias), coef, dy, self._ws("bn"), 1 if self._accumulate else 0)
        if self.sync_bn is not None:
            # global-batch BatchNorm backward: local reduction -> all-reduce {sum dz, sum dz*xhat} -> constants from the global sums
            from .. import ddp
            raw = self.buf(slot, tag + ".rawb", (2 * C,), torch.float32)
            call("wsl_bn_bwd_phase", *args, 1, raw)
            ddp.allreduce_flat(raw, self.sync_bn[1])
            call("wsl_bn_bwd_coef", raw, N * H * W * self.sync_bn[0], ss, save, C, coef)
            call("wsl_bn_bwd_phase", *args, 2, None)
        else:
            call("wsl_bn_bwd", *args)
        self._untag()

    def grad_scale_for(self, N, H, W):
        """Loss scale of the fp16 modes: a power of two near N*H*W/2, so that the largest logit gradient of a mean-type loss
        (1 / #labelled pixels, ~3 % of the pixels with scribbles; 1 / (N*H*W) for dense terms) lands around 2^0..2^4 and the
        smallest regulariser gradients stay far above fp16's subnormal range.  Activation gradients are linear in it; the flat
        parameter-gradient bucket is multiplied by 1/scale (exact) at the end of backward()."""
        if not self.scaled_grads:
            return 1.0
        import math
        return float(2 ** (round(math.log2(N * H * W)) - 1))

    def _finalize_stats(self, L, sb, nrows, P, save, ss):
        """partial rows of a convolution epilogue -> {mean, invstd, scale, shift} (+ running statistics); with sync_bn the rows are
        summed locally, all-reduced over the ranks and finalised against the global pixel count"""
        bn = L.bn
        if self.sync_bn is not None:
            world, pg = self.sync_bn
            C = L.Cout                        # BatchNorm layers have Cout == CoutP (multiples of 16): rows are [2][C]
            raw = sb[: nrows * 2 * C].view(nrows, 2 * C).double().sum(0).float().contiguous()
            from .. import ddp
            ddp.allreduce_flat(raw, pg)
            sb, nrows, P = raw, 1, P * world
        call("wsl_bn_finalize", sb, nrows, P, L.Cout, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked,
             float(bn.momentum), float(bn.eps), save, ss)

    def _layer_seed(self, L):
        return (self.layers.index(L) + 1) * 0x9E3779B1

    # ---------------------------------------------------------------- forward
    def pack_all(self):
        """fp32 master weights -> packed bf16/fp32 operands of every layer, ONE launch (table of pointers on device)."""
        ptrs = tuple(L.conv.weight.data_ptr() for L in self.layers)
        if getattr(self, "_pack_key", None) != (ptrs, str(self.dev)):
            rows, first = [], 0
            for L in self.layers:
                pk = L.packs(self.dev)
                beg = 0
                for i, c in enumerate(L.srcC):
                    rows.append([L.conv.weight.data_ptr(), pk["wf"].data_ptr() if i == 0 else 0, pk["wd"][i].data_ptr(),
                                 pk["bf"].data_ptr() if i == 0 else 0, pk["bd"][i].data_ptr(), L.Cout, L.Cin, L.T, L.CoutP, L.CinP,
                                 beg, c, first])
                    first += L.T * L.CoutP * L.CinP
                    beg += c
            self._pack_table = torch.tensor(rows, dtype=torch.int64).to(self.dev)
            self._pack_total = first
            self._pack_n = len(rows)
            self._pack_key = (ptrs, str(self.dev))
        call("wsl_pack_conv_weights_batched", self._pack_table, self._pack_n, self._pack_total, self.dt)
        if self.split_tc:
            for L in self.layers:
                pk = L.packs(self.dev)
                if "f3" not in pk:
                    pk["f3"] = torch.zeros(L.T * L.CoutP * 3 * L.CinP, dtype=torch.float16, device=self.dev)
                    pk["d3"] = [torch.zeros(L.T * _ceil16(c) * 3 * L.CoutP, dtype=torch.float16, device=self.dev) for c in L.srcC]
                beg = 0
                for i, c in enumerate(L.srcC):
                    call("wsl_pack_split_weights", L.conv.weight, L.Cout, L.Cin, L.ks, L.CoutP, L.CinP, beg, c,
                         pk["f3"] if i == 0 else None, pk["d3"][i])
                    beg += c
        for L in self.layers:                      # biases: share the parameter storage (or copy into the 16-padded buffer)
            pk = L.packs(self.dev)
            if L.Cout == L.CoutP:
                pk["bias"] = L.conv.bias.detach()
            else:
                pk["bias"][: L.Cout].copy_(L.conv.bias.detach())

    def forward(self, x: torch.Tensor, training: bool, need_grad: bool, masks: Optional[dict] = None,
                chan_keep: Optional[list] = None, defer_join: bool = False, bn_per_sample: bool = False):
        """x: fp32 [N, in_chns, H, W] CUDA.  Returns (list of fp32 NCHW logits, slot).

        bn_per_sample (training, no gradient): compute exactly what N batch-1 training forwards compute -- every BatchNorm
        normalises each image by that image's own statistics and the running statistics take the N updates in batch order
        (the ensemble refresh of train_s2l.py:221-228 runs the model on one slice at a time in train mode)."""
        if bn_per_sample:
            assert training and not need_grad, "bn_per_sample is a training-mode forward without gradient"
            self._bn_per_sample = True
            try:
                return self.forward(x, training, need_grad, masks, chan_keep, defer_join)
            finally:
                self._bn_per_sample = False
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4, "input must be a CUDA fp32 NCHW tensor"
        assert x.shape[1] == self.in_chns == 1, "executor is specialised to single-channel inputs (ACDC slices)"
        N, _, H, W = x.shape
        assert H % 16 == 0 and W % 16 == 0, "H, W must be multiples of 16 (4 pooling levels)"
        self.dev = x.device
        if not hasattr(self, "seed_dev") or self.seed_dev.device != self.dev:
            self.seed_dev = torch.full((1,), initial_rng_counter(), dtype=torch.int64, device=self.dev)
        x = x.contiguous()
        slot = self._acquire_slot() if need_grad else "ng"
        with self.on_side("pack"):      # operand packing runs beside the first layer (which reads the raw fp32 weights)
            self.pack_all()
        if training:
            self.seed_dev.add_(1)
        ft = self.ft
        rec = {"N": N, "H": H, "W": W, "x": x, "training": training, "enc": [], "dec": [], "masks": masks}

        def run_block(tag, blk, srcs, h, w, mask, pool, src_f32=False):
            l1, l2 = blk
            C = l1.Cout
            y1 = self.buf(slot, tag + ".y1", (N, h, w, C))
            a1 = self.buf(slot, tag + ".a1", (N, h, w, C))
            y2 = self.buf(slot, tag + ".y2", (N, h, w, C))
            a2 = self.buf(slot, tag + ".a2", (N, h, w, C))
            stats_in_conv = training and not self._bn_per_sample    # the conv epilogue's statistics are batch-wide
            r1 = self.conv_fwd(l1, srcs, y1, 0, N, h, w, C, src_f32, bn_out=self.bn_bufs(l1, slot, tag + ".bn1") if stats_in_conv else None)
            sv1, ss1 = self.bn_fwd(l1, y1, a1, N, h, w, training, slot, tag + ".bn1", mask, stats_done=r1)
            r2 = self.conv_fwd(l2, [a1], y2, 0, N, h, w, C, bn_out=self.bn_bufs(l2, slot, tag + ".bn2") if stats_in_conv else None)
            pooled = idx = None
            if pool:
                pooled = self.buf(slot, tag + ".pool", (N, h // 2, w // 2, C))
                idx = self.buf(slot, tag + ".pidx", (N, h // 2, w // 2, C), torch.uint8)
            sv2, ss2 = self.bn_fwd(l2, y2, a2, N, h, w, training, slot, tag + ".bn2", None, pooled, idx, stats_done=r2)
            return {"srcs": srcs, "y1": y1, "a1": a1, "y2": y2, "a2": a2, "sv1": sv1, "ss1": ss1, "sv2": sv2, "ss2": ss2,
                    "pool": pooled, "pidx": idx, "mask": mask, "h": h, "w": w, "src_f32": src_f32}

        # ---- encoder (unet.py:92-98) ----
        src = [x]
        h, w = H, W
        for i, blk in enumerate(self.enc_blocks):
            mask = None
            if masks is not None and training:
                mask = masks.get(i)
            r = run_block(f"enc{i}", blk, src, h, w, mask, pool=(i < 4), src_f32=(i == 0))
            rec["enc"].append(r)
            if i < 4:
                src = [r["pool"]]
                h, w = h // 2, w // 2
        feats = [r["a2"] for r in rec["enc"]]

        # ---- decoders (unet.py:123-135; aux branch sees channel-dropped features, :344) ----
        outs = [torch.empty((N, self.n_class, H, W), dtype=torch.float32, device=self.dev) for _ in self.dec]

        def run_decoder(di, ups, oc):
            drec = {"ups": [], "cs": None}
            fe = feats
            if self.aux[di] == "feat_noise":
                # FeatureNoise (unet.py:270-283, :369): one uniform(-0.3, 0.3) tensor of the feature's [C, H, W] shape, shared by the
                # batch: f * noise + f.  model.feature_noise (tests) injects the five tensors; otherwise the counter RNG draws them.
                nz, fe = [], []
                given = getattr(self.model, "feature_noise", None)
                for i, f in enumerate(feats):
                    hwc = f.shape[1] * f.shape[2] * f.shape[3]
                    z = self.buf(slot, f"dec{di}.noise{i}", (f.shape[1], f.shape[2], f.shape[3]), torch.float32)
                    if given is not None:
                        z.copy_(given[i].to(device=self.dev, dtype=torch.float32).permute(1, 2, 0))      # [C,H,W] -> [H,W,C]
                    else:
                        call("wsl_uniform_fill", (di + 1) * 104729 + i, self.seed_dev, hwc, -0.3, 0.3, z)
                    d = self.buf(slot, f"dec{di}.noisy{i}", tuple(f.shape))
                    call("wsl_feat_noise_fwd", f, self.dt, z, N, hwc, d)
                    nz.append(z)
                    fe.append(d)
                drec["noise"] = nz
            elif self.aux[di]:
                cs, fe = [], []
                for i, f in enumerate(feats):
                    c = self.buf(slot, f"dec{di}.cs{i}", (N, ft[i]), torch.float32)
                    if chan_keep is not None:
                        c.copy_(chan_keep[i].to(device=self.dev, dtype=torch.float32) * 2.0)
                    else:
                        call("wsl_chan_mask_gen", (di + 1) * 7919 + i, self.seed_dev, N * ft[i], 0.5, c)
                    d = self.buf(slot, f"dec{di}.drop{i}", tuple(f.shape))
                    call("wsl_chan_scale", f, self.dt, c, N, f.shape[1], f.shape[2], ft[i], d)
                    cs.append(c)
                    fe.append(d)
                drec["cs"] = cs
            xlow = fe[4]
            hh, ww = H // 16, W // 16
            for j, (c1, blk) in enumerate(ups):
                skip = fe[3 - j]
                C2 = c1.Cout
                t = self.buf(slot, f"dec{di}.up{j}.t", (N, hh, ww, C2))
                self.conv_fwd(c1, [xlow], t, 0, N, hh, ww, C2)
                u = self.buf(slot, f"dec{di}.up{j}.u", (N, 2 * hh, 2 * ww, C2))
                self._tag_bytes("up_fwd", c1, N * hh * ww * C2 * (4 if self.dt == 1 else 2) * 5)
                call("wsl_upsample2x_fwd", t, self.dt, N, hh, ww, C2, u)
                self._untag()
                hh, ww = 2 * hh, 2 * ww
                r = run_block(f"dec{di}.up{j}", blk, [skip, u], hh, ww, None, pool=False)
                r["xlow"] = xlow
                drec["ups"].append(r)
                xlow = r["a2"]
                if j in self.ds_heads[di]:       # Decoder_DS: class head on this level, nearest-resized to the input size
                    small = self.buf(slot, f"dec{di}.dp{j}.small", (N, self.n_class, hh, ww), torch.float32)
                    self.conv_fwd(self.ds_heads[di][j], [xlow], small, 1, N, hh, ww, self.n_class)
                    full = torch.empty((N, self.n_class, H, W), dtype=torch.float32, device=self.dev)
                    call("wsl_nearest_resize_fwd", small, N * self.n_class, hh, ww, H, W, full)
                    drec.setdefault("dp", {})[j] = full
            self.conv_fwd(oc, [xlow], outs[di], 1, N, H, W, self.n_class)
            drec["xlast"] = xlow
            return drec

        drecs = [None] * len(self.dec)
        for di in range(1, len(self.dec)):                  # aux passes first, on the side stream, in the reference's order
            with self.on_side():                            # (a decoder that runs twice updates its running statistics twice)
                drecs[di] = run_decoder(di, *self.dec[di])
        drecs[0] = run_decoder(0, *self.dec[0])
        if not (defer_join and need_grad):
            self.join_side()           # otherwise backward() joins: the aux outputs must not be read before that
        rec["dec"] = drecs
        # deep-supervision outputs follow the decoders' main outputs: (dp1, dp2, dp3) = heads of up3, up2, up1 (unet.py:190)
        for di, heads in enumerate(self.ds_heads):
            if heads:
                self.join_side()
                outs = outs + [drecs[di]["dp"][j] for j in (2, 1, 0)]
        if need_grad:
            self._recs[slot] = rec
        return outs, slot

    # ---------------------------------------------------------------- slots
    def _acquire_slot(self):
        if not hasattr(self, "_recs"):
            self._recs = {}
        for s in range(self.MAX_SLOTS):
            if s not in self._live:
                self._live.append(s)
                return s
        s = self._live.pop(0)  # recycle the oldest forward whose backward never came
        self._live.append(s)
        return s

    # ---------------------------------------------------------------- backward
    def backward(self, slot, grad_logits: Sequence[Optional[torch.Tensor]], zero_grads=True):
        rec = self._recs.pop(slot)
        if slot in self._live:
            self._live.remove(slot)
        N, H, W = rec["N"], rec["H"], rec["W"]
        ft = self.ft
        gflat, _ = self.grads()
        S = self.grad_scale_for(N, H, W)
        if zero_grads:
            gflat.zero_()
        elif S != 1.0:
            gflat.mul_(S)                      # the bucket holds unscaled gradients of an earlier pass: bring them to this pass' scale
        self._accumulate = not zero_grads      # BN affine gradients are written (not added) unless accumulating
        if zero_grads or not hasattr(self, "last_backward_param_ids"):
            self.last_backward_param_ids = set()   # ids of the parameters this backward (chain) produced gradients for
        B = lambda name, shape, dt=None: self.buf(slot, "g." + name, shape, dt)

        def block_bwd(tag, blk, r, g0, g1=None, cs1=None, gpool=None, need_dsrc=True):
            """returns list of gradients w.r.t. the block's sources (None for the image)."""
            l1, l2 = blk
            h, w, C = r["h"], r["w"], l1.Cout
            dy2 = B(tag + ".dy2", (N, h, w, C))
            self.bn_bwd(l2, r["y2"], r["ss2"], r["sv2"], g0, g1, cs1, gpool, r["pidx"] if gpool is not None else None,
                        None, dy2, N, h, w, slot, tag + ".bn2")
            with self.on_side():
                self.conv_wgrad(l2, [r["a1"]], dy2, N, h, w)
            da1 = B(tag + ".da1", (N, h, w, C))
            self.conv_dgrad(l2, 0, dy2, da1, N, h, w)
            if r["src_f32"] and l1.Cin == 1 and l1.Cout == 16 and l1.ks == 3 and self.sync_bn is None:
                # first layer: BatchNorm backward + weight gradient in one pass, dY never stored (no data gradient towards the image)
                bn = l1.bn
                self.last_backward_param_ids.update(id(q) for q in (bn.weight, bn.bias, l1.conv.weight, l1.conv.bias))
                coef = self.buf(slot, tag + ".bn1.coef", (2 * C,), torch.float32)
                p1 = l1.drop_p
                self._tag_bytes("bn_bwd_first", l1, N * h * w * C * (4 if self.dt == 1 else 2) * 4)
                call("wsl_bn_bwd_first", r["y1"], self.dt, r["ss1"], r["sv1"], da1, r["mask"], self._layer_seed(l1),
                     self.seed_dev if r["mask"] is None and p1 > 0 else None, p1, LRELU_SLOPE, N, h, w, self.gview(bn.weight),
                     self.gview(bn.bias), coef, r["srcs"][0], self.gview(l1.conv.weight), self._ws("bn"), 1 if self._accumulate else 0)
                self._untag()
                return []
            dy1 = B(tag + ".dy1", (N, h, w, C))
            self.bn_bwd(l1, r["y1"], r["ss1"], r["sv1"], da1, None, None, None, None, r["mask"], dy1, N, h, w, slot,
                        tag + ".bn1")
            with self.on_side():
                self.conv_wgrad(l1, r["srcs"], dy1, N, h, w, r["src_f32"])
            outs = []
            if need_dsrc:
                for i, c in enumerate(l1.srcC):
                    d = B(tag + f".dsrc{i}", (N, h, w, c))
                    self.conv_dgrad(l1, i, dy1, d, N, h, w)
                    outs.append(d)
            return outs

        # ---- decoders ----
        skip_grads = [[] for _ in range(5)]   # per encoder level: list of (grad, cs or None)
        # gradients of the deep-supervision outputs (they follow the decoders' main outputs in forward()'s list)
        ds_grads, nxt = {}, len(self.dec)
        for di, heads in enumerate(self.ds_heads):
            if heads:
                for j in (2, 1, 0):
                    if nxt < len(grad_logits) and grad_logits[nxt] is not None:
                        ds_grads[(di, j)] = grad_logits[nxt]
                    nxt += 1

        def tag_of(drec, lvl):
            """how the encoder feature of level lvl entered this decoder pass: None (as is), a [N,C] channel scale (F.dropout2d)
            or ("noise", z) for FeatureNoise (d feature = d noisy * (1 + z))"""
            if drec.get("noise") is not None:
                return ("noise", drec["noise"][lvl])
            return drec["cs"][lvl] if drec["cs"] else None

        def decoder_bwd(di, ups, oc, g, drec):
            if isinstance(g, tuple):                      # ("nhwc16", tensor): already in the executor's layout
                dl = g[1]
            else:
                g = g.contiguous()
                dl = B(f"dec{di}.dl", (N, H, W, 16))
                call("wsl_nchw_f32_to_nhwc", g, N, self.n_class, H, W, 16, dl, self.dt, S)
            with self.on_side():
                self.conv_wgrad(oc, [drec["xlast"]], dl, N, H, W)
            da = B(f"dec{di}.dlast", (N, H, W, ft[0]))
            self.conv_dgrad(oc, 0, dl, da, N, H, W)
            for j in range(3, -1, -1):
                c1, blk = ups[j]
                r = drec["ups"][j]
                gh = ds_grads.get((di, j))
                dh = None
                if gh is not None:                # gradient arriving at the deep-supervision head of this level
                    hl = self.ds_heads[di][j]
                    hh_, ww_, Ch = r["h"], r["w"], hl.Cin
                    gs = B(f"dec{di}.dp{j}.gs", (N, self.n_class, hh_, ww_), torch.float32)
                    call("wsl_nearest_resize_bwd", gh.contiguous(), N * self.n_class, hh_, ww_, H, W, gs)
                    dl16 = B(f"dec{di}.dp{j}.dl", (N, hh_, ww_, 16))
                    call("wsl_nchw_f32_to_nhwc", gs, N, self.n_class, hh_, ww_, 16, dl16, self.dt, S)
                    with self.on_side():
                        self.conv_wgrad(hl, [r["a2"]], dl16, N, hh_, ww_)
                    dh = B(f"dec{di}.dp{j}.dh", (N, hh_, ww_, Ch))
                    self.conv_dgrad(hl, 0, dl16, dh, N, hh_, ww_)
                dskip, du = block_bwd(f"dec{di}.up{j}", blk, r, da, dh)
                lvl = 3 - j
                skip_grads[lvl].append((dskip, tag_of(drec, lvl)))
                hh, ww, C2 = r["h"] // 2, r["w"] // 2, c1.Cout
                dt = B(f"dec{di}.up{j}.dt", (N, hh, ww, C2))
                self._tag_bytes("up_bwd", c1, N * hh * ww * C2 * (4 if self.dt == 1 else 2) * 5)
                call("wsl_upsample2x_bwd", du, self.dt, N, hh, ww, C2, dt)
                self._untag()
                with self.on_side():
                    self.conv_wgrad(c1, [r["xlow"]], dt, N, hh, ww)
                da = B(f"dec{di}.up{j}.dxlow", (N, hh, ww, c1.Cin))
                self.conv_dgrad(c1, 0, dt, da, N, hh, ww)
            skip_grads[4].append((da, tag_of(drec, 4)))

        # aux decoder chains run on their own streams beside the main decoder's (HBM-bound BatchNorm backward of one chain
        # overlaps the tensor-core data gradients of the other); the encoder needs all of them
        chains = []
        seen_decoders = set()
        base_accumulate = self._accumulate
        for di, (ups, oc) in enumerate(self.dec):
            g = grad_logits[di] if di < len(grad_logits) else None
            if g is None and any(k[0] == di for k in ds_grads):     # only deep-supervision heads were used in the loss
                g = torch.zeros((N, self.n_class, H, W), dtype=torch.float32, device=self.dev)
            if g is None:
                continue
            didx = self.runs[di][0]
            # a second pass through the same decoder ADDS its BatchNorm affine gradients (weight gradients always accumulate) and
            # runs on the same stream as the first one, so the two never touch the shared gradient rows concurrently
            self._accumulate = base_accumulate or (didx in seen_decoders)
            seen_decoders.add(didx)
            if di > 0 and self.multi_stream:
                nm = f"dec{didx}"
                with self.on_side(nm):
                    decoder_bwd(di, ups, oc, g, rec["dec"][di])
                if nm not in chains:
                    chains.append(nm)
            else:
                decoder_bwd(di, ups, oc, g, rec["dec"][di])
        self._accumulate = base_accumulate
        for nm in chains:
            self.join_side(nm)
        if self.on_decoders_done is not None:
            # data-parallel step: every decoder gradient is final once the decoders' weight-gradient launches (side stream) have
            # joined -- the caller starts the all-reduce of that slice of the flat bucket here, underneath the encoder's backward
            self.join_side("side")
            self.on_decoders_done(gflat)

        # ---- encoder ----
        gpool = None
        for i in range(4, -1, -1):
            r = rec["enc"][i]
            srcs = skip_grads[i]
            plain = [g for g, cs in srcs if cs is None]
            noisy = [(g, cs[1]) for g, cs in srcs if isinstance(cs, tuple)]
            scaled = [(g, cs) for g, cs in srcs if cs is not None and not isinstance(cs, tuple)]
            for gn, z in noisy:            # FeatureNoise pass: fold d noisy * (1 + z) into the plain skip gradient (or make it the plain one)
                hwc = gn.shape[1] * gn.shape[2] * gn.shape[3]
                call("wsl_feat_noise_bwd", gn, self.dt, z, N, hwc, plain[0] if plain else None, gn)
                if not plain:
                    plain = [gn]
            assert len(plain) <= 1 and len(scaled) <= 1
            g0 = plain[0] if plain else None
            g1, cs1 = scaled[0] if scaled else (None, None)
            d = block_bwd(f"enc{i}", self.enc_blocks[i], r, g0, g1, cs1, gpool, need_dsrc=(i > 0))
            gpool = d[0] if i > 0 else None
        self.join_side()
        if S != 1.0:
            gflat.mul_(1.0 / S)                # power of two: exact
        return gflat
