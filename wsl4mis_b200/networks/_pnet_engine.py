"""Planned executor for PNet2D (reference networks/pnet.py:87-122; net_factory builds PNet2D(in_chns, class_num, 64, [1, 2, 4, 8, 16])).

Five blocks of two DILATED 3x3 convolutions (dilation = padding = 1, 2, 4, 8, 16) + BatchNorm + LeakyReLU at full resolution, the
concatenation of the five block outputs, two 1x1 convolutions with LeakyReLU and no BatchNorm, and the output block
Dropout2d(0.3) -> conv1x1 -> LeakyReLU -> Dropout2d(0.3) -> conv1x1.  Everything runs on the kernels of the U-Net executor: the
dilated convolutions on the per-tap wgmma kernel (a tap is the TMA box at (y + d*dy, x + d*dx); zero fill = padding), the 1x1
convolutions on the persistent resident-weight kernel, BatchNorm / LeakyReLU / channel dropout on the same elementwise kernels
(LeakyReLU without BatchNorm: `wsl_lrelu_fwd` / `wsl_lrelu_bwd`).  Modes: bf16, fp16 and
fp16x3 (fp32-accurate split operands); there is no dilated CUDA-core kernel, so the plain `fp32` cross-check mode is not offered.

The training steps of engine.py run on it as on the U-Net executor: one output, no aux parameters, and no encoder/decoder split for
a data-parallel step to overlap its all-reduce with (the whole bucket is reduced after backward).  Synchronised BatchNorm over
data-parallel ranks (`sync_bn`, TrainStep(global_batch=True)) is not implemented for it.
"""
import torch

from .._lib import call
from ._engine import ConvLayer, LRELU_SLOPE, UNetExecutor


class PNetExecutor(UNetExecutor):
    def __init__(self, model, precision="bf16"):
        assert precision in ("bf16", "fp16", "fp16x3"), "PNet2D runs in bf16, fp16 or fp16x3 mode (no dilated CUDA-core kernel)"
        self.in_chns, self.n_class, self.nf = model.in_chns, model.out_chns, model.num_filters
        nf = self.nf
        self.layers = []
        self.blocks = []
        for b in range(1, 6):
            blk = getattr(model, f"block{b}")
            l1 = ConvLayer(f"block{b}.conv1", blk.conv1, blk.in1, 0.0, [blk.conv1.in_channels])
            l2 = ConvLayer(f"block{b}.conv2", blk.conv2, blk.in2, 0.0, [nf])
            self.layers += [l1, l2]
            self.blocks.append((l1, l2))
        self.cat1 = ConvLayer("catblock.conv1", model.catblock.conv1, None, 0.0, [nf] * 5)
        self.cat2 = ConvLayer("catblock.conv2", model.catblock.conv2, None, 0.0, [5 * nf])
        self.out1 = ConvLayer("out.conv1", model.out.conv1, None, 0.0, [2 * nf])
        self.out2 = ConvLayer("out.conv2", model.out.conv2, None, 0.0, [nf])
        self.layers += [self.cat1, self.cat2, self.out1, self.out2]
        self._init_runtime(model, precision)
        self.multi_stream = False           # a single chain: nothing to overlap
        self.n_outputs = 1
        self.aux_param_ids = set()
        self.comm_split = None              # no decoder half that finishes early: no all-reduce inside backward()

    @property
    def sync_bn(self):
        return None

    @sync_bn.setter
    def sync_bn(self, value):
        if value is not None:
            raise NotImplementedError("synchronised BatchNorm (TrainStep(global_batch=True)) is not implemented for PNet2D; "
                                      "its data-parallel steps keep per-rank BatchNorm statistics")

    def _lrelu(self, y, act, N, H, W, C):
        """nn.LeakyReLU between the 1x1 convolutions of ConcatBlock / OutPutBlock (pnet.py:60-61,94-95): no BatchNorm in front"""
        call("wsl_lrelu_fwd", y, self.dt, LRELU_SLOPE, N * H * W * C, act)

    def _chan_drop(self, slot, name, x, N, H, W, C, training, keep, salt):
        """nn.Dropout2d(0.3) (pnet.py:72-73): per-(n, c) keep mask scaled by 1 / 0.7; identity in eval mode"""
        if not training:
            return x, None
        cs = self.buf(slot, name + ".cs", (N, C), torch.float32)
        if keep is not None:
            cs.copy_(keep.to(device=self.dev, dtype=torch.float32) * (1.0 / 0.7))
        else:
            call("wsl_chan_mask_gen", 7919 * salt, self.seed_dev, N * C, 0.3, cs)
        d = self.buf(slot, name + ".d", (N, H, W, C))
        call("wsl_chan_scale", x, self.dt, cs, N, H, W, C, d)
        return d, cs

    # ---- forward ------------------------------------------------------------------------------------------------------------------
    def forward(self, x, training, need_grad, masks=None, chan_keep=None, defer_join=False, bn_per_sample=False):
        """x: fp32 [N, 1, H, W] CUDA -> ([fp32 NCHW logits], slot).  chan_keep: the two Dropout2d keep masks [N, 128] and [N, 64]
        (None: drawn on the device).  bn_per_sample (training, no gradient): what N batch-1 training forwards compute -- every
        BatchNorm normalises each image by its own statistics and the running statistics take the N updates in batch order;
        Dropout2d stays on, one mask per image as in N separate forwards (the Scribble2Label refresh, train_s2l.py:221-228)."""
        if bn_per_sample:
            assert training and not need_grad, "bn_per_sample is a training-mode forward without gradient"
            self._bn_per_sample = True
            try:
                return self.forward(x, training, need_grad, masks, chan_keep, defer_join)
            finally:
                self._bn_per_sample = False
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == self.in_chns == 1
        N, _, H, W = x.shape
        assert H % 8 == 0 and W % 16 == 0, "PNet2D on the wgmma kernels needs H % 8 == 0 and W % 16 == 0"
        self.dev = x.device
        if not hasattr(self, "seed_dev") or self.seed_dev.device != self.dev:
            from ._engine import initial_rng_counter
            self.seed_dev = torch.full((1,), initial_rng_counter(), dtype=torch.int64, device=self.dev)
        x = x.contiguous()
        slot = self._acquire_slot() if need_grad else "ng"
        self.pack_all()
        if training:
            self.seed_dev.add_(1)
        nf = self.nf
        rec = {"N": N, "H": H, "W": W, "x": x, "blocks": []}
        src, src_f32 = [x], True
        feats = []
        for b, (l1, l2) in enumerate(self.blocks):
            r = {}
            for k, (L, s_in, f32) in enumerate(((l1, src, src_f32), (l2, None, False))):
                tag = f"pb{b}.{k}"
                y = self.buf(slot, tag + ".y", (N, H, W, nf))
                a = self.buf(slot, tag + ".a", (N, H, W, nf))
                inp = s_in if k == 0 else [r["a0"]]
                self.conv_fwd(L, inp, y, 0, N, H, W, nf, f32)
                sv, ss = self.bn_fwd(L, y, a, N, H, W, training, slot, tag + ".bn")
                r.update({f"y{k}": y, f"a{k}": a, f"sv{k}": sv, f"ss{k}": ss, f"in{k}": inp})
            r["src_f32"] = src_f32
            rec["blocks"].append(r)
            feats.append(r["a1"])
            src, src_f32 = [r["a1"]], False
        cat = self.buf(slot, "cat", (N, H, W, 5 * nf))
        torch.cat(feats, dim=3, out=cat)                                   # torch.cat([x1..x5], 1) (pnet.py:119) in channels-last storage
        y1 = self.buf(slot, "c1.y", (N, H, W, 5 * nf))
        a1 = self.buf(slot, "c1.a", (N, H, W, 5 * nf))
        self.conv_fwd(self.cat1, [cat], y1, 0, N, H, W, 5 * nf, srcC_override=[5 * nf])
        self._lrelu(y1, a1, N, H, W, 5 * nf)
        y2 = self.buf(slot, "c2.y", (N, H, W, 2 * nf))
        a2 = self.buf(slot, "c2.a", (N, H, W, 2 * nf))
        self.conv_fwd(self.cat2, [a1], y2, 0, N, H, W, 2 * nf)
        self._lrelu(y2, a2, N, H, W, 2 * nf)
        d1, cs1 = self._chan_drop(slot, "o.d1", a2, N, H, W, 2 * nf, training, None if chan_keep is None else chan_keep[0], 1)
        y3 = self.buf(slot, "o1.y", (N, H, W, nf))
        a3 = self.buf(slot, "o1.a", (N, H, W, nf))
        self.conv_fwd(self.out1, [d1], y3, 0, N, H, W, nf)
        self._lrelu(y3, a3, N, H, W, nf)
        d2, cs2 = self._chan_drop(slot, "o.d2", a3, N, H, W, nf, training, None if chan_keep is None else chan_keep[1], 2)
        out = torch.empty((N, self.n_class, H, W), dtype=torch.float32, device=self.dev)
        self.conv_fwd(self.out2, [d2], out, 1, N, H, W, self.n_class)
        rec.update({"cat": cat, "y1": y1, "a1": a1, "y2": y2, "a2": a2, "d1": d1, "cs1": cs1, "y3": y3, "a3": a3, "d2": d2, "cs2": cs2})
        if need_grad:
            if not hasattr(self, "_recs"):
                self._recs = {}
            self._recs[slot] = rec
        return [out], slot

    # ---- backward -----------------------------------------------------------------------------------------------------------------
    def backward(self, slot, grad_logits, zero_grads=True):
        rec = self._recs.pop(slot)
        if slot in self._live:
            self._live.remove(slot)
        N, H, W, nf = rec["N"], rec["H"], rec["W"], self.nf
        gflat, _ = self.grads()
        S = self.grad_scale_for(N, H, W)
        if zero_grads:
            gflat.zero_()
        elif S != 1.0:
            gflat.mul_(S)
        self._accumulate = not zero_grads
        self.last_backward_param_ids = set()
        B = lambda name, shape: self.buf(slot, "g." + name, shape)
        nvec = lambda C: N * H * W * C
        g = grad_logits[0]
        if isinstance(g, tuple):                # ("nhwc16", tensor): already in the executor's layout and scaled by S
            dl = g[1]
        else:
            dl = B("dl", (N, H, W, 16))
            call("wsl_nchw_f32_to_nhwc", g.contiguous(), N, self.n_class, H, W, 16, dl, self.dt, S)
        # out.conv2 <- Dropout2d <- LeakyReLU <- out.conv1 <- Dropout2d <- LeakyReLU <- catblock.conv2 <- LeakyReLU <- catblock.conv1
        self.conv_wgrad(self.out2, [rec["d2"]], dl, N, H, W)
        dd2 = B("dd2", (N, H, W, nf))
        self.conv_dgrad(self.out2, 0, dl, dd2, N, H, W)
        if rec["cs2"] is not None:
            call("wsl_chan_scale", dd2, self.dt, rec["cs2"], N, H, W, nf, dd2)
        dy3 = B("dy3", (N, H, W, nf))
        call("wsl_lrelu_bwd", rec["y3"], self.dt, dd2, LRELU_SLOPE, nvec(nf), dy3)
        self.conv_wgrad(self.out1, [rec["d1"]], dy3, N, H, W)
        dd1 = B("dd1", (N, H, W, 2 * nf))
        self.conv_dgrad(self.out1, 0, dy3, dd1, N, H, W)
        if rec["cs1"] is not None:
            call("wsl_chan_scale", dd1, self.dt, rec["cs1"], N, H, W, 2 * nf, dd1)
        dy2 = B("dy2", (N, H, W, 2 * nf))
        call("wsl_lrelu_bwd", rec["y2"], self.dt, dd1, LRELU_SLOPE, nvec(2 * nf), dy2)
        self.conv_wgrad(self.cat2, [rec["a1"]], dy2, N, H, W)
        da1 = B("da1", (N, H, W, 5 * nf))
        self.conv_dgrad(self.cat2, 0, dy2, da1, N, H, W)
        dy1 = B("dy1", (N, H, W, 5 * nf))
        call("wsl_lrelu_bwd", rec["y1"], self.dt, da1, LRELU_SLOPE, nvec(5 * nf), dy1)
        self.conv_wgrad(self.cat1, [rec["cat"]], dy1, N, H, W, srcC_override=[5 * nf])
        gfeat = []
        for i in range(5):                                     # data gradient per concatenated source: d x_{i+1}
            d = B(f"dfeat{i}", (N, H, W, nf))
            self.conv_dgrad(self.cat1, i, dy1, d, N, H, W)
            gfeat.append(d)
        # blocks 5 .. 1: x_b feeds the concat AND block b+1
        carry = None
        for b in range(4, -1, -1):
            l1, l2 = self.blocks[b]
            r = rec["blocks"][b]
            dyb = B(f"pb{b}.dy1", (N, H, W, nf))
            self.bn_bwd(l2, r["y1"], r["ss1"], r["sv1"], gfeat[b], carry, None, None, None, None, dyb, N, H, W, slot, f"pb{b}.1.bn")
            self.conv_wgrad(l2, [r["a0"]], dyb, N, H, W)
            da0 = B(f"pb{b}.da0", (N, H, W, nf))
            self.conv_dgrad(l2, 0, dyb, da0, N, H, W)
            dya = B(f"pb{b}.dy0", (N, H, W, nf))
            self.bn_bwd(l1, r["y0"], r["ss0"], r["sv0"], da0, None, None, None, None, None, dya, N, H, W, slot, f"pb{b}.0.bn")
            self.conv_wgrad(l1, r["in0"], dya, N, H, W, r["src_f32"])
            if b > 0:
                carry = B(f"pb{b}.dsrc", (N, H, W, nf))
                self.conv_dgrad(l1, 0, dya, carry, N, H, W)
        if S != 1.0:
            gflat.mul_(1.0 / S)
        return gflat
