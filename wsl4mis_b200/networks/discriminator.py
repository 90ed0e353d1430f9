"""FCDiscriminator with the reference's public names, constructor signature and state_dict layout (networks/discriminator.py:58-101),
executed on the wsl4mis_b200 kernels.

Every nn.Conv2d(k=4, stride=2, padding=1) runs as a 3x3 / stride-1 / pad-1 convolution over the space-to-depth tensor
T[n, Y, X, (a*2+b)*Cin + c] = x[n, 2Y+a, 2X+b, c] with a structured weight (each 4x4 tap in one of the 36 (tap, phase) slots, the rest
zero), so the forward, data gradient and weight gradient are the existing 3x3 convolutions: the per-tap wgmma kernel in bf16 mode, the
CUDA-core direct kernels in fp32 mode.  conv0 (map) and conv1 (feature) are one convolution over the packed pair with bias b0 + b1.
The parameters are ordinary fp32 nn.Parameters (the DAN script updates them with torch.optim.Adam); the operands are repacked on every
forward.  Only 256 x 256 inputs are accelerated: that is the scripts' patch size, and the only size of the reference's valid range
(conv4 output 14..20, fixed by Linear(ndf*32, 2)) whose half-resolution maps tile the 8 x 16 pixel tiles of the kernels."""
import torch
import torch.nn as nn

from .._lib import call, workspace
from ._engine import initial_rng_counter

SLOPE = 0.2                 # nn.LeakyReLU(negative_slope=0.2) (discriminator.py:74)
DROP_P = 0.5                # nn.Dropout2d(0.5) (:75)
HW = 256
_DT = {"bf16": 0, "fp32": 1}


def _ceil16(c):
    return (c + 15) // 16 * 16


class _Layer:
    """one space-to-depth convolution: input C channels at h x w -> Cout channels at h/2 x w/2; CP = 4C padded to 16"""

    def __init__(self, convs, h):
        self.convs = convs                      # (conv0, conv1) for the first layer, (convK,) otherwise
        self.cins = [c.in_channels for c in convs]
        self.C = sum(self.cins)
        self.CP = _ceil16(4 * self.C)
        self.Cout = convs[0].out_channels
        self.h = h                              # output resolution


class _DiscExecutor:
    def __init__(self, model, precision):
        self.model, self.precision, self.dt = model, precision, _DT[precision]
        self.act = torch.bfloat16 if self.dt == 0 else torch.float32
        m = model
        self.layers = [_Layer((m.conv0, m.conv1), HW // 2), _Layer((m.conv2,), HW // 4), _Layer((m.conv3,), HW // 8),
                       _Layer((m.conv4,), HW // 16)]
        self.seed_dev = None
        self._partials = None

    # ---- operands ----------------------------------------------------------------------------------------------------------------
    def _pack(self, L, need_dgrad, dev):
        """structured 3x3 weight -> forward pack (and the flipped / transposed data-gradient pack); bias (b0 + b1 for the first layer)"""
        c = L.convs
        w3 = torch.empty(L.Cout * L.CP * 9, dtype=torch.float32, device=dev)
        bias = torch.empty(L.Cout, dtype=torch.float32, device=dev)
        w1, b1 = (c[1].weight, c[1].bias) if len(c) > 1 else (None, None)
        call("wsl_disc_scatter_weights", c[0].weight.detach(), c[0].bias.detach(), L.cins[0], None if w1 is None else w1.detach(),
             None if b1 is None else b1.detach(), L.cins[1] if len(c) > 1 else 0, L.Cout, L.CP, w3, bias)
        n = 9 * L.Cout * L.CP
        if self.dt == 0:
            fwd = torch.empty(n, dtype=torch.bfloat16, device=dev)
            dgr = torch.empty(n, dtype=torch.bfloat16, device=dev) if need_dgrad else None
            call("wsl_pack_conv_weights", w3, L.Cout, L.CP, 3, L.Cout, L.CP, 0, L.CP, None, None, fwd, dgr, 0)
        else:
            fwd = torch.empty(n, dtype=torch.float32, device=dev)
            dgr = torch.empty(n, dtype=torch.float32, device=dev) if need_dgrad else None
            call("wsl_pack_conv_weights", w3, L.Cout, L.CP, 3, L.Cout, L.CP, 0, L.CP, fwd, dgr, None, None, 0)
        return fwd, dgr, bias

    def _conv(self, L, T, wpk, bias, N):
        h = L.h
        y = torch.empty((N, h, h, L.Cout), dtype=self.act, device=T.device)
        if self.dt == 0:
            call("wsl_conv_tc", T, L.CP, None, 0, wpk, bias, y, 0, N, h, h, L.Cout, L.Cout, 3, 0)
        else:
            call("wsl_conv_direct", T, L.CP, None, 0, 1, wpk, bias, y, 2, N, h, h, L.CP, L.Cout, L.Cout, 3)
        return y

    def _dgrad(self, L, dy, dpk, N):
        h = L.h
        dT = torch.empty((N, h, h, L.CP), dtype=self.act, device=dy.device)
        if self.dt == 0:
            call("wsl_conv_tc", dy, L.Cout, None, 0, dpk, None, dT, 0, N, h, h, L.CP, L.CP, 3, 0)
        else:
            call("wsl_conv_direct", dy, L.Cout, None, 0, 1, dpk, None, dT, 2, N, h, h, L.Cout, L.CP, L.CP, 3)
        return dT

    def _wgrad(self, L, T, dy, N):
        """-> (weight gradients of the layer's convs in torch layout, bias gradient)"""
        h, dev = L.h, dy.device
        dw3 = torch.zeros(L.Cout * L.CP * 9, dtype=torch.float32, device=dev)
        if self.dt == 0:
            if self._partials is None or self._partials.device != dev:
                self._partials = torch.empty(8 * 1024 * 1024, dtype=torch.float32, device=dev)   # split-K tiles: bit-stable sums
            call("wsl_wgrad_tc", T, L.CP, None, 0, dy, L.Cout, dw3, N, h, h, L.Cout, 3, 0, self._partials, self._partials.numel())
        else:
            call("wsl_wgrad_direct", T, L.CP, None, 0, 1, dy, 1, L.Cout, dw3, None, N, h, h, L.Cout, 3)
        dws = [torch.empty_like(c.weight) for c in L.convs]
        call("wsl_disc_gather_wgrad", dw3, L.Cout, L.CP, L.cins[0], L.cins[1] if len(L.cins) > 1 else 0, dws[0],
             dws[1] if len(dws) > 1 else None)
        db = torch.zeros(L.Cout, dtype=torch.float32, device=dev)
        call("wsl_channel_sum", dy, self.dt, N * h * h, L.Cout, L.Cout, db, workspace("disc_csum", dev))
        return dws, db

    # ---- forward / backward ------------------------------------------------------------------------------------------------------
    def forward(self, mp, feat, training, need_grad, need_input_grad, keep):
        N, dev = mp.shape[0], mp.device
        if self.seed_dev is None or self.seed_dev.device != dev:
            self.seed_dev = torch.full((1,), initial_rng_counter(), dtype=torch.int64, device=dev)
        if training:
            self.seed_dev.add_(1)
        L0 = self.layers[0]
        packs = [self._pack(L, need_grad and (i > 0 or need_input_grad), dev) for i, L in enumerate(self.layers)]
        T = torch.empty((N, HW // 2, HW // 2, L0.CP), dtype=self.act, device=dev)
        call("wsl_disc_pack_input", mp, L0.cins[0], feat, L0.cins[1], N, HW, HW, L0.CP, T, self.dt)
        Ts, ys, css = [T], [], []
        for i, L in enumerate(self.layers):
            y = self._conv(L, Ts[-1], packs[i][0], packs[i][2], N)
            ys.append(y)
            if i == 3:
                break
            # conv0 + conv1 has no activation (discriminator.py:83-85); conv2, conv3: LeakyReLU -> Dropout2d (:86-91)
            slope, cs = (1.0, None) if i == 0 else (SLOPE, self._mask(i, N, L.Cout, training, keep, dev))
            css.append(cs)
            Tn = torch.empty((N, L.h // 2, L.h // 2, 4 * L.Cout), dtype=self.act, device=dev)
            call("wsl_s2d_act_fwd", y, self.dt, N, L.h, L.h, L.Cout, slope, cs, Tn)
            Ts.append(Tn)
        m = self.model
        C4 = self.layers[3].Cout
        pooled = torch.empty((N, 4 * C4), dtype=torch.float32, device=dev)
        logits = torch.empty((N, 2), dtype=torch.float32, device=dev)
        call("wsl_disc_head_fwd", ys[3], self.dt, N, C4, SLOPE, m.classifier.weight.detach(), m.classifier.bias.detach(), pooled, logits)
        rec = {"N": N, "Ts": Ts, "ys": ys, "css": css, "packs": packs, "pooled": pooled} if need_grad else None
        return logits, rec

    def _mask(self, i, N, C, training, keep, dev):
        """Dropout2d(0.5) scale [N, C] in {0, 2} after conv2 (i = 1) / conv3 (i = 2); None in eval mode"""
        if not training:
            return None
        cs = torch.empty((N, C), dtype=torch.float32, device=dev)
        if keep is not None:
            cs.copy_(keep[i - 1].to(device=dev, dtype=torch.float32) * (1.0 / (1.0 - DROP_P)))
        else:
            call("wsl_chan_mask_gen", 6271 * i, self.seed_dev, N * C, DROP_P, cs)
        return cs

    def backward(self, rec, dlogits, need_map, need_feat):
        """-> (d map, d feature, [12 parameter gradients in model.parameters() order])"""
        N, Ts, ys, css, packs = rec["N"], rec["Ts"], rec["ys"], rec["css"], rec["packs"]
        m, dev = self.model, dlogits.device
        C4 = self.layers[3].Cout
        dy = torch.empty_like(ys[3])
        dwc, dbc = torch.empty_like(m.classifier.weight), torch.empty_like(m.classifier.bias)
        call("wsl_disc_head_bwd", dlogits.contiguous(), rec["pooled"], ys[3], self.dt, N, C4, SLOPE, m.classifier.weight.detach(), dwc, dbc, dy)
        grads = {}
        dmap = dfeat = None
        for i in range(3, -1, -1):
            L = self.layers[i]
            dws, db = self._wgrad(L, Ts[i], dy, N)
            for conv, dw in zip(L.convs, dws):
                grads[id(conv.weight)], grads[id(conv.bias)] = dw, db
            if i == 0 and not (need_map or need_feat):
                break
            dT = self._dgrad(L, dy, packs[i][1], N)
            if i == 0:
                L0 = self.layers[0]
                dmap = torch.empty((N, L0.cins[0], HW, HW), dtype=torch.float32, device=dev) if need_map else None
                dfeat = torch.empty((N, L0.cins[1], HW, HW), dtype=torch.float32, device=dev) if need_feat else None
                call("wsl_disc_unpack_input_grad", dT, self.dt, N, HW, HW, L0.CP, L0.cins[0], L0.cins[1], dmap, dfeat)
                break
            P = self.layers[i - 1]
            dy = torch.empty_like(ys[i - 1])
            if i == 1:      # conv0 + conv1 output: no activation
                call("wsl_d2s_act_bwd", dT, None, self.dt, N, P.h, P.h, P.Cout, 1.0, None, dy)
            else:
                call("wsl_d2s_act_bwd", dT, ys[i - 1], self.dt, N, P.h, P.h, P.Cout, SLOPE, css[i - 1], dy)
        grads[id(m.classifier.weight)], grads[id(m.classifier.bias)] = dwc, dbc
        grads[id(m.conv1.bias)] = grads[id(m.conv0.bias)].clone()   # both biases feed the same sum
        return dmap, dfeat, [grads[id(p)] for p in m.parameters()]


class _DiscFn(torch.autograd.Function):
    """Whole-discriminator autograd node: forward = executor.forward, backward = executor.backward."""

    @staticmethod
    def forward(ctx, mp, feat, holder, training, need, keep, *params):
        ex = holder.executor
        need_in = need and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        logits, rec = ex.forward(mp, feat, training, need, need_in, keep)
        ctx.ex, ctx.rec = ex, rec
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        rec, ctx.rec = ctx.rec, None
        dmap, dfeat, grads = ctx.ex.backward(rec, dlogits, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        grads = [g if ctx.needs_input_grad[6 + i] else None for i, g in enumerate(grads)]
        return (dmap, dfeat, None, None, None, None) + tuple(grads)


class _Holder:
    def __init__(self, executor):
        self.executor = executor


class FCDiscriminator(nn.Module):
    """reference discriminator.py:58-101: FCDiscriminator(num_classes, ndf=64, n_channel=1); forward(map, feature) -> [N, 2] fp32 logits.
    ``channel_keep`` (tests): the two [N, C] keep masks of the Dropout2d layers after conv2 and conv3; otherwise they come from the
    device counter RNG.  ``set_precision('bf16' | 'fp32')``: wgmma on bf16 operands (default) or the CUDA-core fp32 cross-check."""

    precision = "bf16"

    def __init__(self, num_classes, ndf=64, n_channel=1):
        super().__init__()
        if ndf % 16 != 0:
            raise ValueError(f"FCDiscriminator: ndf must be a multiple of 16 on the tensor-core kernels (got {ndf})")
        self.num_classes, self.ndf, self.n_channel = num_classes, ndf, n_channel
        self.conv0 = nn.Conv2d(num_classes, ndf, kernel_size=4, stride=2, padding=1)
        self.conv1 = nn.Conv2d(n_channel, ndf, kernel_size=4, stride=2, padding=1)
        self.conv2 = nn.Conv2d(ndf, ndf * 2, kernel_size=4, stride=2, padding=1)
        self.conv3 = nn.Conv2d(ndf * 2, ndf * 4, kernel_size=4, stride=2, padding=1)
        self.conv4 = nn.Conv2d(ndf * 4, ndf * 8, kernel_size=4, stride=2, padding=1)
        self.classifier = nn.Linear(ndf * 32, 2)
        self.avgpool = nn.AvgPool2d((7, 7))
        self.leaky_relu = nn.LeakyReLU(negative_slope=SLOPE, inplace=True)
        self.dropout = nn.Dropout2d(DROP_P)
        self.channel_keep = None
        self._holder = None

    def set_precision(self, precision):
        """'bf16' (default): bf16 activations and operands on the wgmma kernels; 'fp32': fp32 storage on the CUDA-core direct
        convolutions, the arithmetic cross-check"""
        if precision not in _DT:
            raise ValueError(f"FCDiscriminator precision must be one of {sorted(_DT)} (got {precision!r})")
        object.__setattr__(self, "precision", precision)
        object.__setattr__(self, "_holder", None)
        return self

    @property
    def executor(self):
        if self._holder is None:
            object.__setattr__(self, "_holder", _Holder(_DiscExecutor(self, self.precision)))
        return self._holder.executor

    def forward(self, map, feature):
        for name, t, c in (("map", map, self.num_classes), ("feature", feature, self.n_channel)):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
                raise TypeError(f"FCDiscriminator: {name} must be a CUDA fp32 tensor (got {getattr(t, 'dtype', type(t))} on "
                                f"{getattr(t, 'device', '-')}); there is no CPU path")
            if t.dim() != 4 or t.shape[1] != c or t.shape[2] != HW or t.shape[3] != HW or t.shape[0] != map.shape[0]:
                raise ValueError(f"FCDiscriminator: {name} of shape {tuple(t.shape)}; the kernels take [N, {c}, {HW}, {HW}] "
                                 f"(the scripts' patch size)")
        self.executor
        params = list(self.parameters())
        need = torch.is_grad_enabled() and (map.requires_grad or feature.requires_grad or any(p.requires_grad for p in params))
        return _DiscFn.apply(map.contiguous(), feature.contiguous(), self._holder, self.training, need, self.channel_keep, *params)
