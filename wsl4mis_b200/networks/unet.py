"""2D U-Net family with the reference's public names, constructor signatures, return types and
state_dict layout (networks/unet.py), executed by the wsl4mis_b200 planned executor.

The nn.Module tree below exists to own parameters/buffers under the reference's key names (202 keys for
UNet_CCT) and to consume torch's RNG in the reference's construction order, so that
``torch.manual_seed(s); UNet(1, 4)`` yields the reference's initial weights and checkpoints load both
ways.  ``forward`` of the whole-network classes never calls the per-layer modules: it hands the input to
``_engine.UNetExecutor`` (hand-written CUDA kernels, channels-last bf16 activations, fp32 master weights).
"""
import numpy as np
import torch
import torch.nn as nn
from torch.distributions.uniform import Uniform

from ._engine import UNetExecutor

_FT = [16, 32, 64, 128, 256]              # reference: unet.py:291
_DROP = [0.05, 0.1, 0.2, 0.3, 0.5]        # reference: unet.py:292


def _only_whole_network(self, *a, **k):
    raise NotImplementedError(
        f"{type(self).__name__} is a parameter container in wsl4mis_b200; run it through UNet / UNet_CCT "
        "(the fused executor owns the arithmetic of the hot path)")


class ConvBlock(nn.Module):
    """conv3x3-BN-LeakyReLU-Dropout-conv3x3-BN-LeakyReLU (reference unet.py:13-29); key prefix ``conv_conv.{0,1,4,5}``."""

    def __init__(self, in_channels, out_channels, dropout_p):
        super().__init__()
        layers = []
        for cin, p in ((in_channels, dropout_p), (out_channels, None)):
            layers += [nn.Conv2d(cin, out_channels, kernel_size=3, padding=1), nn.BatchNorm2d(out_channels), nn.LeakyReLU()]
            if p is not None:
                layers.append(nn.Dropout(p))
        self.conv_conv = nn.Sequential(*layers)

    forward = _only_whole_network


class DownBlock(nn.Module):
    """MaxPool2d(2) then ConvBlock (reference unet.py:32-44); key prefix ``maxpool_conv.1``."""

    def __init__(self, in_channels, out_channels, dropout_p):
        super().__init__()
        self.maxpool_conv = nn.Sequential(nn.MaxPool2d(2), ConvBlock(in_channels, out_channels, dropout_p))

    forward = _only_whole_network


class UpBlock(nn.Module):
    """conv1x1 -> bilinear x2 -> cat -> ConvBlock (reference unet.py:47-68, bilinear branch; the
    ConvTranspose branch is unreachable from every shipped model, SURVEY F4)."""

    def __init__(self, in_channels1, in_channels2, out_channels, dropout_p, bilinear=True):
        super().__init__()
        if not bilinear:
            raise NotImplementedError("only the bilinear UpBlock is on the WSL4MIS hot path (SURVEY F4)")
        self.bilinear = True
        self.conv1x1 = nn.Conv2d(in_channels1, in_channels2, kernel_size=1)
        self.up = nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True)
        self.conv = ConvBlock(in_channels2 * 2, out_channels, dropout_p)

    forward = _only_whole_network


class Encoder(nn.Module):
    """reference unet.py:71-98"""

    def __init__(self, params):
        super().__init__()
        self.params = params
        self.in_chns, self.ft_chns, self.n_class = params['in_chns'], params['feature_chns'], params['class_num']
        self.bilinear, self.dropout = params['bilinear'], params['dropout']
        assert len(self.ft_chns) == 5
        chans = [self.in_chns] + list(self.ft_chns)
        self.in_conv = ConvBlock(chans[0], chans[1], self.dropout[0])
        for i in range(1, 5):
            setattr(self, f"down{i}", DownBlock(chans[i], chans[i + 1], self.dropout[i]))

    forward = _only_whole_network


class Decoder(nn.Module):
    """reference unet.py:101-135"""

    def __init__(self, params):
        super().__init__()
        self.params = params
        self.in_chns, self.ft_chns, self.n_class = params['in_chns'], params['feature_chns'], params['class_num']
        self.bilinear = params['bilinear']
        assert len(self.ft_chns) == 5
        f = self.ft_chns
        for j in range(1, 5):
            setattr(self, f"up{j}", UpBlock(f[5 - j], f[4 - j], f[4 - j], dropout_p=0.0))
        self.out_conv = nn.Conv2d(f[0], self.n_class, kernel_size=3, padding=1)

    forward = _only_whole_network


def _params(in_chns, class_num):
    return {'in_chns': in_chns, 'feature_chns': list(_FT), 'dropout': list(_DROP), 'class_num': class_num,
            'bilinear': False, 'acti_func': 'relu'}


class _NetFn(torch.autograd.Function):
    """Whole-network autograd node: forward = executor.forward, backward = executor.backward."""

    @staticmethod
    def forward(ctx, x, holder, training, need, masks, chan_keep, *params):
        ex = holder.executor
        outs, slot = ex.forward(x, training, need, masks, chan_keep)
        ctx.ex, ctx.slot, ctx.nparams = ex, slot, len(params)
        ctx.set_materialize_grads(False)       # an output the loss never touched arrives as None, not as a zero tensor
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        ex = ctx.ex
        gflat = ex.backward(ctx.slot, list(gouts))
        # ONE copy of the flat bucket (the executor reuses it next step); parameters whose sub-network received no gradient
        # (an unused aux decoder / deep-supervision head, Decoder_DS.out_conv_dp4) get None, exactly like autograd on the
        # reference modules -- torch.optim.SGD then skips them instead of applying weight decay and momentum
        flat = gflat.clone()
        live = ex.last_backward_param_ids
        grads, off = [], 0
        for p in ex.params:
            n = p.numel()
            grads.append(flat[off:off + n].view_as(p) if id(p) in live else None)
            off += n
        return (None, None, None, None, None, None) + tuple(grads)


class _Holder:
    def __init__(self, executor):
        self.executor = executor


class _PlannedNet(nn.Module):
    _decoders = ()
    _aux = ()
    _decoder_cls = Decoder

    def _build(self, in_chns, class_num):
        p = _params(in_chns, class_num)
        self.encoder = Encoder(p)
        for name in self._decoders:
            setattr(self, name, self._decoder_cls(p))
        self._holder = None
        self.dropout_masks = None      # {encoder level: uint8 NHWC keep-mask}  (tests / parity runs)
        self.channel_keep = None       # [five [N,C] keep masks]               (tests / parity runs)

    precision = "bf16"     # see set_precision

    def set_precision(self, precision):
        """Execution mode of the fused executor (networks/_engine.py:PRECISIONS):
          'bf16'   default: activations / activation gradients stored in bf16, wgmma convolutions;
          'fp16'   the same kernels on fp16 storage (11-bit mantissa, same speed; gradients carry a power-of-two loss scale);
          'fp16x3' fp32 storage, tensor-core convolutions on fp16 hi/lo split operands: fp32-accurate (the reference computes
                   in fp32, networks/unet.py:18-26), a few times slower than bf16;
          'fp32'   fp32 storage, CUDA-core direct convolutions: the arithmetic cross-check, ~100x slower."""
        from ._engine import PRECISIONS
        assert precision in PRECISIONS, f"precision must be one of {sorted(PRECISIONS)}"
        object.__setattr__(self, "precision", precision)
        object.__setattr__(self, "_holder", None)
        return self

    _runs = None           # decoder passes (decoder index, feature transform) when they differ from one pass per decoder

    @property
    def executor(self):
        if self._holder is None:
            ex = UNetExecutor(self, self.encoder, [getattr(self, n) for n in self._decoders], list(self._aux), self.precision,
                              runs=self._runs)
            object.__setattr__(self, "_holder", _Holder(ex))
        return self._holder.executor

    def _run(self, x):
        self.executor  # build lazily
        params = list(self.parameters())
        need = torch.is_grad_enabled() and any(p.requires_grad for p in params)   # (grad mode is off inside Function.forward)
        return _NetFn.apply(x, self._holder, self.training, need, self.dropout_masks, self.channel_keep, *params)


class UNet(_PlannedNet):
    """reference unet.py:286-303: returns logits [N, class_num, H, W]."""
    _decoders = ("decoder",)
    _aux = (False,)

    def __init__(self, in_chns, class_num):
        super().__init__()
        self._build(in_chns, class_num)

    def forward(self, x):
        return self._run(x)[0]


class UNet_CCT(_PlannedNet):
    """reference unet.py:327-346: returns (main_seg, aux_seg1); the aux decoder always sees
    F.dropout2d(feature, 0.5) (active in eval too, SURVEY F5)."""
    _decoders = ("main_decoder", "aux_decoder1")
    _aux = (False, True)

    def __init__(self, in_chns, class_num):
        super().__init__()
        self._build(in_chns, class_num)

    def forward(self, x):
        main_seg, aux_seg1 = self._run(x)
        return main_seg, aux_seg1


# ---- API-surface names of the reference module that are off the north-star path --------------------------
def Dropout(x, p=0.5):
    """reference unet.py:254-256 (functional channel dropout, always in training mode)."""
    return torch.nn.functional.dropout2d(x, p)


def FeatureDropout(x):
    """reference unet.py:259-268."""
    attention = torch.mean(x, dim=1, keepdim=True)
    max_val, _ = torch.max(attention.view(x.size(0), -1), dim=1, keepdim=True)
    threshold = (max_val * np.random.uniform(0.7, 0.9)).view(x.size(0), 1, 1, 1).expand_as(attention)
    return x.mul((attention < threshold).float())


class FeatureNoise(nn.Module):
    """reference unet.py:271-283."""

    def __init__(self, uniform_range=0.3):
        super().__init__()
        self.uni_dist = Uniform(-uniform_range, uniform_range)

    def forward(self, x):
        noise = self.uni_dist.sample(x.shape[1:]).to(x.device).unsqueeze(0)
        return x.mul(noise) + x


class _OffPath(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError(f"{type(self).__name__} is outside the accelerated hot path (SURVEY 8(f) rank 4)")


class Decoder_DS(Decoder):
    """reference unet.py:138-190: the Decoder plus 3x3 class heads on the outputs of up1 / up2 / up3 (out_conv_dp3 / dp2 / dp1),
    each resized to the input size by nearest interpolation.  ``out_conv_dp4`` is registered (state_dict parity) and, as in
    the reference, never used."""

    def __init__(self, params):
        super().__init__(params)
        f = self.ft_chns
        for lvl in (4, 3, 2, 1):
            setattr(self, f"out_conv_dp{lvl}", nn.Conv2d(f[lvl], self.n_class, kernel_size=3, padding=1))


class Decoder_URDS(Decoder_DS):
    """reference unet.py:191-251: Decoder_DS's layers plus a FeatureNoise module; its forward perturbs the inputs of the three
    deep-supervision heads in training mode.  No network class of the reference instantiates it (grep: only its definition), so it
    is kept as a constructible parameter container with the reference's state_dict layout."""

    def __init__(self, params):
        super().__init__(params)
        self.feature_noise = FeatureNoise()


class UNet_DS(_PlannedNet):
    """reference unet.py:306-324: forward returns (dp0, dp1, dp2, dp3), all at the input resolution."""
    _decoders = ("decoder",)
    _aux = (False,)
    _decoder_cls = Decoder_DS

    def __init__(self, in_chns, class_num):
        super().__init__()
        self._build(in_chns, class_num)

    def forward(self, x):
        return self._run(x)


class UNet_CCT_3H(_PlannedNet):
    """reference unet.py:349-371, as written: returns (main_seg, aux_seg1, aux_seg2) where aux_seg1 = aux_decoder1 on
    F.dropout2d'ed features and aux_seg2 = aux_decoder1 AGAIN on FeatureNoise'd features (:369-370); ``aux_decoder2`` owns
    parameters (state_dict parity) and never runs, so its parameters get no gradient.  ``feature_noise`` (tests) injects the five
    [C, H, W] noise tensors the reference draws from torch's RNG."""
    _decoders = ("main_decoder", "aux_decoder1", "aux_decoder2")
    _aux = (False, True, True)
    _runs = ((0, None), (1, "chan_drop"), (1, "feat_noise"))

    def __init__(self, in_chns, class_num):
        super().__init__()
        self._build(in_chns, class_num)
        self.feature_noise = None

    def forward(self, x):
        main_seg, aux_seg1, aux_seg2 = self._run(x)
        return main_seg, aux_seg1, aux_seg2
