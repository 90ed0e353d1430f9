"""CPU restatement of FCDiscriminator (networks/discriminator.py:58-101) for the tests of the tensor-core discriminator.

  forward          conv0(map) + conv1(feature) -> conv2 -> LeakyReLU(0.2) -> Dropout2d -> conv3 -> LeakyReLU -> Dropout2d -> conv4 ->
                   LeakyReLU -> AvgPool2d(7) -> flatten -> Linear(ndf*32, 2), functional, in the dtype of the inputs (fp32 / fp64);
                   quant=torch.bfloat16 rounds the tensors the bf16 executor stores (inputs, packed weights, conv outputs,
                   activations) to bf16 and leaves the rest in the working dtype; Dropout2d keep masks are injected.
  space-to-depth   the plan of wsl4mis_b200/networks/discriminator.py restated with torch ops: s2d / d2s, the structured 3x3 weight
                   (scatter) and the gather of its gradient, so that a 4x4 / stride-2 / pad-1 convolution, its input gradient and its
                   weight gradient can be checked against F.conv2d(stride=2, padding=1) and fed to the bit-exact tests of the packers.
"""
import numpy as np
import torch
import torch.nn.functional as F

SLOPE = 0.2


def param_shapes(num_classes=4, ndf=64, n_channel=1):
    """ordered {state_dict key: shape} (discriminator.py:62-71 registration order)"""
    out = {}
    for name, cin, cout in (("conv0", num_classes, ndf), ("conv1", n_channel, ndf), ("conv2", ndf, 2 * ndf), ("conv3", 2 * ndf, 4 * ndf),
                            ("conv4", 4 * ndf, 8 * ndf)):
        out[name + ".weight"], out[name + ".bias"] = (cout, cin, 4, 4), (cout,)
    out["classifier.weight"], out["classifier.bias"] = (2, 32 * ndf), (2,)
    return out


def synth_params(seed, num_classes=4, ndf=64, n_channel=1, dtype=torch.float32):
    """seeded uniform weights with He scale (bound sqrt(6 / fan_in)), so that activations keep their magnitude through the five
    layers and the logits are O(1)"""
    rs = np.random.RandomState(seed)
    p = {}
    shapes = param_shapes(num_classes, ndf, n_channel)
    for k, shp in shapes.items():
        fan_in = int(np.prod(shapes[k.replace(".bias", ".weight")][1:]))
        p[k] = torch.from_numpy(rs.uniform(-1.0, 1.0, size=shp) * np.sqrt(6.0 / fan_in)).to(dtype)
    return p


def synth_inputs(seed, n, num_classes=4, n_channel=1, hw=256, dtype=torch.float32):
    """(map, feature): a softmax over smooth random logits (what the DAN script feeds, train_deep_adversarial_network_2D.py:143-153)
    and an image in [0, 1]"""
    rs = np.random.RandomState(seed)
    logits = rs.randn(n, num_classes, hw // 8, hw // 8)
    logits = np.repeat(np.repeat(logits, 8, axis=2), 8, axis=3) + 0.5 * rs.randn(n, num_classes, hw, hw)
    mp = torch.softmax(torch.from_numpy(logits), dim=1)
    feat = torch.from_numpy(rs.rand(n, n_channel, hw, hw))
    return mp.to(dtype), feat.to(dtype)


def chan_keep(seed, n, ndf=64):
    """the two Dropout2d keep masks [n, 2ndf], [n, 4ndf] (uint8)"""
    rs = np.random.RandomState(seed)
    return [torch.from_numpy((rs.rand(n, c) >= 0.5).astype(np.uint8)) for c in (2 * ndf, 4 * ndf)]


class _Round(torch.autograd.Function):
    """storage rounding in the forward, identity in the backward"""

    @staticmethod
    def forward(ctx, x, dt):
        return x.to(dt).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g, None


def _q(x, quant):
    return x if quant is None else _Round.apply(x, quant)


def forward(p, mp, feat, training, keep=None, quant=None):
    """FCDiscriminator.forward (discriminator.py:79-101) -> [N, 2] logits.  keep: the two uint8 [N, C] masks (train mode)."""
    w = {k: (_q(v, quant) if k.endswith(".weight") and not k.startswith("classifier") else v) for k, v in p.items()}
    conv = lambda x, name: F.conv2d(x, w[name + ".weight"], w[name + ".bias"], stride=2, padding=1)
    x = _q(conv(_q(mp, quant), "conv0") + conv(_q(feat, quant), "conv1"), quant)
    for i, name in enumerate(("conv2", "conv3")):
        x = _q(conv(x, name), quant)
        x = F.leaky_relu(x, SLOPE)
        if training:
            x = x * (keep[i].to(x.dtype) * 2.0)[:, :, None, None]
        x = _q(x, quant)
    x = _q(conv(x, "conv4"), quant)
    x = F.avg_pool2d(F.leaky_relu(x, SLOPE), 7)
    return F.linear(x.reshape(x.shape[0], -1), p["classifier.weight"], p["classifier.bias"])


# ---- the space-to-depth plan ----------------------------------------------------------------------------------------------------
def s2d(x, CP=None):
    """NCHW x -> NHWC T [N, H/2, W/2, CP] with T[n, Y, X, (a*2+b)*C + c] = x[n, c, 2Y+a, 2X+b]; channels above 4C zero"""
    N, C, H, W = x.shape
    t = x.reshape(N, C, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(N, H // 2, W // 2, 4 * C)
    CP = 4 * C if CP is None else CP
    return F.pad(t, (0, CP - 4 * C))


def d2s(t, C):
    """transpose of s2d: NHWC [N, h, w, >= 4C] -> NCHW [N, C, 2h, 2w]"""
    N, h, w, _ = t.shape
    return t[..., :4 * C].reshape(N, h, w, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(N, C, 2 * h, 2 * w)


def scatter(w4, CP=None):
    """4x4 weight [Cout, C, 4, 4] -> structured 3x3 weight [Cout, CP, 3, 3]: tap k of an axis at 3x3 tap (k+1)>>1, phase (k+1)&1"""
    Cout, C = w4.shape[:2]
    CP = 4 * C if CP is None else CP
    w3 = w4.new_zeros(Cout, CP, 3, 3)
    for ky in range(4):
        for kx in range(4):
            q = ((ky + 1) & 1) * 2 + ((kx + 1) & 1)
            w3[:, q * C:(q + 1) * C, (ky + 1) >> 1, (kx + 1) >> 1] = w4[:, :, ky, kx]
    return w3


def gather(dw3, C):
    """the 16 used slots of a structured 3x3 weight (gradient) [Cout, CP, 3, 3] -> [Cout, C, 4, 4]"""
    out = dw3.new_zeros(dw3.shape[0], C, 4, 4)
    for ky in range(4):
        for kx in range(4):
            q = ((ky + 1) & 1) * 2 + ((kx + 1) & 1)
            out[:, :, ky, kx] = dw3[:, q * C:(q + 1) * C, (ky + 1) >> 1, (kx + 1) >> 1]
    return out


def s2d_conv(x, w4, b=None):
    """4x4 / stride-2 / pad-1 convolution of NCHW x as the 3x3 / pad-1 convolution of s2d(x) -> NCHW"""
    t = s2d(x).permute(0, 3, 1, 2)
    return F.conv2d(t, scatter(w4), b, padding=1)


def s2d_conv_input_grad(dy, w4, C):
    """d x of s2d_conv: the 3x3 data gradient (flipped, transposed weight, pad 1) gives dT; depth-to-space of dT is dx"""
    w3 = scatter(w4)
    dt = F.conv2d(dy, w3.flip(2, 3).transpose(0, 1), padding=1)
    return d2s(dt.permute(0, 2, 3, 1), C)


def s2d_conv_weight_grad(x, dy):
    """d w4 of s2d_conv: the 3x3 weight gradient over (T, dY), gathered"""
    t = s2d(x).permute(0, 3, 1, 2)
    dw3 = torch.nn.grad.conv2d_weight(t, (dy.shape[1], t.shape[1], 3, 3), dy, padding=1)
    return gather(dw3, x.shape[1])
