"""Per-element error bounds for the tensor-core convolutions and a localiser that names the work item and the CTA that wrote a
violating output.  Pure torch, so the GPU scale test and its CPU self-test (tests/test_conv_check_cpu.py) share one checker.

Outputs.  With S = conv(|x|, |w|) + |b| evaluated by the same fp64 reference, an output passes when
    |got - ref| <= u * |ref| + slack * S
u is the unit roundoff of the stored type (2^-8 bf16, 2^-11 fp16, 0 for fp32 outputs) and covers the final rounding; slack * S
(2^-16 for 16-bit operands, 2^-20 .. 2^-17 by accumulation depth for the fp16 hi/lo split path, see split_slack) covers
fp32 accumulation noise.  A missing tap, k-block or
tile is about S / (taps * k-blocks), far above the slack, and the bound is per element, so one wrong 8 x 16 tile cannot hide
under the tensor's maximum.  NaN (an output never written) always fails.

Weight gradients.  rel-L2 against fp64 <= 1e-4, per (output-channel block, input-channel block), i.e. per output tile of the
split-K kernels: leaving out one 128-pixel chunk of P pixels moves a tile by about sqrt(128 / P)."""
import math

import torch
import torch.nn.functional as F

SLACK_16 = 2.0 ** -16       # 16-bit operands, fp32 accumulation
UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}
WGRAD_TOL = 1e-4
CHUNK_PX = 128              # pixels per split-K chunk of every weight-gradient kernel (16 x 8 or 8 x 16)


def split_slack(K):
    """Accumulation allowance (times S) of the fp16 hi/lo split path with K = taps * Cin.  Its planes carry 22 significant bits
    (representation error ~2^-22 S), but each output sums 3K exact products in fp32 on the tensor cores, and that zero-mean
    rounding noise grows as sqrt(3K) fp32 ulps: on an H100 the worst output of a launch was 0.56 .. 1.2 x sqrt(3K) 2^-24 S for
    K = 64 .. 2304, i.e. above 2^-20 S from K ~ 300 on, against 0.3 x 2^-20 S for the planes' own representation error.
    The allowance is 2.5 sqrt(3K) 2^-24, and never below 2^-20.  A dropped hi x hi k-block is ~S / (K / 16), orders of magnitude
    above it; a dropped lo plane is ~2^-12 S / sqrt(K) typically and several times that at the worst output of a tile."""
    return max(2.0 ** -20, 2.5 * math.sqrt(3 * K) * 2.0 ** -24)


def reference(x, w, b, dil=1):
    """fp64 NCHW convolution (padding = dil * (k // 2)) and its magnitude S = conv(|x|, |w|) + |b|."""
    pad = dil * (w.shape[-1] // 2)
    ref = F.conv2d(x, w, b, padding=pad, dilation=dil)
    S = F.conv2d(x.abs(), w.abs(), b.abs() if b is not None else None, padding=pad, dilation=dil)
    return ref, S


def wgrad_reference(x, dy, ks, dil=1):
    """fp64 weight gradient sum_pixels dY^T X of an NCHW pair: [Cout, Cin, ks, ks]."""
    return torch.nn.grad.conv2d_weight(x, (dy.shape[1], x.shape[1], ks, ks), dy, padding=dil * (ks // 2), dilation=dil)


def chunks_missing_margin(P):
    """relative change of a weight gradient over P pixels when one 128-pixel chunk is left out (or counted twice)"""
    return math.sqrt(CHUNK_PX / P)


class Tiling:
    """Which work item wrote output (n, y, x, c).  Pixel tiles of th x tw are numbered image by image; order 'yx' numbers an
    image's tiles row by row (conv_tc, conv_tc2), 'xy' column strip by column strip (conv_row: item = (n, strip, row segment)).
    Output channel c belongs to the N tile c // nt (blockIdx.y).  A persistent kernel with `grid` CTAs along x gives tile t to
    CTA t % grid; grid None means one CTA per tile."""

    def __init__(self, H, W, th, tw, nt, grid=None, order="yx"):
        assert H % th == 0 and W % tw == 0 and order in ("yx", "xy")
        self.H, self.W, self.th, self.tw, self.nt, self.grid, self.order = H, W, th, tw, nt, grid, order

    @property
    def tiles_per_image(self):
        return (self.H // self.th) * (self.W // self.tw)

    def tile(self, n, y, x):
        ty, tx = self.H // self.th, self.W // self.tw
        if self.order == "yx":
            return (n * ty + y // self.th) * tx + x // self.tw
        return (n * tx + x // self.tw) * ty + y // self.th

    def owner(self, n, y, x, c):
        """-> (tile, N tile, CTA x index)"""
        t = self.tile(n, y, x)
        return t, c // self.nt, (t % self.grid if self.grid else t)


def check_output(got, ref, S, u, slack, tiling=None, n0=0, max_listed=1 << 20):
    """got / ref / S: NCHW tensors of images n0 .. n0 + len.  Returns {'worst': max error / bound, 'bad': count,
    'first': (n, y, x, c) of the first violation in NHWC order or None, 'owner': (tile, N tile, CTA) of it, 'tiles': sorted
    set of (tile, N tile) with a violation (when there are at most max_listed violations)}."""
    err = (got.double() - ref).abs()
    bound = u * ref.abs() + slack * S
    ok = err <= bound                                  # NaN compares False: an unwritten output fails
    ratio = torch.where(err == err, err / bound.clamp_min(1e-300), torch.full_like(err, math.inf))
    rep = {"worst": ratio.max().item(), "bad": int((~ok).sum().item()), "first": None, "owner": None, "tiles": None}
    if rep["bad"]:
        bad = (~ok).permute(0, 2, 3, 1)
        i = int(bad.reshape(-1).to(torch.uint8).argmax().item())
        _, H, W, C = bad.shape
        n, rem = divmod(i, H * W * C)
        y, rem = divmod(rem, W * C)
        x, c = divmod(rem, C)
        rep["first"] = (n + n0, y, x, c)
        if tiling is not None:
            rep["owner"] = tiling.owner(n + n0, y, x, c)
            if rep["bad"] <= max_listed:
                nz = bad.nonzero()
                t = tiling.tile(nz[:, 0] + n0, nz[:, 1], nz[:, 2])
                rep["tiles"] = sorted(set(zip(t.tolist(), (nz[:, 3] // tiling.nt).tolist())))
    return rep


def merge(reports):
    """combine the reports of consecutive image chunks (in image order)"""
    out = {"worst": 0.0, "bad": 0, "first": None, "owner": None, "tiles": []}
    for r in reports:
        out["worst"] = max(out["worst"], r["worst"])
        out["bad"] += r["bad"]
        if out["first"] is None and r["first"] is not None:
            out["first"], out["owner"] = r["first"], r["owner"]
        if r["bad"]:
            out["tiles"] = None if (r["tiles"] is None or out["tiles"] is None) else out["tiles"] + r["tiles"]
    return out


def describe(rep):
    if not rep["bad"]:
        return f"ok (worst error / bound {rep['worst']:.3g})"
    s = f"{rep['bad']} outputs over the bound (worst {rep['worst']:.3g} x); first at (n, y, x, c) = {rep['first']}"
    if rep["owner"] is not None:
        t, nb, cta = rep["owner"]
        s += f", pixel tile {t}, N tile {nb}, CTA {cta}"
    return s


def check_wgrad(got, ref, co_blk, ci_blk, tol=WGRAD_TOL):
    """dw [Cout, Cin, k, k] against fp64, rel-L2 per (co_blk x ci_blk) block.  Returns {'worst': max rel-L2 / tol,
    'bad': [(co block, ci block, rel-L2), ...] over tol, 'rel': rel-L2 of the whole tensor}."""
    got, ref = got.double(), ref.double()
    Cout, Cin = ref.shape[:2]
    worst, bad = 0.0, []
    for cb in range(0, Cout, co_blk):
        for ib in range(0, Cin, ci_blk):
            r = ref[cb:cb + co_blk, ib:ib + ci_blk]
            d = got[cb:cb + co_blk, ib:ib + ci_blk] - r
            e = (d.norm() / r.norm().clamp_min(1e-300)).item()
            if not e <= tol:
                bad.append((cb // co_blk, ib // ci_blk, e))
            worst = max(worst, e / tol if e == e else math.inf)
    rel = ((got - ref).norm() / ref.norm().clamp_min(1e-300)).item()
    return {"worst": worst, "bad": bad, "rel": rel}
