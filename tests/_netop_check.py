"""Bounds, fp64 references, the counter-RNG restatement and a fault localiser for the non-convolution launches of the network
executor (BatchNorm, activation, pooling, upsample, dropout, layout and packing kernels).  Pure numpy / torch, so the GPU scale test
(tests/test_gpu_netops_at_scale.py) and its CPU self-test (tests/test_netop_check_cpu.py) share one checker.

Storage types: dtype 0 = bf16, 1 = fp32, 2 = fp16.  u_T is the unit roundoff of the stored type (2^-8, 0, 2^-11): a value computed
in fp32 and stored once is within u_T |v| of v.  TINY_T is half the smallest subnormal spacing of the stored type (only fp16's,
2^-25, is ever reached: LeakyReLU outputs slope * z of small z underflow there).

Bit-exact.  Dropout keep bits (wsl_rand8x16: two splitmix64 rounds of seed + vec * 0x9E3779B97F4A7C15 give eight 16-bit draws of
the 8-channel vector vec = p * (C / 8) + g, element j is kept when r_j >= (uint32)(float32(p) * 65536.0f)); wsl_uniform (the
murmur3 fmix64 finaliser of seed * 0x9E3779B97F4A7C15 + i, top 24 bits of the low word, times 2^-24); max-pool values and the
index of the first maximum in scan order over the activations as stored; every kernel whose result is one fp32 expression
rounded once to the storage type.

One rounding (activations).  act = dropout(leaky(fmaf(y, scale, shift))) makes at most three fp32 roundings before the store
(fmaf, * slope, * 1/(1-p)); with the reference evaluated in fp64 at the kernel's own fp32 scale / shift / slope / 1/(1-p),
    |got - ref| <= (u_T + 2^-22) |ref| + TINY_T,          2^-22 = 4 * 2^-24 > 3 roundings (+ u_T * 3 * 2^-24 < 2^-24).

Sums.  A per-channel (or per-pixel) sum formed in fp32 partials and fp64 totals passes when |got - ref| <= STAT_TOL * sum |terms|;
STAT_TOL = 1e-5 covers fp32 partial sums of up to ~160 terms in the worst case (160 * 2^-24) and far longer ones on average,
while a missing 8-channel group, image or block partial moves a sum by about 1 / (number of partials) of sum |terms|.
Mean and invstd: |mean - ref| <= 1e-5 rms and |invstd * sqrt(var + eps) - 1| <= 1e-4 (the bounds wsl_bn_finalize is held to
by the convolution scale test).

BatchNorm backward dY = sc * (dz - c1 - xhat * c2), c1 = sum dz / P, c2 = sum dz * xhat / P (P global), per element:
    |got - ref| <= u_T |ref| + |sc| (dc1 + |xhat| dc2) + 2^-22 |sc| (|dz| + |c1| + (|xhat| + 2 |mean| invstd) |c2|) + TINY_T
dc1, dc2 = STAT_TOL * sum |dz| / P and STAT_TOL * sum |dz xhat| / P carry the sum tolerance into the coefficients; the 2^-22 term
covers the fp32 evaluation dz * sc + (y * B + D) with B = -sc c2 invstd and D = -sc c1 + sc c2 mean invstd rounded to fp32 (each
off by 2^-24 of |sc c2| (|xhat| + |mean| invstd) and |sc| (|c1| + |c2 mean| invstd)) and the fp32 gradient sum behind dz (|dz|
is taken over the magnitudes of the summed sources)."""
import math

import numpy as np
import torch

STAT_TOL = 1e-5
U = {0: 2.0 ** -8, 1: 0.0, 2: 2.0 ** -11}
TINY = {0: 0.0, 1: 0.0, 2: 2.0 ** -25}
ACT_REL = 2.0 ** -22
TORCH_T = {0: torch.bfloat16, 1: torch.float32, 2: torch.float16}
GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


# ---------------------------------------------------------------------------------------------------------------- counter RNG
def splitmix64_int(z):
    """pure-Python big-int wsl_splitmix64"""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def splitmix64(z):
    """vectorised wsl_splitmix64 on numpy uint64 (multiplication wraps mod 2^64 as on the device)"""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def rand8x16(seed, vec):
    """wsl_rand8x16: uint32 [len(vec), 8] random 16-bit draws of the 8-element vectors `vec` (uint32 indices)"""
    vec = np.asarray(vec, dtype=np.uint64)
    with np.errstate(over="ignore"):
        a = splitmix64(np.uint64(seed & M64) + vec * np.uint64(GOLDEN))
        b = splitmix64(a + np.uint64(0xD1B54A32D192ED03))
    out = np.empty((vec.size, 8), dtype=np.uint32)
    for j in range(4):
        out[:, j] = ((a >> np.uint64(16 * j)) & np.uint64(0xFFFF)).astype(np.uint32)
        out[:, 4 + j] = ((b >> np.uint64(16 * j)) & np.uint64(0xFFFF)).astype(np.uint32)
    return out


def drop_threshold(p):
    """(uint32)(p * 65536.0f), the product formed in fp32"""
    return int(np.float32(p) * np.float32(65536.0))


def inv_keep(p):
    """1.f / (1.f - p) in fp32, as make_drop forms it"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


def keep_mask(seed, P, C, p, vec_offset=0):
    """bool [P, C]: the dropout keep decisions of bn_act_fwd / bn_bwd for a [P][C] channels-last tensor (vector index
    p * (C / 8) + g, 32-bit, as the kernels form it)"""
    if p <= 0:
        return np.ones((P, C), dtype=bool)
    cg = C // 8
    vec = (np.arange(P * cg, dtype=np.uint64) + np.uint64(vec_offset)) & np.uint64(0xFFFFFFFF)
    return (rand8x16(seed, vec) >= drop_threshold(p)).reshape(P, C)


def hash32(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xFF51AFD7ED558CCD)
        x = x ^ (x >> np.uint64(33))
        x = x * np.uint64(0xC4CEB9FE1A85EC53)
        x = x ^ (x >> np.uint64(33))
    return (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def uniform(seed, n):
    """wsl_uniform(seed, i) for i < n: float32, multiples of 2^-24 in [0, 1)"""
    with np.errstate(over="ignore"):
        base = np.uint64(seed & M64) * np.uint64(GOLDEN)
        h = hash32(base + np.arange(n, dtype=np.uint64))
    return (h >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


# ---------------------------------------------------------------------------------------------------------------- localiser
class Layout:
    """Which CTA of a grid-stride kernel owns (pixel p, channel c) of a [P][C] channels-last tensor.
    'rows': a thread owns one 8-channel group and walks pixels p = block * rows + r + k * grid * rows, rows = 256 / (C / 8)
    (BatchNorm statistics / apply / backward, bn_act_fwd); 'vec': thread i of the grid walks 8-element vectors i + k * grid * 256
    with vector index p * (C / 8) + g (elementwise kernels); 'pool': like 'rows' over the pooled pixels q."""

    def __init__(self, kind, C, grid, HW=None, W=None):
        self.kind, self.C, self.grid, self.HW, self.W = kind, C, grid, HW, W

    def block(self, p, c):
        cg = self.C // 8
        if self.kind == "rows":
            return (p // (256 // cg)) % self.grid
        if self.kind == "pool":
            n, rem = divmod(p, self.HW)
            y, x = divmod(rem, self.W)
            q = (n * (self.HW // self.W // 2) + y // 2) * (self.W // 2) + x // 2
            return (q // (256 // cg)) % self.grid
        return ((p * cg + c // 8) // 256) % self.grid


def locate(bad, shape):
    """bad: bool tensor [P, C]; shape (N, H, W) -> (n, y, x, c) of the first violation in NHWC order, or None"""
    flat = bad.reshape(-1)
    if not bool(flat.any()):
        return None
    i = int(flat.to(torch.uint8).argmax().item())
    C = bad.shape[-1]
    p, c = divmod(i, C)
    N, H, W = shape
    n, rem = divmod(p, H * W)
    y, x = divmod(rem, W)
    return (n, y, x, c), p


def report(got, ref, bound, shape=None, layout=None, what="value"):
    """Element-wise |got - ref| <= bound over [P, C] tensors (NaN fails).  -> {'worst', 'bad', 'msg'}"""
    err = (got.double() - ref.double()).abs()
    ok = err <= bound
    ratio = torch.where(err == err, err / bound.clamp_min(1e-300), torch.full_like(err, math.inf))
    worst = ratio.max().item() if ratio.numel() else 0.0
    nbad = int((~ok).sum().item())
    rep = {"worst": worst, "bad": nbad, "msg": None, "first": None, "p": None}
    if nbad:
        msg = f"{what}: {nbad} elements over the bound (worst {worst:.3g} x)"
        if shape is not None:
            (n, y, x, c), p = locate((~ok).reshape(-1, ref.shape[-1]), shape)
            rep["first"], rep["p"] = (n, y, x, c), p
            msg += f"; first at (n, y, x, c) = ({n}, {y}, {x}, {c}), 8-channel group {c // 8}"
            if layout is not None:
                msg += f", block {layout.block(p, c)}"
            msg += f": got {got.reshape(-1, ref.shape[-1])[p, c].item():.6g}, expected {ref.reshape(-1, ref.shape[-1])[p, c].item():.6g}"
        rep["msg"] = msg
    return rep


def exact(got, ref, shape=None, layout=None, what="value"):
    """bit-exact comparison of two tensors of the same dtype (reported like report())"""
    if got.dtype in (torch.bfloat16, torch.float16):
        a, b = got.view(torch.int16), ref.view(torch.int16)
    elif got.dtype == torch.float32:
        a, b = got.view(torch.int32), ref.view(torch.int32)
    else:
        a, b = got, ref
    bad = a != b
    nbad = int(bad.sum().item())
    rep = {"worst": 0.0 if nbad == 0 else math.inf, "bad": nbad, "msg": None, "first": None, "p": None}
    if nbad:
        msg = f"{what}: {nbad} elements differ"
        if shape is not None:
            C = ref.shape[-1]
            (n, y, x, c), p = locate(bad.reshape(-1, C), shape)
            rep["first"], rep["p"] = (n, y, x, c), p
            msg += (f"; first at (n, y, x, c) = ({n}, {y}, {x}, {c}), 8-channel group {c // 8}"
                    + (f", block {layout.block(p, c)}" if layout is not None else "")
                    + f": got {got.reshape(-1, C)[p, c].item()}, expected {ref.reshape(-1, C)[p, c].item()}")
        rep["msg"] = msg
    return rep


def sums(got, ref, mag, tol=STAT_TOL, what="sum", extra=None):
    """per-channel (or per-pixel) sums: |got - ref| <= tol * mag (+ extra)"""
    bound = tol * mag.double() + (0.0 if extra is None else extra)
    err = (got.double() - ref.double()).abs()
    ok = err <= bound
    worst = torch.where(err == err, err / bound.clamp_min(1e-300), torch.full_like(err, math.inf)).max().item()
    nbad = int((~ok).sum().item())
    msg = None
    if nbad:
        i = int((~ok).reshape(-1).to(torch.uint8).argmax().item())
        msg = (f"{what}: {nbad} of {ok.numel()} over {tol:g} x sum|terms| (worst {worst:.3g} x); first at index {i} "
               f"(8-channel group {i // 8}): got {got.reshape(-1)[i].item():.8g}, expected {ref.reshape(-1)[i].item():.8g}")
    return {"worst": worst, "bad": nbad, "msg": msg}


# ---------------------------------------------------------------------------------------------------------------- references
def stats_ref(y2d):
    """fp64 per-channel {sum, sum |y|, sum y^2} of a [P, C] tensor"""
    y = y2d.double()
    return y.sum(0), y.abs().sum(0), (y * y).sum(0)


def check_mean_invstd(mean_got, invstd_got, s, sq, P, eps):
    """mean / invstd of wsl_bn_stats / wsl_bn_finalize against the fp64 sums s, sq of P values"""
    mean = s / P
    var = (sq / P - mean * mean).clamp_min(0)
    rms = (sq / P).sqrt().clamp_min(1e-300)
    e_mean = ((mean_got.double() - mean).abs() / rms)
    e_inv = (invstd_got.double() * (var + eps).sqrt() - 1).abs()
    worst = max((e_mean / 1e-5).max().item(), (e_inv / 1e-4).max().item())
    msg = None
    if not worst <= 1.0:
        c = int(torch.maximum(e_mean / 1e-5, e_inv / 1e-4).argmax().item())
        msg = (f"mean / invstd: channel {c} (group {c // 8}) mean off by {e_mean[c].item():.2e} of rms, invstd by "
               f"{e_inv[c].item():.2e} relative")
    return {"worst": worst, "bad": 0 if msg is None else 1, "msg": msg}, mean, var


def act_ref(y2d, sc, sh, slope, keep, p):
    """fp64 dropout(leaky(y * sc + sh)) at the kernel's fp32 sc / sh ([C] or per-row [P, C])"""
    z = y2d.double() * sc.double() + sh.double()
    a = torch.where(z > 0, z, z * float(np.float32(slope)))
    return torch.where(keep, a * inv_keep(p), torch.zeros_like(a))


def act_bound(ref, dt):
    return (U[dt] + ACT_REL) * ref.abs() + TINY[dt]


def pool_ref(act):
    """act: [N, H, W, C] as stored -> (pooled [N, H/2, W/2, C] in act's dtype, idx uint8 = first maximum in scan order
    (dy, dx) = (0,0), (0,1), (1,0), (1,1), number of windows whose maximum is tied)"""
    N, H, W, C = act.shape
    v = act.reshape(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(N, H // 2, W // 2, C, 4).float()
    best, idx = v[..., 0], torch.zeros(v.shape[:-1], dtype=torch.uint8, device=act.device)
    for k in range(1, 4):
        gt = v[..., k] > best
        best = torch.where(gt, v[..., k], best)
        idx = torch.where(gt, torch.full_like(idx, k), idx)
    ties = int(((v == best.unsqueeze(-1)).sum(-1) >= 2).sum().item())
    return best.to(act.dtype), idx, ties


def route_pool(gp, idx, H, W):
    """[N, H/2, W/2, C] pooled gradient routed to the window element named by idx -> [N, H, W, C] (fp64)"""
    N, Hp, Wp, C = gp.shape
    out = torch.zeros(N, Hp, 2, Wp, 2, C, dtype=torch.float64, device=gp.device)
    g = gp.double()
    for k in range(4):
        out[:, :, k >> 1, :, k & 1, :] = torch.where(idx == k, g, torch.zeros_like(g))
    return out.reshape(N, H, W, C)


def bn_bwd_ref(y2d, sc, sh, mean, invstd, dA, dA_abs, keep, p, slope, P):
    """fp64 BatchNorm + LeakyReLU + dropout backward at the kernel's fp32 save / ss.  dA / dA_abs: summed incoming gradient and
    the sum of its sources' magnitudes, [P, C].  -> dict of dz, |dz|, xhat, dbeta, dgamma, their magnitudes, dY and its bound
    without the u_T term (see dy_bound)."""
    y = y2d.double()
    z = y * sc.double() + sh.double()
    f = torch.where(z > 0, torch.ones_like(z), torch.full_like(z, float(np.float32(slope))))
    f = torch.where(keep, f * inv_keep(p), torch.zeros_like(f))
    dz, dz_abs = dA * f, dA_abs * f.abs()
    xhat = (y - mean.double()) * invstd.double()
    return {"dz": dz, "dz_abs": dz_abs, "xhat": xhat, "dbeta": dz.sum(0), "dbeta_mag": dz_abs.sum(0),
            "dgamma": (dz * xhat).sum(0), "dgamma_mag": (dz_abs * xhat.abs()).sum(0)}


def dy_ref(r, sc, mean, invstd, P, dt):
    """dY reference and bound for the statistics r (possibly summed over ranks) of bn_bwd_ref, P the global pixel count"""
    sc = sc.double()
    c1, c2 = r["dbeta"] / P, r["dgamma"] / P
    d1, d2 = STAT_TOL * r["dbeta_mag"] / P, STAT_TOL * r["dgamma_mag"] / P
    ref = sc * (r["dz"] - c1 - r["xhat"] * c2)
    off = 2 * mean.double().abs() * invstd.double()
    bound = (U[dt] * ref.abs() + sc.abs() * (d1 + r["xhat"].abs() * d2)
             + ACT_REL * sc.abs() * (r["dz_abs"] + c1.abs() + (r["xhat"].abs() + off) * c2.abs()) + TINY[dt])
    return ref, bound
