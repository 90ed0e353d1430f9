"""fp64 references, bounds and kernel-arithmetic emulations for the loss-head launches of the training steps (wsl4mis_b200/csrc/
losses.cu).  Pure numpy / torch, so the GPU scale test (tests/test_gpu_losses_at_scale.py) and its CPU self-test
(tests/test_loss_check_cpu.py) share one checker.

References.  Every reference is the reference's own formula from oracle/wsl_oracle.py, semi_oracle.py and s2l_oracle.py (pinned to
the reference by tests/test_oracle_golden.py) evaluated in fp64, and every reference gradient is torch autograd of that formula.
Each consumer is evaluated at the kernel's own fp32 operands: a backward that reads `probs` is differentiated at the logits
L = log(probs), whose softmax is probs (to the 2^-22 by which fp32 probabilities miss a unit sum), with the label count, centroids
or Dice sums the forward kernel wrote.  A loss that is a sum over samples is evaluated one sample (or a few) at a time.

Storage types: dtype 0 = bf16, 1 = fp32, 2 = fp16; u_T and STAT_TOL are _netop_check's (u_T = 2^-8, 0, 2^-11; STAT_TOL = 1e-5).

One rounding.  Probabilities: expf, the sum and the product with 1/s make a few fp32 roundings, and x - max is rounded before
expf, so |got - ref| <= (2^-21 + 2^-23 |x - max|) |ref| + 2^-126 (2^-126 also floors every gradient bound: fp32 subnormals).  rot90 (a permutation, plus one fp32 add with accumulate = 1): bit-exact, resp. 2^-24 |ref|.  The 16-bit channels-last
logit gradient (NHWC16) is the fp32 gradient (within 2^-20 mag of the reference, mag the magnitude of the terms of the fp32
expression) rounded once: |got - ref| <= u_T |ref| + 2^-19 mag + TINY_T, 2^-19 >= (1 + u_T) 2^-20; its channels 4..15 must be exactly zero and no element may be +-inf.  With the fp32 output
written in the same launch the 16-bit one must equal it rounded to nearest, bit for bit.

Sums and loss scalars.  |got - ref| <= STAT_TOL * sum |terms| / normaliser (fp32 per-thread and per-block partials, fp64 totals).
A lost block partial moves a sum by about 1 / (number of blocks) of sum |terms|, far more than STAT_TOL for the grids used here.

Gated CRF gradient, per pixel i and class:  |got - ref| <= 2^-16 |gscale| sum_j k_ij |y_j|.  The kernel forms s_i = sum_j k_ij y_j
with 120 fp32 FMAs (at most 120 * 2^-24 < 2^-17 of sum_j k_ij |y_j|) over k_ij from ex2.approx (2^-22 relative) of an fp32
exponent, and sigma_rgb = 0.1 rounded to fp32 moves an exponent of up to -50 by 1.5e-6 (k by the same relative amount, and only
where k < e^-5 of its centre weight); 2^-16 covers all of it.  Dropping the outermost window tap (|dxy|^2 = 50) removes a term of
exp(-50 / 72) ~ 0.5 of a centre-weight term from a sum of ~ 120 such terms in a flat region: about 4e-3 relative, 250 times the
bound.  A halo row read from the wrong tile changes five of the eleven rows of the window.

Labels and masks, bit-exact: mix_argmax (the first maximum wins on exact ties; the mix in fp32 with two products and one add, as
torch computes beta * p1 + (1 - beta) * p2); the S2L u-labels (the last class whose weight is > thr_conf wins, strictly greater);
the UAMT uncertainty mask except where the fp64 uncertainty lies within UNC_BAND (1 + sum_c |q_c log(q_c + 1e-6)|) of the
threshold (the fp32 evaluation of softmax, mean and logf is within that of fp64); TV's routing of +-gscale to the first extremum
in scan order, which the atomics add up to |got - ref| <= 2^-22 |ref| + 2^-14 |gscale|.

Edge behaviour is asserted as such: the class-variance backward gives no intra-class term where a class's std is 0 (torch.std's
backward gives 0 there as well, so the two are compared directly), and pCE / S2L return NaN when no pixel qualifies, with a zero
gradient from that term.

The UAMT Monte-Carlo buffer's row of pass t of sample b is (t >> 1) * 2B + (t & 1) * B + b (T / 2 calls on the twice-repeated
batch), which equals t * B + b, the oracle's reshape(T, B, ...); a sample-major layout b * T + t is the mistake to catch."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import _netop_check as K
import s2l_oracle as SO
import wsl_oracle as O

STAT_TOL, U, TINY = K.STAT_TOL, K.U, K.TINY
TORCH_T = K.TORCH_T
P_REL = 2.0 ** -21
CRF_REL = 2.0 ** -16
UNC_BAND = 2.0 ** -18
FP32_MIN = 2.0 ** -126
report, exact, sums, uniform = K.report, K.exact, K.sums, K.uniform


def scalar(got, ref, mag, what, tol=STAT_TOL):
    """one loss scalar (or a vector of them): |got - ref| <= tol * mag"""
    t = lambda v: torch.as_tensor(v, dtype=torch.float64).reshape(-1).cpu()
    return K.sums(t(got), t(ref), t(mag), tol, what)


def chunks(n, size):
    return [(i, min(n, i + size)) for i in range(0, n, size)]


def logits_of(p):
    """fp64 logits whose softmax is p (a zero probability becomes 1e-300, which is zero to fp64 precision)"""
    return p.double().clamp_min(1e-300).log()


# ---------------------------------------------------------------------------------------------------------------- softmax + pCE
def probs_ref(logits):
    return torch.softmax(logits.double(), 1)


def softmax_rel(logits):
    """relative error of an fp32 softmax: a few roundings (2^-21) plus the rounding of x - max, which expf turns into a relative
    error of 2^-24 |x - max| (2^-23 here)"""
    x = logits.double()
    return P_REL + 2.0 ** -23 * (x.max(1, keepdim=True).values - x)


def probs_bound(ref, logits):
    return softmax_rel(logits) * ref.abs() + FP32_MIN


def labelled(label, ignore):
    lab = label.long()
    return (lab != ignore) & (lab < 4)


def pce_ref(logits, label, ignore, per=8):
    """-> (pCE mean = wsl_oracle.pce_loss in fp64, labelled count, sum over the labelled pixels of |log s| + |x_l - m|)"""
    tot, cnt, mag = 0.0, 0, 0.0
    for a, b in chunks(logits.shape[0], per):
        x, lab = logits[a:b].double(), label[a:b].long()
        on = labelled(lab, ignore)
        n = int(on.sum())
        if n:
            tot += O.pce_loss(x, torch.where(on, lab, torch.full_like(lab, ignore)), ignore).item() * n
        m = x.max(1).values
        lse = torch.logsumexp(x, 1)
        xl = x.gather(1, lab.clamp(max=3).unsqueeze(1))[:, 0]
        mag += ((lse - m).abs() + (xl - m).abs())[on].sum().item()
        cnt += n
    return (tot / cnt if cnt else math.nan), cnt, mag


# ---------------------------------------------------------------------------------------------------------------- head backward
def head_bwd_ref(p, label, ignore, w_ce, count, gprobs, gs, per=8):
    """d(w_ce * pce_loss(L, label) + gs * <gprobs, softmax(L)>) / dL at L = log(p), autograd, count = the forward's label count
    -> (ref fp64 [N,4,H,W], mag: the magnitude of the terms of the kernel's fp32 expression)"""
    refs, mags = [], []
    for a, b in chunks(p.shape[0], per):
        L = logits_of(p[a:b]).requires_grad_()
        f = L.new_zeros(())
        pd = p[a:b].double()
        mag = torch.zeros_like(pd)
        if label is not None and w_ce != 0 and count > 0:
            lab = label[a:b].long()
            on = labelled(lab, ignore)
            if bool(on.any()):
                f = f + w_ce * F.cross_entropy(L, torch.where(on, lab, torch.full_like(lab, ignore)), ignore_index=ignore,
                                               reduction="sum") / count
            hot = F.one_hot(lab.clamp(max=3), 4).permute(0, 3, 1, 2).double()
            mag = mag + abs(w_ce / count) * (pd + hot) * on.unsqueeze(1)
        if gprobs is not None and gs != 0:
            g = gprobs[a:b].double()
            f = f + gs * (g * torch.softmax(L, 1)).sum()
            mag = mag + abs(gs) * pd * (g.abs() + (g.abs() * pd).sum(1, keepdim=True))
        ref = torch.autograd.grad(f, L)[0] if f.requires_grad else torch.zeros_like(pd)
        refs.append(ref.detach())
        mags.append(mag)
    return torch.cat(refs), torch.cat(mags)


def grad_bound(ref, mag, dt=1):
    return U[dt] * ref.abs() + 2.0 ** -19 * mag + TINY[dt] + FP32_MIN


def check_nhwc16(d16, ref, mag, dt, what):
    """the channels-last 16-bit logit gradient [N,H,W,16]: the bound on channels 0..3, exact zeros on 4..15, no +-inf"""
    N, _, H, W = ref.shape
    reps = [report(d16[..., :4].reshape(-1, 4), ref.permute(0, 2, 3, 1).reshape(-1, 4),
                   grad_bound(ref, mag, dt).permute(0, 2, 3, 1).reshape(-1, 4), (N, H, W), what=what)]
    pad = d16[..., 4:].float()
    nz = int((pad != 0).sum())
    ninf = int(torch.isinf(d16.float()).sum())
    msg = None
    if nz or ninf:
        msg = f"{what}: {nz} nonzero padding channels, {ninf} infinite elements"
    reps.append({"worst": 0.0 if msg is None else math.inf, "bad": nz + ninf, "msg": msg})
    return reps


def round16(x, dt, truncate=False):
    """fp32 -> the 16-bit storage type, round to nearest even (as __floats2bfloat162_rn / __floats2half2_rn), or truncated"""
    x = x.float()
    if not truncate:
        return x.to(TORCH_T[dt])
    if dt == 0:
        return ((x.view(torch.int32) >> 16).to(torch.int16)).view(torch.bfloat16)
    h = x.to(torch.float16)
    over = h.float().abs() > x.abs()                        # rounded away from zero: step one ulp toward zero
    return torch.where(over, (h.view(torch.int16) - 1).view(torch.float16), h)


# ---------------------------------------------------------------------------------------------------------------- Gated CRF
def crf_ref(y, image, radius=5, sigma_xy=6.0, sigma_rgb=0.1, weight=1.0):
    """wsl_oracle's Gated CRF one sample at a time -> (loss over the batch, sum k over the batch, d loss / dy, sum_j k_ij |y_j| * |d
    loss / d s| as the bound's magnitude, |loss terms|).  The unfold formulation runs on the GPU, the loop one on the CPU."""
    fn = O.gated_crf_loss_unfold if y.is_cuda else O.gated_crf_loss
    N, C, H, W = y.shape
    loss, ksum, grads, mags = 0.0, 0.0, [], []
    for n in range(N):
        yn = y[n:n + 1].double().requires_grad_()
        img = image[n:n + 1].double()
        ln = fn(yn, img, radius, sigma_xy, sigma_rgb, weight) / N
        g = torch.autograd.grad(ln, yn)[0]
        kn = (fn(torch.zeros_like(yn), img, radius, sigma_xy, sigma_rgb, weight) / N).item()   # y = 0 leaves sum k / (N H W)
        loss += ln.item()
        ksum += kn * N * H * W
        if bool((y[n] >= 0).all()):
            m = g.abs()                                   # d loss / dy_i = -2 sum_j k_ij y_j / (N H W), so |g| = |gscale| sum_j k_ij |y_j|
        else:
            ya = y[n:n + 1].double().abs().requires_grad_()
            m = torch.autograd.grad(fn(ya, img, radius, sigma_xy, sigma_rgb, weight) / N, ya)[0].abs()
        grads.append(g.detach())
        mags.append(m.detach())
        del yn, g
    pair = ksum - loss * N * H * W
    return loss, ksum, torch.cat(grads), torch.cat(mags), (ksum + abs(pair)) / (N * H * W)


def crf_s(y, image, radius=5, sigma_xy=6.0, sigma_rgb=0.1, weight=1.0, drop=None, seam=None):
    """fp64 s_i = sum_j k_ij y_j over the in-bounds window of every pixel, restated tap by tap with explicit neighbour indices, so
    a kernel mistake can be planted: drop = (dy, dx) leaves that tap out; seam = (TH, TW) reads every halo row above a TH-row
    tile from the tile TW columns to the right (zero beyond the image)"""
    N, C, H, W = y.shape
    dev = y.device
    Y = torch.arange(H, device=dev).view(H, 1).expand(H, W)
    X = torch.arange(W, device=dev).view(1, W).expand(H, W)
    yd, I = y.double(), image.double()[:, 0]
    s = torch.zeros_like(yd)
    for dy in range(-radius, radius + 1):
        for dx in range(-radius, radius + 1):
            if (dy == 0 and dx == 0) or (dy, dx) == drop:
                continue
            NY, NX = Y + dy, X + dx
            if seam is not None:
                NX = torch.where(NY < (Y // seam[0]) * seam[0], NX + seam[1], NX)
            ok = (NY >= 0) & (NY < H) & (NX >= 0) & (NX < W)
            idx = (NY.clamp(0, H - 1) * W + NX.clamp(0, W - 1)).reshape(-1)
            In = I.reshape(N, -1)[:, idx].reshape(N, H, W)
            k = weight * torch.exp(-0.5 * ((dx * dx + dy * dy) / sigma_xy ** 2 + (In - I) ** 2 / sigma_rgb ** 2))
            k = torch.where(ok, k, torch.zeros_like(k))
            yn = yd.reshape(N, C, -1)[:, :, idx].reshape(N, C, H, W)
            s += k.unsqueeze(1) * yn
    return s


# ---------------------------------------------------------------------------------------------------------------- Mumford-Shah
def ms_ref(image, p, scale):
    """wsl_oracle.mumford_shah_loss one sample at a time -> (loss, sum |terms|, centroids [N,4], scale * d loss / dp)"""
    N = p.shape[0]
    loss, mag, cents, grads = 0.0, 0.0, [], []
    for n in range(N):
        I, pn = image[n:n + 1].double(), p[n:n + 1].double().requires_grad_()
        ln = O.mumford_shah_loss(I, pn)
        grads.append(scale * torch.autograd.grad(ln, pn)[0])
        q = pn.detach()
        c = (q * I).sum((2, 3)) / I.sum((2, 3))
        cents.append(c[0])
        tv = (q[:, :, 1:] - q[:, :, :-1]).abs().sum() + (q[:, :, :, 1:] - q[:, :, :, :-1]).abs().sum()
        mag += ((q * q * I).sum() + (c * (q * I).sum((2, 3))).sum() + tv).item()
        loss += ln.item()
    return loss, mag, torch.stack(cents), torch.cat(grads)


def ms_bwd_bound(image, p, cent_got, cent_ref, scale):
    """2 (p - c) I + four signs, in fp32 at the forward's fp32 centroid: the level term within 2^-20 of its magnitude, the sign
    terms exact, and the centroid's own error 2 |c_got - c_ref| I"""
    I = image.double()
    c = cent_got.double().view(p.shape[0], 4, 1, 1)
    dc = (cent_got.double() - cent_ref.reshape(-1)).abs().view(p.shape[0], 4, 1, 1)
    return abs(scale) * (2.0 ** -20 * (2 * (p.double().abs() + c.abs()) * I + 4) + 2 * dc * I) + FP32_MIN


# ---------------------------------------------------------------------------------------------------------------- Dice
def dice_ref(p, target, mode, scale, ignore=4):
    """mode 'dice': wsl_oracle.dice_loss (no mask, M = 1); 'pdice': wsl_oracle.pdice_loss (M = the batch-summed ignore mask)
    -> (loss, sums [12] = I, Y, Z per class, scale * d loss / dp, M [H,W])"""
    P = p.double().requires_grad_()
    t = target.long().unsqueeze(1)
    loss = O.dice_loss(P, t) if mode == "dice" else O.pdice_loss(P, t, 4, ignore)
    g = scale * torch.autograd.grad(loss, P)[0]
    q = p.double()
    M = torch.ones(p.shape[-2:], dtype=torch.float64, device=p.device) if mode == "dice" else \
        (target != ignore).double().sum(0)
    s = []
    for k in range(3):
        for c in range(4):
            tt = (target.long() == c).double()
            s.append(((q[:, c] * tt if k == 0 else tt if k == 1 else q[:, c] ** 2) * M).sum())
    return loss.item(), torch.stack(s), g, M


def dice_loss_tol(sums):
    """the loss error the STAT_TOL sum errors allow: (1/C) sum_c 2 dI / den + (2I + eps) (dY + dZ) / den^2"""
    I, Y, Z = sums[:4], sums[4:8], sums[8:]
    den = Z + Y + 1e-5
    return (STAT_TOL * (2 * I / den + (2 * I + 1e-5) * (Y + Z) / den ** 2)).sum().item() / 4 + 2.0 ** -24


def dice_bwd_bound(p, target, M, sums, scale):
    """(a_c t + b_c s) M with a, b from the forward's sums: their STAT_TOL error, and the fp32 evaluation"""
    I, Y, Z = sums[:4].view(1, 4, 1, 1), sums[4:8].view(1, 4, 1, 1), sums[8:].view(1, 4, 1, 1)
    den, num = Z + Y + 1e-5, 2 * I + 1e-5
    t = F.one_hot(target.long().clamp(max=4), 5)[..., :4].permute(0, 3, 1, 2).double()
    a, b = abs(scale) / 4 * 2 / den, abs(scale) / 4 * 2 * num / den ** 2
    return (a * t * (STAT_TOL + 2.0 ** -21) + b * p.double().abs() * (3 * STAT_TOL + 2.0 ** -21)) * M + FP32_MIN


# ---------------------------------------------------------------------------------------------------------------- TV
def tv_ref(p, grad_scale):
    """wsl_oracle.tv_loss of the planes p [P,H,W] -> (loss, sum |contour|, grad_scale * d loss / dp)"""
    P = p.double().unsqueeze(0).requires_grad_()
    loss = O.tv_loss(P)
    g = grad_scale * torch.autograd.grad(loss, P)[0][0]
    return loss.item(), loss.item() * p.numel(), g


def tv_route(p, gscale, last=False):
    """tv_kernel's routing emulated: +gscale to the argmin of the window whose min is largest, -gscale to the argmin of the centre
    window, over the in-bounds 3 x 3 windows; ties to the first extremum in row-major scan order (last=True: the last)"""
    Pn, H, W = p.shape
    x = p.double().unsqueeze(1)

    def arg(v, pad, fmin):
        win = F.unfold(F.pad(v, (1, 1, 1, 1), value=pad), 3)            # [P, 9, H*W], window in row-major order
        w = win if fmin else -win
        j = (8 - w.flip(1).argmin(1)) if last else w.argmin(1)
        return win.gather(1, j.unsqueeze(1))[:, 0], j

    mn, jc = arg(x, math.inf, True)
    mx, jm = arg(mn.view(Pn, 1, H, W), -math.inf, False)
    pos = torch.arange(H * W, device=p.device).expand(Pn, H * W)
    ofs = lambda j: (j // 3 - 1) * W + (j % 3 - 1)
    argc = pos + ofs(jc)                                                   # the centre window's argmin
    q = pos + ofs(jm)                                                      # the neighbour whose min is the max
    argm = argc.gather(1, q)
    on = (mx - mn) > 0
    g = torch.zeros(Pn, H * W, dtype=torch.float64, device=p.device)
    w = on.double() * gscale
    g.scatter_add_(1, argm, w)
    g.scatter_add_(1, argc, -w)
    return g.view(Pn, H, W)


def tv_bound(ref, gscale):
    return 2.0 ** -22 * ref.abs() + 2.0 ** -14 * abs(gscale)


# ---------------------------------------------------------------------------------------------------------------- entropy
def entropy_ref(p, scale):
    """wsl_oracle.entropy_loss -> (loss, sum |terms| + the fp32 rounding of p + 1e-6, scale * d loss / dp, the backward's bound)"""
    P = p.double().requires_grad_()
    loss = O.entropy_loss(P, 4)
    g = scale * torch.autograd.grad(loss, P)[0]
    q = p.double()
    lg = torch.log(q + 1e-6)
    norm = q.numel() / 4 * math.log(4)
    # per term, logf(p + 1e-6f) is off by up to 2^-23 (1 + |log|) (the rounded argument, then logf): carried into the magnitude
    mag = ((q * lg).abs() + 2.0 ** -22 / STAT_TOL * q * (1 + lg.abs())).sum().item() / norm
    bound = abs(scale) / norm * 2.0 ** -21 * (1 + lg.abs()) + 2.0 ** -22 * g.abs() + FP32_MIN
    return loss.item(), mag, g, bound


# ---------------------------------------------------------------------------------------------------------------- class variance
def variance_ref(image, p, scale):
    """wsl_oracle.class_variance_loss -> dict of the loss, inter, intra, per-(n, c) {mean, std}, per-n {mean, std}, scale * the
    autograd gradient, the mask of the zero-std (n, c) and the sums the bounds need.  torch.std's backward gives a zero gradient
    where the std is 0, which is what the kernel does there."""
    I = image.double()
    P = p.double().requires_grad_()
    loss = O.class_variance_loss(P, I)
    g = scale * torch.autograd.grad(loss, P)[0]
    v = I * p.double()
    sd = torch.std(v, dim=[2, 3])
    mean = v.mean((2, 3))
    inter = torch.std(mean, dim=1).mean().item()
    return {"loss": loss.item(), "inter": inter, "intra": sd.mean().item(), "mean": mean, "sd": sd, "mbar": mean.mean(1),
            "sdn": torch.std(mean, dim=1), "grad": g, "zero": sd == 0, "S2": (v * v).sum((2, 3)), "S1": v.sum((2, 3)),
            "M": v.shape[2] * v.shape[3]}


def variance_tols(r):
    """std of M values from fp32 sums: |sd - ref| <= STAT_TOL (S2 + S1^2 / M) / (M - 1) / sd; means STAT_TOL |S1| / M + 2^-24"""
    M = r["M"]
    dvar = STAT_TOL * (r["S2"] + r["S1"] ** 2 / M) / (M - 1)
    dsd = torch.where(r["sd"] > 0, dvar / r["sd"].clamp_min(1e-300), dvar.sqrt()) + 2.0 ** -24 * r["sd"]
    dmean = STAT_TOL * r["S1"].abs() / M + 2.0 ** -24 * r["mean"].abs()
    dsdn = dmean.sum(1) + 2.0 ** -24 * r["sdn"]
    return dsd, dmean, dsdn


def variance_bwd_bound(image, p, r, scale, dsd, dmean, dsdn):
    """the fp32 evaluation (2^-20 of the terms) and the forward's statistics errors carried through the two quotients"""
    N, M = p.shape[0], r["M"]
    I = image.double().abs()
    v = (image.double() * p.double()).abs()
    mean, sd, dm, ds = (r["mean"].view(N, 4, 1, 1), r["sd"].view(N, 4, 1, 1), dmean.view(N, 4, 1, 1), dsd.view(N, 4, 1, 1))
    mbar, sdn, dsn = r["mbar"].view(N, 1, 1, 1), r["sdn"].view(N, 1, 1, 1), dsdn.view(N, 1, 1, 1)
    sdn_, sd_ = sdn.clamp_min(1e-300), sd.clamp_min(1e-300)
    inter = (mean - mbar).abs() / (3 * sdn_ * M * N)
    intra = (v + mean.abs()) / ((M - 1) * sd_ * N * 4)
    d_inter = (dm + dm.mean(1, keepdim=True)) / (3 * sdn_ * M * N) + inter * dsn / sdn_
    d_intra = dm / ((M - 1) * sd_ * N * 4) + intra * ds / sd_
    z = torch.zeros_like(inter)
    return abs(scale) * I * (torch.where(sdn > 0, 2.0 ** -20 * inter + d_inter, z) + torch.where(sd > 0, 2.0 ** -20 * intra + d_intra, z))


# ---------------------------------------------------------------------------------------------------------------- UAMT / MT
def mc_rows(T, B, layout="kernel"):
    """row of the Monte-Carlo buffer holding pass t of sample b -> long [T, B]; 'kernel' the step's layout, 'sample_major' a fault"""
    t = torch.arange(T).view(T, 1)
    b = torch.arange(B).view(1, B)
    if layout == "kernel":
        return (t >> 1) * 2 * B + (t & 1) * B + b
    return b * T + t


def uncertainty_ref(mc, T, B):
    """wsl_oracle.uamt_losses' uncertainty in fp64 -> (unc [B,H,W], its band UNC_BAND (1 + sum_c |q log(q + 1e-6)|))"""
    preds = F.softmax(mc.double(), dim=1).reshape(T, B, *mc.shape[1:]).mean(0)
    terms = preds * torch.log(preds + 1e-6)
    return -terms.sum(1), UNC_BAND * (1 + terms.abs().sum(1))


def uncertainty_fp32(mc, T, B, layout="kernel"):
    """the kernel's fp32 arithmetic: softmax of each pass, the sum over passes in pass order, / T, -sum q logf(q + 1e-6f)"""
    rows = mc_rows(T, B, layout).to(mc.device)
    pbar = torch.zeros(B, 4, *mc.shape[2:], device=mc.device)
    for t in range(T):
        pbar = pbar + torch.softmax(mc[rows[t]].float(), 1)
    q = pbar / T
    return -(q * torch.log(q + np.float32(1e-6))).sum(1)


def mask_check(mask, unc, band, thr, what="uncertainty mask"):
    """bit-exact outside the band around the threshold -> (report, fraction of pixels in the band)"""
    ref = (unc < thr).to(torch.uint8)
    near = (unc - thr).abs() <= band
    got = torch.where(near, ref, mask)
    B, H, W = mask.shape
    rep = exact(got.view(-1, 1), ref.view(-1, 1), (B, H, W), what=what)
    return rep, near.double().mean().item()


def consistency_ref(student, teacher, mask, w):
    """mean teacher (mask None, semi_oracle.mt_losses' term: softmax_mse(...).mean()) or UAMT (wsl_oracle.uamt_losses' masked term)
    -> (loss, sum of the (masked) distance, count, w * d loss / d student, the backward's bound)"""
    S = student.double().requires_grad_()
    dist = O.softmax_mse(S, teacher.double())
    if mask is None:
        m = torch.ones_like(dist[:, :1])
        cnt = float(dist.numel())
        loss = dist.mean()
        coef = 2 * abs(w) / cnt
    else:
        m = mask.double().unsqueeze(1)
        cnt = m.sum().item()
        loss = (m * dist).sum() / (2 * m.sum() + 1e-16)
        coef = 2 * abs(w) / (2 * cnt + 1e-16)
    g = torch.autograd.grad(w * loss, S)[0]
    ps, pt = torch.softmax(student.double(), 1), torch.softmax(teacher.double(), 1)
    rs, rt = softmax_rel(student), softmax_rel(teacher)
    e = ps * rs + pt * rt                               # the fp32 softmaxes' absolute errors
    bound = coef * m * ps * 4 * (e + (e * ps).sum(1, keepdim=True)) + (2.0 ** -22 + rs) * g.abs() + FP32_MIN
    return loss.item(), (m * dist).sum().item(), cnt, g, bound


# ---------------------------------------------------------------------------------------------------------------- S2L
def s2l_ref(logits, scribble, weight, thr, w_u):
    """s2l_oracle.u_labels and the step loss pCE + w_u * CE_u (train_s2l.py:123-147) in fp64 -> dict"""
    ul = SO.u_labels(weight.float(), scribble, float(np.float32(thr)))
    x = logits.double()
    ce, n, mag = pce_ref(x, scribble, 4)
    ce_u, n_u, mag_u = pce_ref(x, ul.to(torch.uint8), 4)
    loss = ce + w_u * ce_u if w_u != 0 else ce
    return {"ulab": ul.to(torch.uint8), "ce": ce, "n": n, "mag": mag, "ce_u": ce_u, "n_u": n_u, "mag_u": mag_u, "loss": loss}


def u_labels_first_wins(weight, scribble, thr):
    """the mistaken rule: the FIRST class whose weight is > thr wins"""
    ul = torch.full(scribble.shape, 4, dtype=torch.uint8, device=scribble.device)
    for c in (3, 2, 1, 0):
        ul = torch.where((weight[..., c] > float(np.float32(thr))) & (scribble == 4), torch.full_like(ul, c), ul)
    return ul


def s2l_bwd_ref(p, scribble, ulab, S, w_u, n, n_u):
    """d(S * pCE + S * w_u * CE_u)/dL at L = log p (autograd), the forward's counts; no u-term when no pixel qualifies"""
    g1, m1 = head_bwd_ref(p, scribble, 4, S, n, None, 0.0)
    if w_u == 0 or n_u == 0:
        return g1, m1
    u = torch.where(scribble == 4, ulab, torch.full_like(ulab, 4))
    g2, m2 = head_bwd_ref(p, u, 4, S * w_u, n_u, None, 0.0)
    return g1 + g2, m1 + m2


# ---------------------------------------------------------------------------------------------------------------- noise / EMA
def noise_ref(x, reps, sigma, clampv, seed):
    """x.repeat(reps) + clamp(sigma * N(0, 1), +-c), N(0, 1) by Box-Muller of wsl_uniform draws 2i, 2i + 1, in fp64 at the fp32
    sigma / clamp -> (ref, bound)"""
    n = x.numel()
    u = torch.from_numpy(uniform(seed, 2 * n * reps).astype(np.float64)).to(x.device)
    u1, u2 = u[0::2].clamp_min(float(np.float32(1e-7))), u[1::2]
    r = torch.sqrt(-2 * torch.log(u1))
    z = r * torch.cos(2 * math.pi * u2)
    sg, c = float(np.float32(sigma)), float(np.float32(clampv))
    nz = (z * sg).clamp(-c, c)
    xr = x.double().reshape(-1).repeat(reps)
    ref = xr + nz
    return ref, 2.0 ** -24 * (xr.abs() + ref.abs()) + 2.0 ** -20 * sg * r


def ema_ref(ema, param, alpha):
    """update_ema_variables' ema * alpha + (1 - alpha) * param in fp64 at the fp32 alpha -> (ref, bound: three fp32 roundings)"""
    a = float(np.float32(alpha))
    e, p = ema.double(), param.double()
    ref = e * a + (1 - a) * p
    return ref, 2.0 ** -22 * ((e * a).abs() + ((1 - a) * p).abs())
