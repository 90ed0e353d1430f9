import numpy as np
import torch

import wsl_oracle as O


def nhwc(x_nchw, dtype=torch.bfloat16):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(dtype)


def nchw(x_nhwc):
    return x_nhwc.float().permute(0, 3, 1, 2).contiguous()


def bf16_round(x):
    return x.to(torch.bfloat16).float()


def elem_masks_nchw(seed, n, h, w):
    rs = np.random.RandomState(seed)
    return [torch.from_numpy((rs.uniform(size=(n, O.FT[i], h >> i, w >> i)) >= O.ENC_DROP[i]).astype(np.uint8))
            for i in range(5)]


def chan_masks(seed, n):
    rs = np.random.RandomState(seed)
    return [torch.from_numpy((rs.uniform(size=(n, c)) >= 0.5).astype(np.uint8)) for c in O.FT]


ENC_MASK_KEYS = ["encoder.in_conv.conv_conv.3"] + [f"encoder.down{i}.maxpool_conv.1.conv_conv.3" for i in range(1, 5)]


def pack_conv_weights(w, c_slices, dt=0):
    """Packed operands of a torch-layout weight w [Cout, Cin, k, k] on the GPU: 'wf' / 'bf' the forward packs (fp32 / 16-bit,
    dt 0 = bf16, 2 = fp16 bits), 'wd' / 'bd' the data-gradient packs per input-channel slice in c_slices."""
    from wsl4mis_b200._lib import call
    dev = w.device
    Cout, Cin, ks, _ = w.shape
    T = ks * ks
    CoutP, CinP = (Cout + 15) // 16 * 16, (Cin + 15) // 16 * 16
    pk = {"wf": torch.zeros(T * CinP * CoutP, device=dev), "bf": torch.zeros(T * CinP * CoutP, device=dev, dtype=torch.bfloat16),
          "wd": [], "bd": [], "CoutP": CoutP, "CinP": CinP}
    beg = 0
    for i, c in enumerate(c_slices):
        sp = (c + 15) // 16 * 16
        wd = torch.zeros(T * CoutP * sp, device=dev)
        bd = torch.zeros(T * CoutP * sp, device=dev, dtype=torch.bfloat16)
        call("wsl_pack_conv_weights", w, Cout, Cin, ks, CoutP, CinP, beg, c, pk["wf"] if i == 0 else None, wd,
             pk["bf"] if i == 0 else None, bd, dt)
        pk["wd"].append(wd)
        pk["bd"].append(bd)
        beg += c
    return pk


class LaunchRecorder:
    """Stands in for wsl4mis_b200._lib.PROFILE: runs every C-ABI call as call() does (a nonzero return code raises) and keeps the
    distinct launches whose entry point `keep(name)` accepts, as (entry, ((scalar name, value), ...), (names of pointer arguments
    passed as NULL, ...)) -> number of calls.  on_record(key, name, vals), when given, sees every kept call (pointer values included)."""

    def __init__(self, keep, on_record=None):
        self.meta = None
        self.keep = keep
        self.on_record = on_record
        self.launches = {}

    def record(self, name, fn, vals):
        import ctypes
        from wsl4mis_b200._lib import LIB
        rc = fn(*vals)
        if rc != 0:
            raise RuntimeError(f"{name} failed ({rc}): {LIB.last_error()}")
        if self.keep(name):
            args = [(nm, ty, v) for (ty, nm), v in zip(LIB.protos[name][1], vals) if nm != "stream"]
            key = (name, tuple((nm, v) for nm, ty, v in args if ty is not ctypes.c_void_p),
                   tuple(nm for nm, ty, v in args if ty is ctypes.c_void_p and v is None))
            self.launches[key] = self.launches.get(key, 0) + 1
            if self.on_record is not None:
                self.on_record(key, name, vals)


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cosine(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return (torch.dot(a, b) / (a.norm() * b.norm() + 1e-30)).item()
