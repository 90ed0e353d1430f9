"""ctypes binding of libwsl4mis_b200.so, generated from include/wsl4mis_b200.h.

The product path has NO fallback: if the CUDA library is missing or a kernel call fails, an
exception is raised.  (PyTorch is only plumbing here: device memory, streams, autograd glue.)
"""
import ctypes
import os
import re

import torch

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
HEADER = os.path.join(ROOT, "include", "wsl4mis_b200.h")
LIB_PATH = os.path.join(PKG, "libwsl4mis_b200.so")

_SCALARS = {
    "int": ctypes.c_int,
    "float": ctypes.c_float,
    "double": ctypes.c_double,
    "long long": ctypes.c_longlong,
    "unsigned long long": ctypes.c_ulonglong,
    "unsigned int": ctypes.c_uint,
    "cudaStream_t": ctypes.c_void_p,
}


def parse_header(path=HEADER):
    """-> {name: (restype, [(ctype, argname), ...])} for every prototype in the header."""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"(const char\*|int)\s+(wsl_\w+)\s*\(([^)]*)\)\s*;", src):
        ret, name, args = m.group(1), m.group(2), m.group(3).strip()
        alist = []
        if args and args != "void":
            for a in args.split(","):
                a = " ".join(a.split())
                if "*" in a:
                    alist.append((ctypes.c_void_p, a.split("*")[-1].strip()))
                else:
                    ty, nm = a.rsplit(" ", 1)
                    alist.append((_SCALARS[ty], nm))
        protos[name] = (ctypes.c_char_p if ret.startswith("const char") else ctypes.c_int, alist)
    return protos


class _Lib:
    def __init__(self):
        self._dll = None
        self.protos = parse_header()

    def load(self):
        if self._dll is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"{LIB_PATH} not found: build it with `python -m wsl4mis_b200._build` "
                    "(or __graft_entry__.build()). There is no CPU / PyTorch fallback.")
            dll = ctypes.CDLL(LIB_PATH)
            for name, (ret, args) in self.protos.items():
                fn = getattr(dll, name)  # AttributeError if the header and the library disagree
                fn.restype = ret
                fn.argtypes = [t for t, _ in args]
            self._dll = dll
        return self._dll

    def last_error(self):
        return self.load().wsl_last_error().decode()


LIB = _Lib()


def _ptr(x):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.data_ptr()
    return int(x)


def stream_handle():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    """Call an int-returning entry point; the trailing cudaStream_t argument is filled in automatically
    with torch's current stream.  Tensors are passed as raw device pointers."""
    dll = LIB.load()
    ret, proto = LIB.protos[name]
    vals = []
    args = list(args)
    if len(args) == len(proto) - 1 and proto and proto[-1][1] == "stream":
        args.append(stream_handle())
    if len(args) != len(proto):
        raise TypeError(f"{name}: expected {len(proto)} arguments ({[n for _, n in proto]}), got {len(args)}")
    for (ty, _), a in zip(proto, args):
        vals.append(_ptr(a) if ty is ctypes.c_void_p else a)
    COUNTERS["launch_calls"] += 1
    if PROFILE is not None:
        PROFILE.record(name, getattr(dll, name), vals)
        return 0
    rc = getattr(dll, name)(*vals)
    if ret is ctypes.c_int and rc != 0 and name not in ("wsl_abi_version", "wsl_workspace_floats", "wsl_tc_available"):
        raise RuntimeError(f"{name} failed ({rc}): {LIB.last_error()}")
    return rc


COUNTERS = {"launch_calls": 0}
PROFILE = None   # set to a _Profiler by bench.py to time every C-ABI call with CUDA events


class Profiler:
    """Per-call CUDA-event timing of the C-ABI launches (used by bench.py for the roofline table)."""

    def __init__(self):
        self.rows = []   # (name, start_event, stop_event, meta)
        self.meta = None

    def record(self, name, fn, vals):
        s = torch.cuda.Event(enable_timing=True)
        e = torch.cuda.Event(enable_timing=True)
        s.record()
        rc = fn(*vals)
        e.record()
        if rc != 0:
            raise RuntimeError(f"{name} failed ({rc}): {LIB.last_error()}")
        self.rows.append((name, s, e, self.meta))

    def table(self):
        torch.cuda.synchronize()
        agg = {}
        for name, s, e, meta in self.rows:
            key = (name, meta)
            ms = s.elapsed_time(e)
            a = agg.setdefault(key, [0, 0.0])
            a[0] += 1
            a[1] += ms
        return agg


_WS = {}


def workspace(tag, device=None):
    """Zero-initialised reduction workspace, one per call site tag and device."""
    device = torch.device(device if device is not None else torch.cuda.current_device())
    key = (tag, str(device))
    if key not in _WS:
        n = LIB.load().wsl_workspace_floats()
        _WS[key] = torch.zeros(n, dtype=torch.float32, device=device)
    return _WS[key]
