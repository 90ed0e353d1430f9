"""Build the C-ABI CUDA library in-tree with nvcc (sm_90a only).

    python -m wsl4mis_b200._build        # or __graft_entry__.build()

Objects are cached under wsl4mis_b200/csrc/build/ keyed by source mtime; the resulting
``wsl4mis_b200/libwsl4mis_b200.so`` is git-ignored but travels with the tree to the GPU box.
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(PKG, "libwsl4mis_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--use_fast_math=false"]
FLAGS = [f for f in FLAGS if not f.startswith("--use_fast_math")]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr_m = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    objs, rebuilt = [], False
    procs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_m):
            cmd = [NVCC, *ARCH, *FLAGS, "-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
            rebuilt = True
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out.decode()}")
        if verbose and out:
            print(out.decode())
    if rebuilt or not os.path.exists(LIB):
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart"]
        if verbose:
            print(" ".join(cmd))
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout.decode())
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
