"""ptxas must keep the halo convolution (conv_tc2) fully asynchronous, C7518 included.

conv_tc2 issues the next tile's first MMA group before it finishes the current tile's epilogue.  If the MMAs are issued on a
path that joins one without a group in flight, or the thread that stores the tile branches on its index while a group is in
flight, ptxas serialises every wgmma of the kernel and reports C7518 ("compiler-inserted WG.DP in divergent path").  The
pipeline test checks C7515 / C7519 for the whole file; this one adds C7518 for the conv_tc2 instantiations."""
import os
import re
import subprocess

import pytest

from wsl4mis_b200 import _build


def test_conv_tc2_wgmma_not_serialised(tmp_path):
    if not os.path.exists(_build.NVCC):
        pytest.skip(f"nvcc not found at {_build.NVCC}")
    src = os.path.join(_build.CSRC, "conv_tc.cu")
    cmd = [_build.NVCC, *_build.ARCH, *_build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "conv_tc.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    assert re.search(r"Compiling entry function '\S*conv_tc2_kernel", r.stdout), "ptxas -v printed no conv_tc2 report"
    bad = [ln for ln in r.stdout.splitlines() if re.search(r"\(C751[589]\)", ln) and "conv_tc2_kernel" in ln]
    assert not bad, f"{len(bad)} wgmma serialisation warnings in conv_tc2, e.g.:\n" + "\n".join(bad[:5])
