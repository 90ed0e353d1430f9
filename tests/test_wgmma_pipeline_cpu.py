"""ptxas must keep every wgmma kernel of conv_tc.cu asynchronous.

ptxas reports C7515 ("wgmma.mma_async instructions are serialized") when a non-wgmma instruction writes accumulator
registers while an MMA group may be in flight, and C7519 when it has to insert a warpgroup.arrive before an MMA (for
example after a runtime branch between two MMAs).  Either makes every MMA of the kernel wait for the previous one, which
the consumer pipelines in conv_tc.cu are built to avoid.  The check compiles the file exactly as the build does (no GPU
needed) and fails on any such line."""
import os
import re
import subprocess

import pytest

from wsl4mis_b200 import _build


def test_no_serialised_wgmma_in_conv_tc(tmp_path):
    if not os.path.exists(_build.NVCC):
        pytest.skip(f"nvcc not found at {_build.NVCC}")
    src = os.path.join(_build.CSRC, "conv_tc.cu")
    cmd = [_build.NVCC, *_build.ARCH, *_build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "conv_tc.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    assert "Compiling entry function" in r.stdout and "conv_row_kernel" in r.stdout, "ptxas -v printed no kernel report"
    bad = [ln for ln in r.stdout.splitlines() if re.search(r"\(C75(15|19)\)", ln)]
    names = sorted({m.group(1) for ln in bad for m in [re.search(r"function '([^']+)'", ln)] if m})
    assert not bad, f"{len(bad)} wgmma serialisation warnings in {len(names)} kernels, e.g.:\n" + "\n".join(bad[:5])
