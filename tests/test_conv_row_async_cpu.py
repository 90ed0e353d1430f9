"""ptxas must keep the row convolution (conv_row) fully asynchronous and free of register spills.

conv_row issues the next input row's MMA group before it stores the row it has just completed.  A branch on the thread index
while that group is in flight (a per-thread store guard, say) makes ptxas serialise every wgmma of the kernel (C7518), and so
does an accumulator it cannot keep beside the in-flight one (C7511); C7515 / C7519 are the other serialisation reports.  Every
instantiation runs at ptxas's 168-register allocation for a 384-thread CTA, so any added live state that does not fit shows up
as spill stores: none are allowed."""
import os
import re
import subprocess

import pytest

from wsl4mis_b200 import _build


def test_conv_row_wgmma_not_serialised_and_no_spills(tmp_path):
    if not os.path.exists(_build.NVCC):
        pytest.skip(f"nvcc not found at {_build.NVCC}")
    src = os.path.join(_build.CSRC, "conv_tc.cu")
    cmd = [_build.NVCC, *_build.ARCH, *_build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "conv_tc.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    bad, spills, seen, cur = [], [], 0, None
    for ln in r.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1) if "conv_row_kernel" in m.group(1) else None
            seen += cur is not None
            continue
        if re.search(r"\(C751\d\)", ln) and "conv_row_kernel" in ln:
            bad.append(ln)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if cur is not None and m and (int(m.group(1)) or int(m.group(2))):
            spills.append(f"{cur}: {ln.strip()}")
    assert seen, "ptxas -v printed no conv_row report"
    assert not bad, f"{len(bad)} wgmma serialisation warnings in conv_row, e.g.:\n" + "\n".join(bad[:5])
    assert not spills, f"{len(spills)} conv_row instantiations spill:\n" + "\n".join(spills[:5])
