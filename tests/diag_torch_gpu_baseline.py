"""Diagnostic (not collected by pytest): the reference step as STOCK EAGER PYTORCH ON THE SAME GPU -- SURVEY 8(d)'s "real
kernel to beat" (the reference is a plain PyTorch program; /root/reference does not exist on the GPU box, so its pinned
functional restatement oracle/wsl_oracle.py is run on cuda tensors: same ATen/cuDNN operators, GatedCRF in the reference's
materialising F.unfold formulation).  Batch 16 bounds the unfold temporaries (~12 GB with autograd); images/s is reported
for PyTorch's default settings (cudnn.allow_tf32 = True) and for strict fp32.

    python tests/diag_torch_gpu_baseline.py
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import wsl_oracle as O  # noqa: E402

dev = torch.device("cuda", 0)
N = int(os.environ.get("N", "16"))
O.CRF_IMPL = "unfold"
p = {k: v.to(dev) for k, v in O.synth_params(1, 4, ("main_decoder", "aux_decoder1"), 7).items()}
image, label = O.synth_batch(N, 256, 256, seed=3)
image, label = image.to(dev), label.to(dev)
for tf32 in (True, False):
    torch.backends.cudnn.allow_tf32 = tf32
    moms = {}
    params = {k: v.clone() for k, v in p.items()}

    def step():
        loss, grads, _ = O.full_step(params, image, label, "pce_gatedcrf", True)
        O.sgd_step({k: params[k] for k in grads}, grads, moms, 0.01)
        return loss

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    K = 5
    for _ in range(K):
        step()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / K
    print(f"stock eager PyTorch on cuda (cudnn tf32={tf32}), unet_cct pCE+GatedCRF, batch {N}: {dt * 1e3:.1f} ms/step = {N / dt:.0f} images/s; "
          f"peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
