"""wsl4mis_b200 -- H100-native (sm_90a) kernels for the WSL4MIS segmentation-training hot path.

Public surface mirrors the reference's ``code/networks`` and ``code/utils`` modules:
    wsl4mis_b200.networks.unet / net_factory
    wsl4mis_b200.utils.losses / gate_crf_loss / ramps
plus ``wsl4mis_b200.engine`` (the fused per-step training body used by bench.py).
"""
__version__ = "0.1.0"
