"""Launcher for the reference's UNCHANGED training scripts on the H100 modules:

    cd /path/to/WSL4MIS/code
    python -m wsl4mis_b200.run train_weakly_supervised_pCE_GatedCRFLoss_2D.py --model unet --batch_size 64 ...

Equivalent to `PYTHONPATH=<repo>/dropin:<repo> python <script> ...` (the shim packages in dropin/ are regular packages and
therefore win over the namespace directories of code/ wherever they sit on sys.path); the launcher only spares the user
the path bookkeeping, aliases `tensorboardX` to `torch.utils.tensorboard` when the former is not installed, and reports
which files the scripts' module names resolved to."""
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(argv):
    if not argv:
        print(__doc__)
        return 2
    script = os.path.abspath(argv[0])
    for p in (ROOT, os.path.join(ROOT, "dropin")):
        if p in sys.path:
            sys.path.remove(p)
    sys.path[:0] = [os.path.dirname(script), os.path.join(ROOT, "dropin"), ROOT]      # sys.path[0] = script dir, as python sets it
    try:
        import tensorboardX  # noqa: F401
    except ImportError:
        try:
            import types
            from torch.utils.tensorboard import SummaryWriter
            mod = types.ModuleType("tensorboardX")
            mod.SummaryWriter = SummaryWriter
            sys.modules["tensorboardX"] = mod
        except Exception:
            pass
    import networks.net_factory
    import utils.losses
    print(f"[wsl4mis_b200.run] networks.net_factory -> {networks.net_factory.__file__}\n"
          f"[wsl4mis_b200.run] utils.losses         -> {utils.losses.__file__}", file=sys.stderr)
    sys.argv = [script] + list(argv[1:])
    runpy.run_path(script, run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
