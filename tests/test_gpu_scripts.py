"""The reference's OWN training scripts, unchanged, on the H100 modules (SURVEY 8(b); VERDICT r1 item 5).

The unmodified `train_*.py` files come from the archive `oracle/build_ref.py` staged in the build container (git-ignored, it
travels with the tree; /root/reference does not exist on the GPU box).  Each test unpacks it into a scratch `code/` directory,
puts `dropin/` + the repo + the harness stand-ins (tensorboardX, medpy, skimage, h5py) on PYTHONPATH and runs the script as
`python train_....py --root_path synthetic:30 --max_iterations K ...` from that directory, exactly as a user of the reference would."""
import os
import re
import subprocess
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stage(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    try:
        import build_ref
        code = build_ref.extract(str(tmp_path))
    finally:
        sys.path.pop(0)
    if code is None:
        pytest.skip("oracle/_ref/reference_code.tar not staged (run __graft_entry__.build() where /root/reference exists)")
    return code


def _run(code, script, *args, timeout=900):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, os.path.join(ROOT, "tests", "harness")])
    t0 = time.time()
    r = subprocess.run([sys.executable, script, *args], cwd=code, env=env, capture_output=True, text=True, timeout=timeout)
    return r, time.time() - t0


@pytest.mark.parametrize("script,model,exp", [
    ("train_weakly_supervised_pCE_GatedCRFLoss_2D.py", "unet", "ACDC_pCE_GatedCRFLoss"),
    ("train_weakly_supervised_segmentation_pCE_ours_proposed.py", "unet_cct", "ACDC_pCE_ours"),
    ("train_weakly_supervised_pCE_MumfordShah_Loss_2D.py", "unet", "ACDC_pCE_MS"),
])
def test_reference_script_runs_unchanged(tmp_path, script, model, exp):
    code = _stage(tmp_path)
    r, dt = _run(code, script, "--root_path", "synthetic:30", "--model", model, "--max_iterations", "6", "--batch_size", "4",
                 "--exp", exp, "--sup_type", "scribble")
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    its = [int(m.group(1)) for m in re.finditer(r"iteration (\d+) : loss : ([-+0-9.eE]+)", r.stdout + r.stderr)]
    assert its[-1] == 6 and len(its) == 6, tail
    losses = [float(m.group(2)) for m in re.finditer(r"iteration (\d+) : loss : ([-+0-9.eE]+)", r.stdout + r.stderr)]
    assert all(l == l and abs(l) < 1e4 for l in losses), losses
    # the script wrote its snapshot / log where it always does (../model/<exp>_<fold>/<sup_type>/)
    assert os.path.exists(os.path.join(os.path.dirname(code), "model", f"{exp}_fold1", "scribble", "log.txt"))


def test_script_mode_throughput_and_validation(tmp_path):
    """train_weakly_supervised_pCE_GatedCRFLoss_2D.py with its validation pass (every 200 iterations, val_2D.test_single_volume over
    the fold's 20 test volumes) at batch 16: reports the images/s a user of the reference's own entry point sees."""
    code = _stage(tmp_path)
    r, dt = _run(code, "train_weakly_supervised_pCE_GatedCRFLoss_2D.py", "--root_path", "synthetic:40", "--model", "unet",
                 "--max_iterations", "200", "--batch_size", "16", "--sup_type", "scribble", timeout=1500)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "mean_dice" in out, out[-2000:]
    stamps = re.findall(r"\[(\d\d):(\d\d):(\d\d)\.(\d+)\] iteration (\d+) :", open(os.path.join(os.path.dirname(code), "model", "ACDC_pCE_GatedCRFLoss_fold1", "scribble", "log.txt")).read())
    t = {int(s[4]): int(s[0]) * 3600 + int(s[1]) * 60 + int(s[2]) + int(s[3]) / 1000.0 for s in stamps}
    if 50 in t and 190 in t and t[190] > t[50]:
        print(f"script mode (unchanged train script, DataLoader with 8 host workers, torch SGD / CE): {140 * 16 / (t[190] - t[50]):.0f} images/s at batch 16")
