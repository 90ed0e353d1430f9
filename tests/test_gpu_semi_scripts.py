"""The reference's five semi-supervised scripts, UNCHANGED, on the H100 modules: mean teacher, entropy minimisation, uncertainty-aware
mean teacher, partially / fully supervised and the adversarial network (DAN).  All of them import dataloaders.dataset_semi and
networks.discriminator; through dropin/ both resolve to this repository (the BaseDataSets split on the synthetic stand-in, the
tensor-core FCDiscriminator).  The scripts come from the staged copies (oracle/build_ref.py's archive and oracle/stage_semi.py)."""
import glob
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stage(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    try:
        import build_ref
        import stage_semi
        code = build_ref.extract(str(tmp_path))
        if code is None or not stage_semi.extract(code):
            pytest.skip("reference scripts not staged (run __graft_entry__.build() where the reference exists)")
    finally:
        sys.path.pop(0)
    return code


def _env():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, os.path.join(ROOT, "tests", "harness")])
    return env


def test_semi_modules_resolve_into_dropin(tmp_path):
    code = _stage(tmp_path)
    probe = ("import dataloaders.dataset_semi as d, networks.discriminator as n\n"
             "print(d.__file__); print(n.__file__); print(d.BaseDataSets.__module__, n.FCDiscriminator.__module__)")
    r = subprocess.run([sys.executable, "-c", probe], cwd=code, env=_env(), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = r.stdout.split("\n")
    dropin = os.path.realpath(os.path.join(ROOT, "dropin"))
    assert os.path.realpath(lines[0]).startswith(dropin) and os.path.realpath(lines[1]).startswith(dropin), lines
    assert lines[2].split() == ["wsl4mis_b200.dataloaders.dataset_semi", "wsl4mis_b200.networks.discriminator"], lines


@pytest.mark.parametrize("script", ["train_mean_teacher_2D.py", "train_entropy_minimization_2D.py",
                                    "train_uncertainty_aware_mean_teacher_2D.py", "train_partially_fully_supervised.py",
                                    "train_deep_adversarial_network_2D.py"])
def test_semi_script_runs_unchanged(tmp_path, script):
    code = _stage(tmp_path)
    r = subprocess.run([sys.executable, script, "--root_path", "synthetic:40", "--max_iterations", "6", "--batch_size", "4"],
                       cwd=code, env=_env(), capture_output=True, text=True, timeout=1200)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    found = re.findall(r"iteration (\d+) : loss : ([-+0-9.eEnaif]+)", out)
    assert [int(i) for i, _ in found] == [1, 2, 3, 4, 5, 6], out[-3000:]
    losses = [float(v) for _, v in found]
    assert all(l == l and abs(l) < 1e4 for l in losses), losses
    logs = glob.glob(os.path.join(os.path.dirname(code), "model", "**", "log.txt"), recursive=True)
    assert logs and "iteration 6 : loss" in open(logs[0]).read(), logs
