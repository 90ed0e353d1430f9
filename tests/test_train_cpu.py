"""The native trainer's host side (wsl4mis_b200/train.py): every recipe's flags against the staged script's own parser, the loop's
bookkeeping with a fake step, loader and validator, the two-stream feed's replay of the labelled batches, and the error for a
script without a recipe."""
import argparse
import ast
import hashlib
import os
import re

import pytest
import torch

import wsl4mis_b200.train as T

import build_ref
import stage_rw
import stage_s2l
import stage_semi
import stage_train

WSS_ARGV = ["--fold", "fold1", "--num_classes", "4", "--root_path", "../data/ACDC", "--exp", "ACDC/X", "--max_iterations", "60000",
            "--batch_size", "12"]           # the pattern of every line of train_wss.sh / train_semi.sh


def _checked(path):
    data = open(path, "rb").read()
    assert hashlib.sha256(data).hexdigest() == open(path + ".sha256").read().strip(), f"staged {path} was modified"
    return data


_code_dir = []


def _script_source(name):
    """the unmodified script from whichever build recipe stages it; None when nothing is staged"""
    for data in (stage_train.read(name), stage_semi.read(name)):
        if data is not None:
            return data.decode()
    for path in (os.path.join(stage_rw.OUT, name), stage_s2l.DST if name == "train_s2l.py" else None):
        if path and os.path.exists(path):
            return _checked(path).decode()
    if not _code_dir:
        _code_dir.append(build_ref.extract())
    if _code_dir[0] and os.path.exists(os.path.join(_code_dir[0], name)):
        return open(os.path.join(_code_dir[0], name)).read()
    return None


def _script_parser(name):
    """the script's parser, executed from its source up to parse_args (its imports need packages this image lacks)"""
    src = _script_source(name)
    if src is None:
        pytest.skip("reference training scripts not staged (run __graft_entry__.build() where the reference exists)")
    keep = [n for n in ast.parse(src).body if ast.unparse(n).startswith("parser")]
    ns = {"argparse": argparse}
    exec(compile(ast.Module(body=keep, type_ignores=[]), name, "exec"), ns)
    return ns["parser"]


def _actions(p):
    return [(a.dest, a.option_strings, a.type, a.default) for a in p._actions if a.dest != "help"]


@pytest.mark.parametrize("script", sorted(T.RECIPES))
def test_flags_match_the_staged_script(script):
    ref, ours = _script_parser(script), T.parser_for(script)
    assert _actions(ours) == _actions(ref)
    for argv in ([], WSS_ARGV):
        assert str(ours.parse_args(argv)) == str(ref.parse_args(argv))
    name, args, precision = T.parse([script] + WSS_ARGV + ["--precision", "fp16x3"])
    assert (name, precision) == (script, "fp16x3") and str(args) == str(ref.parse_args(WSS_ARGV))
    assert T.parse(["/some/dir/" + script])[2] == "bf16"


def test_sixteen_recipes_and_no_scribblevc():
    assert len(T.RECIPES) == 16 and not any("scribblevc" in s for s in T.RECIPES)


def test_unknown_script_lists_the_supported_ones():
    with pytest.raises(ValueError) as e:
        T.parse(["train_ACDC_scribblevc.py"])
    for s in T.RECIPES:
        assert s in str(e.value)
    with pytest.raises(ValueError):
        T.parser_for("train_nothing.py")


def test_snapshot_path():
    _, args, _ = T.parse(["train_mean_teacher_2D.py", "--exp", "ACDC_Semi/MT", "--fold", "fold3"])
    assert T.snapshot_path(args) == "../model/ACDC_Semi/MT_fold3/label"


# ---------------------------------------------------------------- the loop with fakes
class FakeStep:
    def __init__(self):
        self.calls = 0
        self.loss_parts = {}

    def __call__(self, x):
        self.calls += 1
        self.loss_parts = {"ce": torch.tensor(x * 0.5)}
        return torch.tensor(float(x))


class FakeValidator:
    """scores one volume of one class; the dice of validation k is dice[k]"""

    def __init__(self, dice):
        self.dice, self.calls = list(dice), []

    def score(self, model, classes):
        d = self.dice[len(self.calls)]
        self.calls.append(model.training)
        return [[(d, 2.0 * d)] * (classes - 1), [(d, 2.0 * d)] * (classes - 1)]


def _run(tmp_path, max_iterations, per_epoch, dice, log_fmt=T._LOG2):
    recipe = T.Recipe((), "single", None, log_fmt, (("info/loss_ce", T._part("ce")),))
    args = argparse.Namespace(max_iterations=max_iterations, base_lr=0.01, num_classes=4, model="unet")
    model = torch.nn.Linear(2, 2)
    step, val, lines = FakeStep(), FakeValidator(dice), []
    counter = iter(range(1, 10 ** 6))
    batches = lambda: ((next(counter),) for _ in range(per_epoch))
    out = T.Trainer(args, recipe, model, step, batches, per_epoch, val, str(tmp_path), lines.append, device="cpu").run()
    assert out == "Training Finished!"
    return step, val, lines


def test_loop_bookkeeping(tmp_path):
    dice = [0.5, 0.4, 0.6, 0.6, 0.61234567]
    step, val, lines = _run(tmp_path, 1050, 7, dice)
    assert lines[0] == "7 iterations per epoch"
    assert step.calls == 1050                        # max_epoch = 1050 // 7 + 1 = 151 epochs; stops mid-epoch at max_iterations
    it_lines = [l for l in lines if re.fullmatch(r"iteration \d+ : loss : [\d.]+, loss_ce: [\d.]+", l)]
    assert [int(l.split()[1]) for l in it_lines] == list(range(1, 1051))
    assert it_lines[9] == "iteration 10 : loss : %f, loss_ce: %f" % (10.0, 5.0)
    val_lines = [l for l in lines if "mean_dice" in l]
    assert [int(l.split()[1]) for l in val_lines] == [200, 400, 600, 800, 1000] and len(val.calls) == 5
    assert val_lines[0] == "iteration 200 : mean_dice : %f mean_hd95 : %f" % (0.5, 1.0)
    # every iteration line up to N comes before the validation line of N, and none after it
    for l in val_lines:
        n, k = int(l.split()[1]), lines.index(l)
        assert lines[k - 1] == it_lines[n - 1] and lines[k + 1] == it_lines[n]
    # best model: strict improvement only (0.6 again at 800 does not save), file name rounded to 4 digits
    files = sorted(os.listdir(tmp_path))
    assert files == sorted(["iter_200_dice_0.5.pth", "iter_600_dice_0.6.pth", "iter_1000_dice_0.6123.pth", "unet_best_model.pth"])
    best = torch.load(os.path.join(tmp_path, "unet_best_model.pth"))
    assert set(best) == {"weight", "bias"} and all(v.dtype == torch.float32 for v in best.values())


def test_checkpoints_every_3000(tmp_path):
    step, val, lines = _run(tmp_path, 6100, 500, [0.1 * (k % 3) for k in range(40)])
    saves = [l for l in lines if l.startswith("save model to")]
    assert saves == ["save model to " + os.path.join(str(tmp_path), "iter_3000.pth"),
                     "save model to " + os.path.join(str(tmp_path), "iter_6000.pth")]
    k = lines.index(saves[0])
    assert lines[k - 1] == "iteration 3000 : mean_dice : %f mean_hd95 : %f" % (0.2, 0.4)     # the 15th validation
    assert lines[k + 1].startswith("iteration 3001 : loss")
    assert step.calls == 6100 and lines[-1].startswith("iteration 6100 : loss")
    assert os.path.exists(os.path.join(tmp_path, "iter_6000.pth"))


def test_script_without_iteration_lines(tmp_path):
    step, val, lines = _run(tmp_path, 450, 100, [0.2, 0.3], log_fmt=None)
    assert lines == ["100 iterations per epoch", "iteration 200 : mean_dice : %f mean_hd95 : %f" % (0.2, 0.4),
                     "iteration 400 : mean_dice : %f mean_hd95 : %f" % (0.3, 0.6)]


class Pass:
    """a loader whose every pass yields fresh batches, numbered by pass"""

    def __init__(self, n, tag):
        self.n, self.tag, self.passes = n, tag, 0

    def __len__(self):
        return self.n

    def __iter__(self):
        self.passes += 1
        p = self.passes
        return iter([{"image": (self.tag, p, i), "label": (self.tag, p, i)} for i in range(self.n)])


def test_two_stream_replays_the_labelled_pass():
    ll, lu = Pass(3, "l"), Pass(7, "u")
    epoch = list(T.two_stream(ll, lu))
    assert len(epoch) == 7 and ll.passes == 1           # cycle keeps the first pass and replays it
    assert [b[0] for b in epoch] == [("l", 1, i % 3) for i in range(7)]
    assert [b[2] for b in epoch] == [("u", 1, i) for i in range(7)]
    epoch2 = list(T.two_stream(ll, lu))
    assert [b[0] for b in epoch2] == [("l", 2, i % 3) for i in range(7)]     # a fresh cycle per epoch
    assert all(len(b) == 2 for b in T.two_stream(Pass(3, "l"), Pass(4, "u"), labelled_only=True))
