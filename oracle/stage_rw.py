"""Stage the reference's UNMODIFIED code/train_fully_supervised_2D.py and code/train_weakly_supervised_pCE_random_walker_2D.py under
oracle/_ref/rw/ (git-ignored build output that travels with the tree, like stage_s2l.py's copy) for tests/test_gpu_random_walker.py,
which runs them on top of dropin/.  A no-op where the reference is absent.

    python oracle/stage_rw.py             # __graft_entry__.build() calls it
"""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/code"
OUT = os.path.join(HERE, "_ref", "rw")
SCRIPTS = ("train_fully_supervised_2D.py", "train_weakly_supervised_pCE_random_walker_2D.py")


def build():
    """-> True when staged copies of both scripts exist afterwards"""
    for name in SCRIPTS:
        src = os.path.join(REF, name)
        if os.path.exists(src):
            os.makedirs(OUT, exist_ok=True)
            shutil.copyfile(src, os.path.join(OUT, name))
            with open(os.path.join(OUT, name + ".sha256"), "w") as f:
                f.write(hashlib.sha256(open(src, "rb").read()).hexdigest())
    return all(os.path.exists(os.path.join(OUT, n)) for n in SCRIPTS)


def extract(code_dir):
    """copy the staged scripts into an extracted reference code/ directory; False when nothing is staged"""
    if not all(os.path.exists(os.path.join(OUT, n)) for n in SCRIPTS):
        return False
    for name in SCRIPTS:
        data = open(os.path.join(OUT, name), "rb").read()
        assert hashlib.sha256(data).hexdigest() == open(os.path.join(OUT, name + ".sha256")).read().strip(), f"staged {name} was modified"
        with open(os.path.join(code_dir, name), "wb") as f:
            f.write(data)
    return True


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
