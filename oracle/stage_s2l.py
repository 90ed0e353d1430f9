"""Stage the reference's UNMODIFIED code/train_s2l.py under oracle/_ref/s2l/ (git-ignored build output that travels with the tree,
like build_ref.py's archive) for tests/test_gpu_s2l.py, which runs it on top of dropin/.  A no-op where the reference is absent.

    python oracle/stage_s2l.py            # __graft_entry__.build() calls it
"""
import hashlib
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/code/train_s2l.py"
OUT = os.path.join(HERE, "_ref", "s2l")
DST = os.path.join(OUT, "train_s2l.py")


def build():
    """-> True when a staged copy exists afterwards"""
    if os.path.exists(SRC):
        os.makedirs(OUT, exist_ok=True)
        shutil.copyfile(SRC, DST)
        with open(DST + ".sha256", "w") as f:
            f.write(hashlib.sha256(open(SRC, "rb").read()).hexdigest())
    return os.path.exists(DST)


def extract(code_dir):
    """copy the staged script into an extracted reference code/ directory; False when nothing is staged"""
    if not os.path.exists(DST):
        return False
    data = open(DST, "rb").read()
    assert hashlib.sha256(data).hexdigest() == open(DST + ".sha256").read().strip(), "staged train_s2l.py was modified"
    with open(os.path.join(code_dir, "train_s2l.py"), "wb") as f:
        f.write(data)
    return True


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
