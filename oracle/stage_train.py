"""Stage the reference's UNMODIFIED train_weakly_supervised_pCE_Inter&Intra_Class_2D.py -- the one training script with a native
recipe (wsl4mis_b200/train.py) that no other recipe stages -- under oracle/_ref/train/ (git-ignored build output that travels with
the tree, like stage_semi.py's copies).  tests/test_train_cpu.py compares every recipe's flags with the staged scripts' parsers.
A no-op where the reference is absent.

    python oracle/stage_train.py          # __graft_entry__.build() calls it
"""
import hashlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/code"
OUT = os.path.join(HERE, "_ref", "train")
FILES = ("train_weakly_supervised_pCE_Inter&Intra_Class_2D.py",)


def build():
    """-> True when a staged copy of every file exists afterwards"""
    for rel in FILES:
        src = os.path.join(REF, rel)
        if os.path.exists(src):
            os.makedirs(OUT, exist_ok=True)
            data = open(src, "rb").read()
            with open(os.path.join(OUT, rel), "wb") as f:
                f.write(data)
            with open(os.path.join(OUT, rel) + ".sha256", "w") as f:
                f.write(hashlib.sha256(data).hexdigest())
    return all(os.path.exists(os.path.join(OUT, r)) for r in FILES)


def read(rel):
    """source bytes of a staged file, checked against the digest written at staging time; None when nothing is staged"""
    path = os.path.join(OUT, rel)
    if not os.path.exists(path):
        return None
    data = open(path, "rb").read()
    assert hashlib.sha256(data).hexdigest() == open(path + ".sha256").read().strip(), f"staged {rel} was modified"
    return data


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
