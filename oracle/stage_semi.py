"""Stage the reference's UNMODIFIED semi-supervised scripts that the build_ref.py archive lacks, plus networks/discriminator.py, under
oracle/_ref/semi/ (git-ignored build output that travels with the tree, like stage_s2l.py's copy).  tests/test_gpu_semi_scripts.py runs
the scripts on top of dropin/; profiles/discriminator.py times the reference class on cuDNN.  A no-op where the reference is absent.

    python oracle/stage_semi.py           # __graft_entry__.build() calls it
"""
import hashlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/code"
OUT = os.path.join(HERE, "_ref", "semi")
FILES = ("train_mean_teacher_2D.py", "train_entropy_minimization_2D.py", "train_partially_fully_supervised.py",
         "train_deep_adversarial_network_2D.py", "networks/discriminator.py")


def _staged(rel):
    return os.path.join(OUT, rel.replace("/", "__"))


def build():
    """-> True when staged copies of every file exist afterwards"""
    for rel in FILES:
        src = os.path.join(REF, rel)
        if os.path.exists(src):
            os.makedirs(OUT, exist_ok=True)
            data = open(src, "rb").read()
            with open(_staged(rel), "wb") as f:
                f.write(data)
            with open(_staged(rel) + ".sha256", "w") as f:
                f.write(hashlib.sha256(data).hexdigest())
    return all(os.path.exists(_staged(r)) for r in FILES)


def read(rel):
    """bytes of a staged file, checked against the digest written at staging time; None when nothing is staged"""
    if not os.path.exists(_staged(rel)):
        return None
    data = open(_staged(rel), "rb").read()
    assert hashlib.sha256(data).hexdigest() == open(_staged(rel) + ".sha256").read().strip(), f"staged {rel} was modified"
    return data


def extract(code_dir):
    """copy the staged scripts into an extracted reference code/ directory; False when nothing is staged"""
    if not all(os.path.exists(_staged(r)) for r in FILES):
        return False
    for rel in FILES:
        if rel.endswith(".py") and "/" not in rel:
            with open(os.path.join(code_dir, rel), "wb") as f:
                f.write(read(rel))
    return True


def load_reference_discriminator():
    """the staged reference networks/discriminator.py as a module (for the cuDNN comparison); None when nothing is staged"""
    data = read("networks/discriminator.py")
    if data is None:
        return None
    import types
    mod = types.ModuleType("reference_discriminator")
    exec(compile(data, "reference/networks/discriminator.py", "exec"), mod.__dict__)
    return mod


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
