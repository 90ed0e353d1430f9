"""Writes tests/golden/s2l_augment.npz: the reference's OWN RandomGenerator_s2l (code/dataloaders/dataset_s2l.py:126-153) on seeded
ragged slices with random prediction memories.  Run where /root/reference exists:

    python oracle/make_golden_s2l.py

dataset_s2l.py imports h5py and matplotlib at module level without using them here: tests/harness supplies stand-ins.
Sample i is transformed after random.seed(SEED + i) and np.random.seed(SEED + i), so a test replays the same draws."""
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference/code"
SEED, OUT_HW = 500, (48, 40)
SHAPES = [(40, 36), (36, 44), (50, 30), (33, 47), (44, 44), (31, 38), (45, 35), (38, 50), (29, 41), (47, 32), (36, 36), (42, 39)]


def make():
    sys.path[:0] = [REF, os.path.join(ROOT, "tests", "harness")]
    from dataloaders.dataset_s2l import RandomGenerator_s2l
    rs = np.random.RandomState(77)
    gen = RandomGenerator_s2l(list(OUT_HW))
    out = {"seed": np.array(SEED), "out_hw": np.array(OUT_HW), "n": np.array(len(SHAPES))}
    for i, (h, w) in enumerate(SHAPES):
        img = (rs.randint(0, 256, (h, w)) / 255.0).astype(np.float32)
        mask = rs.randint(0, 4, (h, w)).astype(np.uint8)
        scr = np.where(rs.rand(h, w) < 0.3, mask, 4).astype(np.uint8)
        wgt = (rs.randint(0, 16, (h, w, 4)) / 16.0).astype(np.float32)
        random.seed(SEED + i)
        np.random.seed(SEED + i)
        s = gen({"image": img, "mask": mask, "scribble": scr, "weight": wgt})
        for k, v in (("image", img), ("mask", mask), ("scribble", scr), ("weight", wgt)):
            out[f"in{i}_{k}"] = v
        for k in ("image", "mask", "scribble", "weight"):
            out[f"out{i}_{k}"] = s[k].numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "s2l_augment.npz"), **out)


if __name__ == "__main__":
    make()
