"""Scribble2Label host side: the CPU restatement of RandomGenerator_s2l and the drop-in's host transform against the reference's own
output (tests/golden/s2l_augment.npz), TwoStreamBatchSampler and BaseDataSets_s2l."""
import os
import random

import numpy as np
import pytest

import s2l_oracle as S
from wsl4mis_b200.dataloaders.dataset import BaseDataSets_s2l, RandomGenerator_s2l, TwoStreamBatchSampler


def _fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "s2l_augment.npz"))


def test_oracle_transform_matches_reference_fixture(golden_dir):
    z = _fixture(golden_dir)
    hw = tuple(int(v) for v in z["out_hw"])
    for i in range(int(z["n"])):
        random.seed(int(z["seed"]) + i)
        np.random.seed(int(z["seed"]) + i)
        img, mask, scr, wgt = S.transform(*(z[f"in{i}_{k}"] for k in ("image", "mask", "scribble", "weight")), hw)
        assert np.array_equal(img, z[f"out{i}_image"][0]) and np.array_equal(mask, z[f"out{i}_mask"]), i
        assert np.array_equal(scr, z[f"out{i}_scribble"]) and np.array_equal(wgt, z[f"out{i}_weight"]), i


def test_host_transform_matches_reference_fixture(golden_dir):
    z = _fixture(golden_dir)
    gen = RandomGenerator_s2l([int(v) for v in z["out_hw"]])
    for i in range(int(z["n"])):
        random.seed(int(z["seed"]) + i)
        np.random.seed(int(z["seed"]) + i)
        s = gen({k: z[f"in{i}_{k}"] for k in ("image", "mask", "scribble", "weight")})
        for k in ("image", "mask", "scribble", "weight"):
            assert np.array_equal(s[k].numpy(), z[f"out{i}_{k}"]), (i, k)


def test_two_stream_batch_sampler():
    np.random.seed(0)
    prim, sec = list(range(10)), list(range(10, 17))
    smp = TwoStreamBatchSampler(prim, sec, 5, 2)
    batches = list(smp)
    assert len(smp) == len(batches) == 3
    assert all(len(b) == 5 and all(i in prim for i in b[:3]) and all(i in sec for i in b[3:]) for b in batches)
    seen = [i for b in batches for i in b[:3]]
    assert len(set(seen)) == 9                                       # every primary index at most once per epoch
    tail = [i for b in batches for i in b[3:]]
    assert sorted(tail[:6]) == sorted(set(tail[:6])) and set(tail[:6]) <= set(sec)
    with pytest.raises(ValueError):
        TwoStreamBatchSampler(prim, sec, 5, 0)


def test_base_datasets_s2l_shapes_and_keys():
    ds = BaseDataSets_s2l(base_dir="synthetic:30", fold="fold1", transform=RandomGenerator_s2l([64, 64]))
    assert len(ds) > 0 and len(ds.images) == len(ds)
    rec = ds.images[0]
    assert set(rec) == {"id", "image", "mask", "scribble", "weight"}
    h, w = rec["mask"].shape
    assert rec["image"].shape == rec["scribble"].shape == (h, w) and rec["weight"].shape == (h, w, 4)
    assert rec["weight"].dtype == np.float32 and not rec["weight"].any()
    assert set(np.unique(rec["scribble"])) <= {0, 1, 2, 3, 4} and (rec["scribble"] == 4).mean() > 0.5
    s = ds[0]
    assert set(s) == {"image", "mask", "scribble", "weight", "id"}
    assert tuple(s["image"].shape) == (1, 64, 64) and tuple(s["scribble"].shape) == (64, 64) and tuple(s["weight"].shape) == (64, 64, 4)
    assert s["id"] == rec["id"]
