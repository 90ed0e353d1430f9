"""Drop-in for ``dataloaders/dataset_semi.py`` of the reference, which the five semi-supervised scripts import
(train_mean_teacher_2D.py:25-26, train_deep_adversarial_network_2D.py:25-26, ...).

``BaseDataSets`` adds the labelled / unlabelled split of dataset_semi.py:17-60 to `dataset.BaseDataSets` (same sources: an ACDC
directory with h5py, or ``'synthetic[:<patients>]'``); ``RandomGenerator`` and ``TwoStreamBatchSampler`` are the ones of `dataset`."""
from .dataset import BaseDataSets as _BaseDataSets
from .dataset import RandomGenerator, TwoStreamBatchSampler, fold_ids  # noqa: F401

LABELED_IDS = ["patient{:0>3}".format(10 * i) for i in range(1, 11)]      # dataset_semi.py:27-28


class BaseDataSets(_BaseDataSets):
    """``BaseDataSets(base_dir, num, labeled_type, split, transform, fold, sup_type)`` (dataset_semi.py:17-60).

    split='train': labeled_type 'labeled' keeps the slices of patients 010, 020, ..., 100 that lie in the fold's training set, any
    other value the slices of the fold's remaining training patients.  split='val' yields the fold's test volumes.  ``num`` is
    accepted and ignored, as in the reference (:59-60).  Every sample carries ``idx`` = the case's patient id."""

    def __init__(self, base_dir=None, num=4, labeled_type="labeled", split='train', transform=None, fold="fold1", sup_type="label"):
        super().__init__(base_dir, split, transform, fold, sup_type)
        self.num, self.labeled_type = num, labeled_type
        if split == "train":
            train_ids, _ = fold_ids(fold)
            labeled = [p for p in LABELED_IDS if p in train_ids]
            keep = set(labeled) if labeled_type == "labeled" else set(train_ids) - set(labeled)
            self.sample_list = [c for c in self.sample_list if c.split("_")[0] in keep]
