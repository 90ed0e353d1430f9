"""Drop-in for ``dataloaders/dataset.py`` of the reference (modelled on the working ``dataset_semi.py:17-171``; SURVEY F6).

The reference decodes one h5 slice per sample in DataLoader workers and augments it with numpy/scipy
(``RandomGenerator``: rot90+flip | rotate(order 0), then ``zoom(order 0)`` to the patch size).  At ~10 k images/s per GPU
eight such workers cannot feed the step, so here the 1 902 training slices (about 0.5 GB) live on the GPU in a ragged store
and a whole batch is augmented by ONE kernel (``wsl_augment_batch``).  All stages are nearest-neighbour, i.e. exact index
maps, and the random parameters are drawn on the host from the same ``random`` / ``numpy.random`` streams in the same
order as the reference's transform, so a batch is bit-identical to what the reference pipeline produces for the same
draws (tests/test_gpu_data.py).
"""
import collections
import os
import random

import numpy as np
import torch

from .._lib import LIB, call

_SAMPLE = np.dtype([("off", "<i8"), ("h", "<i4"), ("w", "<i4"), ("mode", "<i4"), ("k", "<i4"), ("axis", "<i4"),
                    ("lab_cval", "<i4"), ("m00", "<f8"), ("m01", "<f8"), ("m10", "<f8"), ("m11", "<f8"), ("o0", "<f8"),
                    ("o1", "<f8")], align=False)


def _rotation(angle, shape):
    """Matrix and offset of ``scipy.ndimage.rotate(..., reshape=False)`` (same float64 expressions as SciPy)."""
    try:
        from scipy import special
        c, s = special.cosdg(angle), special.sindg(angle)
    except ImportError:                                   # pragma: no cover - SciPy is a dependency of the reference too
        c, s = np.cos(np.deg2rad(angle)), np.sin(np.deg2rad(angle))
    rot = np.array([[c, s], [-s, c]])
    plane = np.asarray(shape)
    out_center = rot @ ((plane - 1) / 2)
    in_center = (plane - 1) / 2
    return rot, in_center - out_center


class RandomGenerator:
    """``RandomGenerator(output_size)`` of dataset_semi.py:146-171.  ``draw`` consumes ``random`` / ``np.random`` exactly like
    the reference's ``__call__`` (:155-163) and returns the augmentation parameters instead of applying them."""

    def __init__(self, output_size):
        self.output_size = tuple(int(v) for v in output_size)

    @staticmethod
    def draw(label_has_4, streams=None):
        """streams: (Python Random, numpy RandomState) to draw from instead of the global `random` / `np.random` (`rank_streams`)"""
        py, npr = (random, np.random) if streams is None else streams
        if py.random() > 0.5:
            k = int(npr.randint(0, 4))                    # random_rot_flip, :126-134
            axis = int(npr.randint(0, 2))
            return (1, k, axis, 0, 0)
        elif py.random() > 0.5:
            angle = int(npr.randint(-20, 20))             # random_rotate, :137-143
            return (2, 0, 0, angle, 4 if label_has_4 else 0)
        return (0, 0, 0, 0, 0)

    def __call__(self, sample):
        """Single-sample form with the reference's signature (numpy in, CPU tensors out).  Runs on the HOST: the scripts call
        it inside DataLoader worker processes (train_weakly_supervised_pCE_2D.py:72-73), where the GPU is off limits.  The
        batched GPU kernel (`SliceStore.augment`) produces bit-identical samples for the same draws (tests/test_gpu_data.py)."""
        image = np.asarray(sample["image"], dtype=np.float32)
        label = np.asarray(sample["label"]).astype(np.uint8)
        img, lab = apply_host(image, label, self.draw(bool((label == 4).any())), self.output_size)
        return {"image": torch.from_numpy(img).unsqueeze(0), "label": torch.from_numpy(lab)}


def rank_streams(seed, rank):
    """(random.Random, np.random.RandomState) of one data-parallel rank, seeded from (seed, rank): the ranks of one job draw
    different augmentation parameters for their shards, while the global streams, which the steps' own host draws use, stay
    identical on every rank"""
    ss = np.random.SeedSequence([int(seed), int(rank)])
    return random.Random(int(ss.generate_state(1, np.uint64)[0])), np.random.RandomState(ss.generate_state(4))


def apply_host(image, label, params, output_size):
    """One (mode, k, axis, angle, lab_cval) decision on host arrays with the reference's library calls: rot90 + flip
    (dataset_semi.py:126-134) | scipy rotate, order 0, label padded with lab_cval (:137-143); then zoom(order=0) to the
    patch size (:164-167)."""
    from scipy import ndimage
    mode, k, axis, angle, cval = params
    if mode == 1:
        image, label = np.flip(np.rot90(image, k), axis=axis), np.flip(np.rot90(label, k), axis=axis)
    elif mode == 2:
        image = ndimage.rotate(image, angle, order=0, reshape=False)
        label = ndimage.rotate(label, angle, order=0, reshape=False, mode="constant", cval=cval)
    fy, fx = output_size[0] / image.shape[0], output_size[1] / image.shape[1]
    image = ndimage.zoom(np.ascontiguousarray(image), (fy, fx), order=0)
    label = ndimage.zoom(np.ascontiguousarray(label), (fy, fx), order=0)
    return image.astype(np.float32), label.astype(np.uint8)


class RandomGenerator_s2l:
    """``RandomGenerator_s2l(output_size)`` of dataset_s2l.py:126-153, on the HOST for DataLoader workers: the draws of
    `RandomGenerator` (:132-137); image, mask, scribble and the [h,w,4] weight through the same rot90 / flip / rotate(order 0,
    cval 0 for every array -- the scribble's rotated-in corners become background, SURVEY F15) and zoom(order 0; factor 1 on the
    class axis).  `SliceStore.augment_s2l` produces the same samples on the GPU for the same draws."""

    def __init__(self, output_size):
        self.output_size = tuple(int(v) for v in output_size)

    def __call__(self, sample):
        params = RandomGenerator.draw(False)
        image = np.asarray(sample["image"], dtype=np.float32)
        img, mask = apply_host(image, np.asarray(sample["mask"]).astype(np.uint8), params, self.output_size)
        _, scr = apply_host(image, np.asarray(sample["scribble"]).astype(np.uint8), params, self.output_size)
        weight = np.asarray(sample["weight"], dtype=np.float32)
        wgt = np.stack([apply_host(weight[..., c], mask, params, self.output_size)[0] for c in range(weight.shape[2])], -1)
        return {"image": torch.from_numpy(img).unsqueeze(0), "mask": torch.from_numpy(mask), "scribble": torch.from_numpy(scr),
                "weight": torch.from_numpy(np.ascontiguousarray(wgt, dtype=np.float32))}


class SliceStore:
    """All training slices resident on the GPU: flat fp32 images, flat uint8 labels, per-slice offset / shape.

    With ``scribbles`` (Scribble2Label, dataset_s2l.py:34-46) the store also holds the scribble maps and the per-slice 4-class
    prediction memory, zero-initialised like :46, as ragged channels-last fp32 ([pixels, 4]) in two copies: ``weight_live``,
    which the ensemble refresh updates, and ``weight_epoch``, the snapshot training batches read (SURVEY F16)."""

    def __init__(self, images, labels, offs, shapes, has4, names, scribbles=None):
        self.images, self.labels = images, labels
        self.offs, self.shapes, self.has4, self.names = offs, shapes, has4, names
        assert LIB.load().wsl_augment_sample_bytes() == _SAMPLE.itemsize, "AugSample layout mismatch"
        self.scribbles = scribbles
        self.weight_live = self.weight_epoch = None
        if scribbles is not None:
            assert scribbles.numel() == images.numel()
            self.weight_live = torch.zeros(images.numel(), 4, dtype=torch.float32, device=images.device)
            self.weight_epoch = torch.zeros_like(self.weight_live)

    def weight(self, i, which="live"):
        """the [h, w, 4] prediction memory of slice i (a view)"""
        h, w = int(self.shapes[i, 0]), int(self.shapes[i, 1])
        mem = self.weight_live if which == "live" else self.weight_epoch
        return mem[self.offs[i]: self.offs[i] + h * w].view(h, w, 4)

    def __len__(self):
        return len(self.offs)

    @classmethod
    def from_arrays(cls, images, labels, names=None, device=None, scribbles=None):
        device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        assert len(images) == len(labels) and len(images) > 0
        shapes = np.array([im.shape for im in images], dtype=np.int32)
        for im, lb in zip(images, labels):
            assert im.ndim == 2 and im.shape == lb.shape, "slices are 2-D and image / label shapes agree"
        sizes = shapes[:, 0].astype(np.int64) * shapes[:, 1]
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        flat_i = np.concatenate([np.asarray(im, dtype=np.float32).ravel() for im in images])
        flat_l = np.concatenate([np.asarray(lb).astype(np.uint8).ravel() for lb in labels])
        has4 = np.array([bool((np.asarray(lb) == 4).any()) for lb in labels])
        names = list(names) if names is not None else [str(i) for i in range(len(images))]
        flat_s = None
        if scribbles is not None:
            assert len(scribbles) == len(images) and all(np.shape(sc) == im.shape for sc, im in zip(scribbles, images))
            flat_s = torch.from_numpy(np.concatenate([np.asarray(sc).astype(np.uint8).ravel() for sc in scribbles])).to(device)
        return cls(torch.from_numpy(flat_i).to(device), torch.from_numpy(flat_l).to(device), offs, shapes, has4, names, flat_s)

    @classmethod
    def from_h5_dir(cls, base_dir, cases, sup_type="scribble", device=None):
        """``ACDC_training_slices/<case>`` files with datasets 'image' and `sup_type` (dataset_semi.py:105-121)."""
        try:
            import h5py
        except ImportError as e:                          # no silent substitute: the caller must provide arrays
            raise ImportError("h5py is required to read the ACDC slice files; use SliceStore.from_arrays otherwise") from e
        ims, lbs = [], []
        for case in cases:
            with h5py.File(os.path.join(base_dir, "ACDC_training_slices", case), "r") as f:
                ims.append(f["image"][:])
                lbs.append(f[sup_type][:])
        return cls.from_arrays(ims, lbs, [c.split("_")[0] for c in cases], device)

    def table(self, indices, params):
        """AugSample rows (device, bytes) of the samples: slice ids and (mode, k, axis, angle, lab_cval) per sample."""
        B = len(indices)
        tab = np.zeros(B, dtype=_SAMPLE)
        for b, (i, (mode, k, axis, angle, cval)) in enumerate(zip(indices, params)):
            h, w = int(self.shapes[i, 0]), int(self.shapes[i, 1])
            row = tab[b]
            row["off"], row["h"], row["w"] = self.offs[i], h, w
            row["mode"], row["k"], row["axis"], row["lab_cval"] = mode, k, axis, cval
            if mode == 2:
                rot, off = _rotation(angle, (h, w))
                row["m00"], row["m01"], row["m10"], row["m11"] = rot[0, 0], rot[0, 1], rot[1, 0], rot[1, 1]
                row["o0"], row["o1"] = off[0], off[1]
        return torch.from_numpy(tab.view(np.uint8)).to(self.images.device, non_blocking=True)

    def augment(self, indices, params, output_size):
        """indices: slice ids; params: (mode, k, axis, angle, lab_cval) per sample -> (image [B,1,H,W] fp32, label [B,H,W] u8)."""
        B, dev = len(indices), self.images.device
        tab_d = self.table(indices, params)
        OH, OW = output_size
        img = torch.empty(B, 1, OH, OW, dtype=torch.float32, device=dev)
        lab = torch.empty(B, OH, OW, dtype=torch.uint8, device=dev)
        call("wsl_augment_batch", self.images, self.labels, tab_d, B, OH, OW, img, lab)
        return img, lab

    def augment_s2l(self, indices, params, output_size, which="epoch"):
        """RandomGenerator_s2l (dataset_s2l.py:126-153) for a batch: -> (image [B,1,H,W] fp32, scribble [B,H,W] u8,
        weight [B,H,W,4] fp32) gathered in one launch from the scribble store and the `which` ('epoch' | 'live') memory."""
        assert self.scribbles is not None, "this store has no scribbles / prediction memory (from_arrays(..., scribbles=))"
        B, dev = len(indices), self.images.device
        tab_d = self.table(indices, params)
        OH, OW = output_size
        img = torch.empty(B, 1, OH, OW, dtype=torch.float32, device=dev)
        scr = torch.empty(B, OH, OW, dtype=torch.uint8, device=dev)
        wgt = torch.empty(B, OH, OW, 4, dtype=torch.float32, device=dev)
        mem = self.weight_epoch if which == "epoch" else self.weight_live
        call("wsl_augment_batch_s2l", self.images, self.scribbles, mem, tab_d, B, OH, OW, img, scr, wgt)
        return img, scr, wgt


def fold_ids(fold):
    """ACDC five-fold split of the reference (dataset_semi.py:62-101): fold k tests on patients 20(k-1)+1 .. 20k."""
    k = {"fold1": 1, "fold2": 2, "fold3": 3, "fold4": 4, "fold5": 5}.get(fold)
    if k is None:
        raise ValueError(f"unknown fold {fold!r} (fold1..fold5)")
    test = ["patient{:0>3}".format(i) for i in range(20 * (k - 1) + 1, 20 * k + 1)]
    train = ["patient{:0>3}".format(i) for i in range(1, 101) if "patient{:0>3}".format(i) not in test]
    return train, test


def synthetic_acdc(n_patients=100, seed=2022, slices=(6, 11)):
    """ACDC-shaped synthetic cases for runs without the dataset (no h5py / no files on the box): per patient a short-axis stack
    of `slices` ragged 2-D slices, image in [0, 1] (the reference min-max normalises, acdc_data_processing.py:44-45), dense
    labels 0..3 as nested structures and a scribble map with 4 = unlabelled (~3 % labelled pixels).  Deterministic in `seed`."""
    rs = np.random.RandomState(seed)
    shapes = [(256, 216), (216, 256), (224, 154), (232, 256), (174, 208)]
    cases = {}
    for pid in range(1, n_patients + 1):
        h, w = shapes[rs.randint(len(shapes))]
        d = int(rs.randint(slices[0], slices[1]))
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        cy, cx = h * (0.4 + 0.2 * rs.rand()), w * (0.4 + 0.2 * rs.rand())
        vol_i, vol_l, vol_s = [], [], []
        for z in range(d):
            r0 = min(h, w) * (0.10 + 0.04 * np.sin(z / max(d - 1, 1) * np.pi) + 0.02 * rs.rand())
            rr = np.sqrt((yy - cy) ** 2 + ((xx - cx) * (0.9 + 0.2 * rs.rand())) ** 2)
            lab = np.zeros((h, w), np.uint8)
            lab[rr < 2.2 * r0] = 1
            lab[rr < 1.6 * r0] = 2
            lab[rr < 1.0 * r0] = 3
            img = 0.15 + 0.2 * lab.astype(np.float32) + 0.08 * rs.randn(h, w).astype(np.float32)
            img = (img - img.min()) / (img.max() - img.min())
            scr = np.full((h, w), 4, np.uint8)
            keep = rs.rand(h, w) < 0.03
            scr[keep] = lab[keep]
            vol_i.append(img.astype(np.float32))
            vol_l.append(lab)
            vol_s.append(scr)
        cases["patient{:0>3}".format(pid)] = (np.stack(vol_i), np.stack(vol_l), np.stack(vol_s))
    return cases


def synthetic_spacing(patient, seed=2022):
    """Voxel spacing (x, y, z) in mm of a `synthetic_acdc` case, in SimpleITK's GetSpacing order: slice distance from
    {5, 6.5, 10}, each in-plane axis from {1.25, 1.37, 1.5625} (ACDC's range).  A stream of its own keyed by patient, so the
    draws of `synthetic_acdc` stay as they are.  The two in-plane axes are drawn separately so that a mix-up of x and y shows."""
    pid = int(str(patient).replace("patient", "").split("_")[0])
    rs = np.random.RandomState([seed, pid])
    inplane = (1.25, 1.37, 1.5625)
    return float(inplane[rs.randint(3)]), float(inplane[rs.randint(3)]), float((5.0, 6.5, 10.0)[rs.randint(3)])


class BaseDataSets(torch.utils.data.Dataset):
    """``BaseDataSets(base_dir, split, transform, fold, sup_type)`` as every WSS script constructs it
    (train_weakly_supervised_pCE_GatedCRFLoss_2D.py:75-80; the class the scripts need is the one in dataset_semi.py:17-125 --
    the shipped dataloaders/dataset.py lacks fold= / sup_type=, SURVEY F6).

    split='train': one sample per slice of the fold's training patients, ``{'image': f32 [1,H,W], 'label': u8 [H,W], 'idx'}``
    after `transform`; split='val': one sample per volume of the fold's test patients, ``{'image': [D,h,w], 'label': [D,h,w],
    'idx'}``.  Samples are produced on the HOST (numpy): the scripts iterate this object inside ``DataLoader(num_workers=8)``
    worker processes, which must not touch the GPU.  ``to_slice_store()`` hands the same slices to the resident GPU pipeline
    (`SliceStore` / `GpuLoader`), which is what keeps up with the training step.

    base_dir: the ACDC directory (``ACDC_training_slices/*.h5`` with datasets image / label / scribble and
    ``ACDC_training_volumes/*.h5``; needs h5py), or ``'synthetic'`` / ``'synthetic:<patients>'`` for the deterministic
    ACDC-shaped generator above (what the tests and benchmarks use: the GPU boxes have neither h5py nor the data).

    sup_type='random_walker' (train_weakly_supervised_pCE_random_walker_2D.py): slices without a 'random_walker' dataset get the
    random-walker pseudo labels of their scribbles, computed on the GPU at construction (needs a CUDA device; no fallback)."""

    def __init__(self, base_dir=None, split='train', transform=None, fold="fold1", sup_type="label", num=None):
        self._base_dir, self.split, self.transform, self.sup_type = base_dir, split, transform, sup_type
        train_ids, test_ids = fold_ids(fold)
        ids = set(train_ids if split == "train" else test_ids)
        if split not in ("train", "val"):
            raise ValueError(f"split must be 'train' or 'val' (got {split!r})")
        self._synthetic = None
        if base_dir is None or str(base_dir).startswith("synthetic"):
            n = int(str(base_dir).split(":")[1]) if base_dir is not None and ":" in str(base_dir) else 100
            cases = synthetic_acdc(n)
            self._synthetic = cases
            if split == "train":
                self.sample_list = [f"{pid}_frame01_slice_{z}.h5" for pid in sorted(cases) if pid in ids for z in range(cases[pid][0].shape[0])]
            else:
                self.sample_list = [f"{pid}_frame01.h5" for pid in sorted(cases) if pid in ids]
        else:
            sub = "ACDC_training_slices" if split == "train" else "ACDC_training_volumes"
            names = sorted(os.listdir(os.path.join(base_dir, sub)))
            self.sample_list = [f for f in names if f.split("_")[0] in ids]
        if num is not None and split == "train":
            self.sample_list = self.sample_list[:num]
        self._rw = {}
        if sup_type == "random_walker" and split == "train":
            self._rw = self._random_walker_cache()

    def __len__(self):
        return len(self.sample_list)

    def _random_walker_cache(self):
        """{case: pseudo label} for the training slices whose source has no 'random_walker' dataset (the synthetic stand-in and the
        shipped ACDC slice files, which hold only image / label / scribble).  The labels of the reference's offline generator
        (acdc_pseudo_label_random_walker.py:9-26) are computed once, on the GPU, in this process (`random_walker_labels`) and kept
        on the host: DataLoader workers read them without touching the GPU.  Files that do carry the dataset are read as before."""
        todo, ims, scrs = [], [], []
        for case in self.sample_list:
            if self._synthetic is not None:
                img, _, scr = self._synthetic[case.split("_")[0]]
                z = int(case.rsplit("_", 1)[1].split(".")[0])
                img, scr = img[z], scr[z]
            else:
                import h5py
                with h5py.File(os.path.join(self._base_dir, "ACDC_training_slices", case), "r") as f:
                    if "random_walker" in f:
                        continue
                    img, scr = f["image"][:], f["scribble"][:]
            todo.append(case)
            ims.append(np.asarray(img, np.float32))
            scrs.append(np.asarray(scr).astype(np.uint8))
        if not todo:
            return {}
        from .random_walker import random_walker_labels
        labels, _ = random_walker_labels(ims, scrs, names=todo)
        return dict(zip(todo, labels))

    def _read(self, case):
        """-> (image, label) numpy arrays of one train slice / one validation volume"""
        key = self.sup_type if self.split == "train" else "label"
        if case in self._rw:
            if self._synthetic is not None:
                img = self._synthetic[case.split("_")[0]][0][int(case.rsplit("_", 1)[1].split(".")[0])]
            else:
                import h5py
                with h5py.File(os.path.join(self._base_dir, "ACDC_training_slices", case), "r") as f:
                    img = f["image"][:]
            return img, self._rw[case]
        if self._synthetic is not None:
            img, lab, scr = self._synthetic[case.split("_")[0]]
            if self.split == "train":
                z = int(case.rsplit("_", 1)[1].split(".")[0])
                return img[z], (scr if key == "scribble" else lab)[z]
            return img, lab
        try:
            import h5py
        except ImportError as e:
            raise ImportError("h5py is required to read the ACDC files; pass base_dir='synthetic' for the generated stand-in") from e
        sub = "ACDC_training_slices" if self.split == "train" else "ACDC_training_volumes"
        with h5py.File(os.path.join(self._base_dir, sub, case), "r") as f:
            return f["image"][:], f[key][:]

    def __getitem__(self, idx):
        case = self.sample_list[idx]
        image, label = self._read(case)
        sample = {"image": image, "label": label}
        if self.split == "train" and self.transform is not None:
            sample = self.transform(sample)
        sample["idx"] = case.split("_")[0]
        return sample

    def to_slice_store(self, device=None):
        """the training slices as a resident GPU `SliceStore` (feed it to `GpuLoader`)"""
        assert self.split == "train"
        pairs = [self._read(c) for c in self.sample_list]
        return SliceStore.from_arrays([p[0] for p in pairs], [p[1] for p in pairs], [c.split("_")[0] for c in self.sample_list], device)


class TwoStreamBatchSampler(torch.utils.data.Sampler):
    """Batch sampler of the reference's semi-supervised scripts (imported by train_s2l.py:20): every batch is
    ``batch_size - secondary_batch_size`` indices of `primary_indices`, walked once per epoch in a fresh numpy permutation, followed
    by `secondary_batch_size` indices of `secondary_indices`, cycled through as many fresh permutations as the epoch needs.  An
    epoch has len(primary_indices) // primary batch size batches; a trailing partial primary batch is dropped."""

    def __init__(self, primary_indices, secondary_indices, batch_size, secondary_batch_size):
        self.primary_indices, self.secondary_indices = primary_indices, secondary_indices
        self.secondary_batch_size = int(secondary_batch_size)
        self.primary_batch_size = int(batch_size) - self.secondary_batch_size
        if not 0 < self.primary_batch_size <= len(primary_indices):
            raise ValueError(f"primary batch size {self.primary_batch_size} must be in [1, {len(primary_indices)}]")
        if not 0 < self.secondary_batch_size <= len(secondary_indices):
            raise ValueError(f"secondary batch size {self.secondary_batch_size} must be in [1, {len(secondary_indices)}]")

    def __len__(self):
        return len(self.primary_indices) // self.primary_batch_size

    def _secondary(self):
        while True:
            yield from np.random.permutation(self.secondary_indices)

    def __iter__(self):
        primary = np.random.permutation(self.primary_indices)       # drawn when the epoch's iterator is created
        secondary = self._secondary()
        nb, sb = self.primary_batch_size, self.secondary_batch_size

        def batches():
            for b in range(len(self)):
                yield tuple(primary[b * nb:(b + 1) * nb]) + tuple(next(secondary) for _ in range(sb))
        return batches()


class BaseDataSets_s2l(torch.utils.data.Dataset):
    """``BaseDataSets_s2l(base_dir, transform, fold, num)`` of dataset_s2l.py:19-100: the fold's training slices held in memory as
    ``images[idx] = {'id', 'image', 'mask', 'scribble', 'weight'}`` with a zero-initialised [h, w, 4] fp32 prediction memory
    (:46) that train_s2l.py's ensemble refresh rewrites in place (:243).  base_dir as `BaseDataSets` (ACDC directory with h5py,
    or 'synthetic[:<patients>]').  ``to_slice_store()`` hands the slices to the resident GPU pipeline (`S2LLoader`)."""

    def __init__(self, base_dir=None, transform=None, fold="fold1", num=None):
        src = BaseDataSets(base_dir, "train", None, fold, "label")     # `num` is accepted and ignored, as in the reference
        self._base_dir, self.transform = base_dir, transform
        self.sample_list = list(src.sample_list)
        self.images = collections.defaultdict(dict)
        for idx, case in enumerate(self.sample_list):
            src.sup_type = "label"
            img, mask = src._read(case)
            src.sup_type = "scribble"
            _, scr = src._read(case)
            rec = self.images[idx]
            rec["id"], rec["image"], rec["mask"], rec["scribble"] = case, np.asarray(img), np.asarray(mask), np.asarray(scr)
            rec["weight"] = np.zeros(tuple(np.shape(mask)) + (4,), dtype=np.float32)

    def __len__(self):
        return len(self.sample_list)

    def __getitem__(self, idx):
        rec = self.images[idx]
        sample = {"image": rec["image"], "mask": rec["mask"], "scribble": rec["scribble"], "weight": rec["weight"]}
        sample = self.transform(sample)
        sample["id"] = rec["id"]
        return sample

    def to_slice_store(self, device=None):
        """the slices (mask as label, scribble, zero memory) as a resident GPU `SliceStore` for `S2LLoader` / `S2LStep.refresh`"""
        recs = [self.images[i] for i in range(len(self))]
        return SliceStore.from_arrays([r["image"] for r in recs], [r["mask"] for r in recs], [r["id"].split("_")[0] for r in recs],
                                      device, scribbles=[r["scribble"] for r in recs])


class GpuLoader:
    """Replaces ``DataLoader(db_train, batch_size, shuffle=True)`` + ``RandomGenerator`` for the training split: yields
    ``{'image': [B,1,H,W] fp32 cuda, 'label': [B,H,W] uint8 cuda, 'idx': [...]}`` (script keys, dataset_semi.py:120-124)."""

    def __init__(self, store, batch_size, output_size=(256, 256), shuffle=True, drop_last=False, rank=0, world_size=1, streams=None):
        """`batch_size` is per rank.  With world_size > 1 every rank walks the SAME permutation (all ranks seed torch alike, as
        the scripts do with args.seed) and takes the strided share rank::world_size of it, like DistributedSampler.  streams:
        the (random.Random, np.random.RandomState) the augmentation parameters are drawn from (`rank_streams`); None: the global
        `random` / `np.random`, as the scripts' transform draws."""
        self.store, self.batch_size, self.shuffle, self.drop_last = store, int(batch_size), shuffle, drop_last
        self.rank, self.world_size = int(rank), int(world_size)
        assert 0 <= self.rank < self.world_size
        self.transform = RandomGenerator(output_size)
        self.streams = streams

    @staticmethod
    def shard(order, rank, world_size):
        """DistributedSampler's partition: pad the permutation by wrapping to a multiple of world_size, then stride."""
        if world_size == 1:
            return list(order)
        total = (len(order) + world_size - 1) // world_size * world_size
        padded = list(order) + list(order)[: total - len(order)]
        return padded[rank:total:world_size]

    def __len__(self):
        n = (len(self.store) + self.world_size - 1) // self.world_size
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def _batches(self):
        """slice ids of every batch of one epoch"""
        n = len(self.store)
        if self.shuffle:     # torch.utils.data.RandomSampler: fresh generator seeded from the default stream, then randperm
            seed = int(torch.empty((), dtype=torch.int64).random_().item())
            g = torch.Generator()
            g.manual_seed(seed)
            order = torch.randperm(n, generator=g).tolist()
        else:
            order = list(range(n))
        order = self.shard(order, self.rank, self.world_size)
        n = len(order)
        for s in range(0, n, self.batch_size):
            idx = order[s:s + self.batch_size]
            if len(idx) < self.batch_size and self.drop_last:
                break
            yield idx

    def __iter__(self):
        for idx in self._batches():
            params = [self.transform.draw(bool(self.store.has4[i]), self.streams) for i in idx]
            img, lab = self.store.augment(idx, params, self.transform.output_size)
            yield {"image": img, "label": lab, "idx": [self.store.names[i] for i in idx]}


class S2LLoader(GpuLoader):
    """Replaces ``DataLoader(BaseDataSets_s2l, batch_size, shuffle=True, num_workers=8)`` + ``RandomGenerator_s2l``
    (train_s2l.py:86-99): yields ``{'image': [B,1,H,W] fp32, 'scribble': [B,H,W] u8, 'weight': [B,H,W,4] fp32, 'idx': [...]}``.

    visibility='epoch' (default, SURVEY F16): the script's workers are forked when an epoch's iterator is created, so its
    batches see the prediction memory as it was at that moment; the snapshot is taken when iteration starts and a refresh in
    mid-epoch reaches the batches of the next epoch.  visibility='live': batches read the memory the refresh updates."""

    def __init__(self, store, batch_size, output_size=(256, 256), shuffle=True, drop_last=False, visibility="epoch", rank=0,
                 world_size=1, streams=None):
        """rank, world_size, streams: `GpuLoader`'s (the same `shard` partition of every epoch's permutation)"""
        assert store.scribbles is not None, "S2LLoader needs a SliceStore built with scribbles="
        if visibility not in ("epoch", "live"):
            raise ValueError(f"visibility must be 'epoch' or 'live' (got {visibility!r})")
        super().__init__(store, batch_size, output_size, shuffle, drop_last, rank, world_size, streams)
        self.visibility = visibility

    def __iter__(self):
        if self.visibility == "epoch":
            self.store.weight_epoch.copy_(self.store.weight_live)
        for idx in self._batches():
            # the draws of RandomGenerator_s2l are RandomGenerator's; the scribble is rotated with cval 0 (SURVEY F15)
            params = [self.transform.draw(False, self.streams) for _ in idx]
            img, scr, wgt = self.store.augment_s2l(idx, params, self.transform.output_size, self.visibility)
            yield {"image": img, "scribble": scr, "weight": wgt, "idx": [self.store.names[i] for i in idx]}
