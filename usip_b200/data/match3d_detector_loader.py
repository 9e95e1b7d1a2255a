"""The 3DMatch detector loader on the GPU: data/match3d_detector_loader.py (Match3DDetectorLoader), used by
match3d/train_detector.py, and the builder it shares with the SceneNN loader (scenenn_detector_loader.py).

Both reference loaders are KittiLoader's code with the indoor laws (:110-177): jitter sigma 0.01 clipped at 0.02 for pc,
every sn column and nodes, perturbation angles clip(0.12 randn, +-0.36), augmentation scale U(0.8, 1.2), and the dst
transform's scale_thre 0.1 (:214-216).  sn is always columns 3:3+S (:105); there is no radius mask; a fragment shorter
than input_pc_num is taken whole t times, then a random remainder (:95-102).  They draw an item's randomness in their
own order (:181-190): rows of src, rows of dst, then FPS candidates and start of src, then of dst.  They differ only in
the dataset listing and the FPS candidate count: N/10 here, N/4 for SceneNN.

`IndoorPairBuilder` builds the nine `ModelDetector.set_input` tensors on the device (csrc/pairgen.cu: the shared subset,
candidate and FPS kernels, and `usip_indoor_pair_augment`), with one augmentation switch per pair for SceneNN's mixed
train + val batches.  `Match3DPairSource` feeds them from a 3DMatch training tree.  Fragments may be longer than the
one-CTA subsample kernel holds: the cluster kernel then draws their rows.
"""
import os

import numpy as np
import torch

from usip_b200 import ops

from .kitti_detector_loader import _PairBuilder, _ScanSource, draw_candidates, draw_pair_scalars, draw_rows

MATCH3D_DIVISOR = 10                             # match3d_detector_loader.py:186-190: FPS over N/10 candidates
INDOOR_SCALE = (0.8, 1.2)                        # :134
INDOOR_PERTURBATION = (0.12, 0.36)               # :123
INDOOR_JITTER = ((0.01, 0.02), (0.01, 0.02), (0.01, 0.02))   # :125-132: pc, sn, node
INDOOR_SCALE_THRE = 0.1                          # :214-216
MAX_S = 8                                        # usip_indoor_pair_augment


class IndoorPairBuilder(_PairBuilder):
    """Builds the nine `ModelDetector.set_input` tensors of a batch of 3DMatch or SceneNN pairs on the device.

    `build(scans, offsets, items, step=None, augment=None)`: scans [T, C] f32 (device, or host -- then the items' scans
    are uploaded), offsets (n_scans+1,) int64 row offsets (host), items the scan index of every pair.  Both clouds of a
    pair are independent subsamples of the same fragment.  augment: one bool per item, whether the pair is augmented
    (train mode only; default all True).  A pair with augment False gets only the dst transform, as the reference's
    'val' loader gives it, and makes no augmentation draws in either rng mode.  divisor: MATCH3D_DIVISOR or
    scenenn_detector_loader.SCENENN_DIVISOR.  See `_PairBuilder` for the two rng modes; rng="numpy" replays the
    reference loader's __getitem__, item by item.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device", divisor=MATCH3D_DIVISOR):
        super().__init__(opt, mode, device, seed, rng, divisor)
        if not 1 <= self.S <= MAX_S:
            raise ValueError("surface_normal_len %d: the indoor builder takes 1 to %d sn columns" % (self.S, MAX_S))
        self._pending = None                     # augment flags of the pairs still to be drawn in this build

    def _clouds(self, items):
        items = np.asarray(items, dtype=np.int64).ravel()
        if items.size == 0:
            raise ValueError("no items")
        return np.repeat(items, 2)

    def _draw(self, rng, per_point):
        # called once per pair, in pair order, in both rng modes
        train = self.mode == "train"
        aug = train and next(self._pending)
        p, jit = draw_pair_scalars(rng, self.opt, aug, self.N, self.M, self.S, per_point, INDOOR_SCALE,
                                   INDOOR_PERTURBATION, INDOOR_JITTER, INDOOR_SCALE_THRE)
        if train:
            p[ops.PAIR_AUGMENT_SLOT] = float(aug)
            if per_point and jit is None:        # never read by the kernel; keeps the batch's upload arrays whole
                jit = (np.zeros((2, self.N, 3)), np.zeros((2, self.N, self.S)), np.zeros((2, self.M, 3)))
        return p, jit

    def _draw_item(self, rng, n_valid):
        """match3d_detector_loader.py:181-216: rows of src and dst, then candidates and start of src and of dst, then
        the augmentation and the transform."""
        rows = [draw_rows(rng, n, self.N) for n in n_valid]
        cands = [draw_candidates(rng, self.N, self.divisor) for _ in n_valid]
        return [(r,) + c for r, c in zip(rows, cands)], self._draw(rng, True)

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.indoor_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.S, self.flags,
                                       self.seed, step, *jit)

    def build(self, scans, offsets, items, step=None, augment=None):
        n = np.asarray(items).size
        aug = np.ones(n, bool) if augment is None else np.asarray(augment, dtype=bool).ravel()
        if aug.shape != (n,):
            raise ValueError("augment needs one flag per item: %d flags for %d items" % (aug.size, n))
        self._pending = iter(aug.tolist())
        try:
            return self._build(scans, offsets, step, items)
        finally:
            self._pending = None


class _IndoorSource(_ScanSource):
    """A list of fragment files, one per item, for the indoor builder; resident="disk" reads each batch's fragments
    when the batch is built.  A subclass may give items an augmentation mask (`augment_mask`)."""

    disk_resident = True

    def __init__(self, paths, mode, opt, divisor, device, seed, resident, rng, batch_size, drop_last, augment=None):
        if not paths:
            raise ValueError("no fragments")
        self.augment_mask = None if augment is None else np.asarray(augment, dtype=bool)
        super().__init__(paths, mode, opt,
                         lambda o, m, d, s, r: IndoorPairBuilder(o, m, d, s, r, divisor),
                         device, seed, resident, rng, batch_size, drop_last)

    def _build(self, items):
        items = np.asarray(items, dtype=np.int64)
        scans, offsets, idx = self._batch_scans(items)
        aug = None if self.augment_mask is None else self.augment_mask[items]
        return self.builder.build(scans, offsets, idx, step=self.step, augment=aug), None


# ----------------------------------------------------------------------------------------------- 3DMatch tree
def make_3dmatch_dataset(root, mode):
    """match3d_detector_loader.py:49-73 -> the fragment paths: the folders named by training_list.txt (train) or
    testing_list.txt (test), in the list's order, then every sub-folder of each, then every file of each sub-folder.
    The reference lists folders with os.listdir, whose order depends on the filesystem; here each level is sorted, so an
    item index names the same file on every machine."""
    if mode not in ("train", "test"):
        raise ValueError("mode must be 'train' or 'test'")
    with open(os.path.join(root, "training_list.txt" if mode == "train" else "testing_list.txt")) as f:
        folders = [x.rstrip() for x in f.readlines()]
    paths = []
    for folder in folders:
        for sub in sorted(os.listdir(os.path.join(root, folder))):
            if not os.path.isdir(os.path.join(root, folder, sub)):
                continue
            paths += [os.path.join(root, folder, sub, name) for name in sorted(os.listdir(os.path.join(root, folder,
                                                                                                         sub)))]
    return paths


def write_synthetic_3dmatch_train(root, splits, rows, seed=0):
    """A 3DMatch training tree for tests and benchmarks: splits {"train" | "test": {scene: {sub-folder: n files}}}
    gives training_list.txt / testing_list.txt (the scenes in the dict's order) and <root>/<scene>/<sub>/<k>.npy for
    k < n, each a synthetic_fragment of rows(i) rows (i counts the files in listing order; rows may also be an int).
    Every scene folder also holds a notes.txt, which the listing skips."""
    from usip_b200.evaluation.indoor_test_loader import synthetic_fragment
    os.makedirs(root, exist_ok=True)
    i = 0
    for split, scenes in splits.items():
        name = {"train": "training_list.txt", "test": "testing_list.txt"}[split]
        with open(os.path.join(root, name), "w") as f:
            f.write("".join(s + "\n" for s in scenes))
        for scene, subs in scenes.items():
            os.makedirs(os.path.join(root, scene), exist_ok=True)
            with open(os.path.join(root, scene, "notes.txt"), "w") as f:
                f.write("not a fragment folder\n")
            for sub in sorted(subs):
                os.makedirs(os.path.join(root, scene, sub), exist_ok=True)
                for k in sorted(range(subs[sub]), key=lambda k: "%d.npy" % k):
                    n = rows if np.isscalar(rows) else rows(i)
                    np.save(os.path.join(root, scene, sub, "%d.npy" % k), synthetic_fragment(seed + i, n))
                    i += 1


class Match3DPairSource(_IndoorSource):
    """Shuffled batches of 3DMatch detector pairs (the items of make_3dmatch_dataset(root, mode)), built on the device
    and handed to `ModelDetector` (see `_ScanSource`).  resident: "host" (pinned), "device", or "disk" (each batch's
    fragments are read when it is built, for training sets larger than host memory).

        src = Match3DPairSource(root, "train", opt)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, device=None, seed=0, resident="host", rng="device", batch_size=None,
                 drop_last=True):
        self.dataset = make_3dmatch_dataset(root, mode)
        super().__init__(self.dataset, mode, opt, MATCH3D_DIVISOR, device, seed, resident, rng, batch_size, drop_last)
