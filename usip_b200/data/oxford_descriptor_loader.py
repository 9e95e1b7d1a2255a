"""The Oxford descriptor loader on the GPU: data/oxford_descriptor_loader.py (OxfordDescriptorLoader) and the batch
preparation of oxford/train_descriptor.py:90-138.

Each item is an anchor scan and a positive drawn (Python's `random`) from the anchor's positive list, both subsampled
(N rows without replacement), given FPS nodes over N/4 candidates, mapped from ENU to the camera frame and augmented
per cloud like KITTI's descriptor loader with the scale fixed at 1.0.  The frozen detector turns the clouds into
keypoints and sigmas; then, in train mode, one height scale U(0.25, 1.2) per batch multiplies camera y (the down axis)
of the anchors' and positives' clouds and keypoints, and the negatives are mined among the other items of the batch.
`OxfordDescriptorPairBuilder` builds the clouds on the device (csrc/pairgen.cu: the shared subset, gather and FPS
kernels and `usip_desc_pair_augment` with USIP_PAIR_ENU_TO_CAM); `OxfordDescriptorPairSource` adds the positives,
the frozen detector pass, the height scaling (`usip_scale_channel_f32`) and the mining, and hands the nine
`ModelDescriptor.set_input` tensors over without a host synchronise.
"""
import os
import pickle
import random
import warnings

import numpy as np
import torch

from usip_b200 import ops

from .kitti_descriptor_loader import draw_desc_pair_scalars
from .kitti_detector_loader import _PairBuilder, _ScanSource, _step_rng
from .oxford_detector_loader import (HEIGHT_SCALE_RANGE, OXFORD_TEST_FOLDER, _OxfordRows, check_oxford_opt,
                                     oxford_test_path, oxford_train_path, parse_train_relative)

OXFORD_DESC_DIVISOR = 4                          # oxford_descriptor_loader.py:289: FPS over N/4 candidates


# ----------------------------------------------------------------------------------------------- Oxford tree
def make_dataset_oxford_train(root):
    """oxford_descriptor_loader.py:55-83 -> [{'file', 'pos_line_list', 'nonneg_line_list'}]; the non-negatives include
    the positives (non-negatives first)."""
    return [{"file": f, "pos_line_list": p, "nonneg_line_list": n + p} for f, p, n in parse_train_relative(root)]


def make_dataset_oxford_test(root):
    """oxford_descriptor_loader.py:86-88: the list in test_models_20k_np_nofilter/gt_descriptor_testing.pkl (dicts with
    'anc_idx' and 'pos_idx_list', file numbers)."""
    with open(os.path.join(root, OXFORD_TEST_FOLDER, "gt_descriptor_testing.pkl"), "rb") as f:
        return pickle.load(f)


# ----------------------------------------------------------------------------------------------- host-side draws
def pick_positive(dataset, mode, index, rng=random):
    """get_instance_pos_unaugmented_np (:127-138): one rng.randint over the item's positives -> in train mode a dataset
    index (a line of train_relative.txt), in test mode a FILE number (test_models_20k_np_nofilter/%d.npy)."""
    lst = dataset[index]["pos_line_list" if mode == "train" else "pos_idx_list"]
    return lst[rng.randint(0, len(lst) - 1)]


def mine_negative_sample(dataset, mode, index_batch, rng=random):
    """OxfordDescriptorLoader.mine_negative_sample (:231-281): for every anchor i, a random other item j of the batch
    (candidates in ascending j, one rng.randint) whose line is not among i's non-negatives (train), or whose anchor file
    is not among i's positive files (test).  The reference's test branch runs the whole mining once per anchor -- B
    passes, B times the draws, the last pass wins -- and so does this.  An anchor without a candidate keeps neg_idx 0,
    with a warning.  -> (B,) int64 tensor on the host."""
    if mode not in ("train", "test"):
        raise ValueError("Incorrect dataloader mode")
    index_batch = [int(i) for i in (index_batch.tolist() if hasattr(index_batch, "tolist") else index_batch)]
    B = len(index_batch)
    neg_idx = torch.zeros(B, dtype=torch.int64)
    if mode == "train":
        excluded = [set(dataset[index]["nonneg_line_list"]) for index in index_batch]
        key = index_batch
    else:
        excluded = [set(dataset[index]["pos_idx_list"]) for index in index_batch]
        key = [dataset[index]["anc_idx"] for index in index_batch]
    for _ in range(B if mode == "test" else 1):
        for i in range(B):
            cand = [j for j in range(B) if j != i and key[j] not in excluded[i]]
            if not cand:
                warnings.warn("mine_negative_sample: anchor %d of the batch has no negative; neg_idx stays 0" % i)
            else:
                neg_idx[i] = cand[rng.randint(0, len(cand) - 1)]
    return neg_idx


# ----------------------------------------------------------------------------------------------- the builder
class OxfordDescriptorPairBuilder(_OxfordRows, _PairBuilder):
    """Builds the six cloud tensors (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node) of a batch of Oxford descriptor
    pairs on the device, in the camera frame.

    `build(scans, offsets, anc_items, pos_items, step=None)`: scans [T, C] f32 ENU (device, or host -- then the items'
    scans are uploaded), offsets (n_scans+1,) int64 row offsets (host), anc_items / pos_items the scan index of every
    anchor and positive.  Every scan needs input_pc_num rows; sn is columns 3:3+S with 3 <= S <= 8.

    See `_PairBuilder` for the two rng modes; rng="numpy" replays OxfordDescriptorLoader.__getitem__, whose numpy draws
    come in the order anchor rows, positive rows, candidates and start of the anchor, of the positive, then the
    augmentation (per cloud, no scale draw).  The positive is drawn from Python's `random` only (`pick_positive`).
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device"):
        super().__init__(opt, mode, device, seed, rng, OXFORD_DESC_DIVISOR)
        check_oxford_opt(self)
        self.flags |= ops.PAIR_ENU_TO_CAM

    def _clouds(self, anc_items, pos_items):
        anc = np.asarray(anc_items, dtype=np.int64).ravel()
        pos = np.asarray(pos_items, dtype=np.int64).ravel()
        if anc.size == 0:
            raise ValueError("no items")
        if anc.shape != pos.shape:
            raise ValueError("%d anchors but %d positives" % (anc.size, pos.size))
        return np.stack([anc, pos], 1).ravel()                # cloud 2b = anchor b, 2b+1 = its positive

    def _draw(self, rng, per_point):
        p, _, jit = draw_desc_pair_scalars(rng, self.mode == "train", self.N, self.M, self.S, per_point,
                                           scale_range=None)
        return p, jit

    def _draw_item(self, rng, n_valid):
        sides, _ = self._draw_rows_then_nodes(rng, n_valid)
        return sides, self._draw(rng, True)

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.desc_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.S, self.flags, self.seed,
                                     step, *jit)

    def build(self, scans, offsets, anc_items, pos_items, step=None):
        return self._build(scans, offsets, step, anc_items, pos_items)


def scale_height_(hs, *tensors):
    """oxford/train_descriptor.py:124-130: t[:, 1, :] *= hs (camera y, the down axis) of every (B, C, L) f32 tensor, in
    place, in fp32 as torch does."""
    for t in tensors:
        ops.scale_channel_(t, 1, hs)


class OxfordDescriptorPairSource(_ScanSource):
    """Shuffled batches of Oxford descriptor training inputs, built on the device, for `ModelDescriptor`.

    The items are those of make_dataset_oxford_train(root) (train; item i reads its own line's scan) or
    make_dataset_oxford_test(root) (test; every file number an item or a positive names is loaded once).  For every
    batch, on the build stream: pick each anchor's positive (`pick_positive`), then mine the negatives
    (`mine_negative_sample`), both from one `random.Random`; build the clouds (`OxfordDescriptorPairBuilder`); run the
    frozen `detector.run_model_siamese` on the unscaled clouds; in train mode draw the batch's height scale and, when
    opt.is_height_scaling (the default), apply it to camera y of both clouds and both keypoint sets.  The height scale
    comes from the (seed, step) host RandomState in device mode, and from np.random after the items' draws in parity
    mode (rng="numpy"), as a single-process DataLoader and the training loop draw it.

        src = OxfordDescriptorPairSource(root, "train", opt, detector)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, detector, device=None, seed=0, resident="host", rng="device",
                 batch_size=None, drop_last=True):
        if mode == "train":
            self.dataset = make_dataset_oxford_train(root)
            paths = [oxford_train_path(root, d["file"]) for d in self.dataset]
            self.item_scan = np.arange(len(self.dataset), dtype=np.int64)
            self.scan_of_positive = lambda p: p                    # a positive is a line, i.e. an item
        elif mode == "test":
            self.dataset = make_dataset_oxford_test(root)
            numbers = sorted({int(d["anc_idx"]) for d in self.dataset}
                             | {int(p) for d in self.dataset for p in d["pos_idx_list"]})
            slot = {n: k for k, n in enumerate(numbers)}
            paths = [oxford_test_path(root, n) for n in numbers]
            self.item_scan = np.array([slot[int(d["anc_idx"])] for d in self.dataset], dtype=np.int64)
            self.scan_of_positive = lambda p: slot[int(p)]         # a positive is a file number
        else:
            raise ValueError("mode must be 'train' or 'test'")
        if not self.dataset:
            raise ValueError("no items under %s" % root)
        super().__init__(paths, mode, opt, OxfordDescriptorPairBuilder, device, seed, resident, rng, batch_size,
                         drop_last, n_items=len(self.dataset))
        self.detector = detector
        self.seed, self.rng_mode = int(seed), rng
        self.height_scaling = bool(getattr(opt, "is_height_scaling", True))
        self.rand = random.Random(seed)

    def _height_scale(self, step):
        if self.rng_mode == "numpy":
            return np.random.uniform(low=HEIGHT_SCALE_RANGE[0], high=HEIGHT_SCALE_RANGE[1])
        return _step_rng(self.seed, step, stream=1).uniform(low=HEIGHT_SCALE_RANGE[0], high=HEIGHT_SCALE_RANGE[1])

    def _build(self, items):
        items = [int(i) for i in items]
        pos = [pick_positive(self.dataset, self.mode, i, self.rand) for i in items]
        neg = mine_negative_sample(self.dataset, self.mode, items, self.rand)
        step = self.step
        anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node = self.builder.build(
            self.scans, self.offsets, self.item_scan[items], [self.scan_of_positive(p) for p in pos], step=step)
        (anc_kp, pos_kp), (anc_sig, pos_sig) = self.detector.run_model_siamese((anc_pc, pos_pc), (anc_sn, pos_sn),
                                                                               (anc_node, pos_node))
        hs = None
        if self.mode == "train":                                # oxford/train_descriptor.py:123-130
            hs = self._height_scale(step)
            if self.height_scaling:
                scale_height_(hs, anc_pc, anc_kp, pos_pc, pos_kp)
        neg_d = neg.pin_memory().to(self.device, non_blocking=True)
        info = {"items": np.asarray(items), "positives": np.asarray(pos), "neg_idx": neg, "height_scale": hs, "step": step,
                "clouds": (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node)}
        return (anc_pc, anc_sn, anc_kp, anc_sig, pos_pc, pos_sn, pos_kp, pos_sig, neg_d), info
