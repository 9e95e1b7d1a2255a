"""The KITTI descriptor loader on the GPU: data/kitti_descriptor_loader.py (KittiDescriptorLoader) and the batch
preparation of kitti/train_descriptor.py:94-132.

The descriptor is trained on keypoints of the frozen detector.  Each item is an anchor scan and a positive scan
within `positive_radius_threshold` of it, both subsampled, given FPS nodes and augmented; the frozen detector turns
every cloud into keypoints and sigmas, and the negatives are other anchors of the batch more than
`negative_radius_threshold` away.  `DescriptorPairBuilder` builds the clouds on the device (csrc/pairgen.cu: the
per-cloud subset and candidate kernels the detector builder uses, and `usip_desc_pair_augment`);
`KittiDescriptorPairSource` adds the positive search, the frozen detector pass and negative mining, and hands the nine
`ModelDescriptor.set_input` tensors over without a host synchronise.
"""
import os
import random
import warnings

import numpy as np
import torch

from usip_b200 import ops

from .kitti_detector_loader import _KittiSource, _PairBuilder, angles2rotation_matrix, make_dataset_kitti

DESC_DIVISOR = 4                                 # kitti_descriptor_loader.py:127: FPS over N/4 candidates


# ----------------------------------------------------------------------------------------------- host-side draws
def nearby_index(index, poses, accs, nums, positive_radius_threshold, rng=random):
    """get_nearby_instance_unagumented_np (kitti_descriptor_loader.py:154-197) over preloaded poses: the dataset index of
    a scan of the same sequence whose pose translation is within `positive_radius_threshold` of `index`'s.

    poses (n, 4, 4) in dataset order; accs / nums the accumulated and per-sequence scan counts of make_dataset_kitti;
    rng a `random.Random`-like object (the reference draws from Python's `random`, not numpy).  After 3 * search_interval
    misses the anchor itself is returned, as in the reference."""
    si = next(i for i, a in enumerate(accs) if index < a)
    base = accs[si - 1] if si else 0
    index_in_seq = index - base
    pose = poses[index]
    search_interval = int(positive_radius_threshold / 0.8 * 2)
    lo = max(index_in_seq - search_interval, 0)
    hi = min(index_in_seq + search_interval, nums[si] - 1)
    counter = 0
    while True:
        nearby = rng.randint(lo, hi)
        distance = np.linalg.norm((poses[base + nearby] - pose)[0:3, 3])
        if distance < positive_radius_threshold:
            break
        if nearby < index_in_seq:
            lo = nearby + 1
        else:
            hi = nearby - 1
        counter += 1
        if counter >= search_interval * 3:
            nearby = index_in_seq
            break
    return base + nearby


def mine_negative_sample(anc_seq, anc_pose, threshold, rng=np.random):
    """KittiDescriptorLoader.mine_negative_sample (:278-317): for every anchor, a random other anchor of another
    sequence or more than `threshold` away.  Float32 poses, np.linalg.inv and np.dot in float32, candidates in
    ascending j, one rng.randint per anchor that has candidates.  An anchor without a candidate keeps neg_idx 0 (as in
    the reference) and raises a warning.  -> (B,) int64 tensor on the host."""
    poses = np.asarray(anc_pose.numpy() if torch.is_tensor(anc_pose) else anc_pose, dtype=np.float32)
    seq = [int(s) for s in (anc_seq.tolist() if hasattr(anc_seq, "tolist") else anc_seq)]
    B = poses.shape[0]
    neg_idx = torch.zeros(B, dtype=torch.int64)
    for i in range(B):
        cand = []
        for j in range(B):
            if j == i:
                continue
            if seq[i] != seq[j]:
                cand.append(j)
            else:
                i_j = np.dot(np.linalg.inv(poses[i]), poses[j])
                if np.linalg.norm(i_j[0:3, 3]) > threshold:
                    cand.append(j)
        if not cand:
            warnings.warn("mine_negative_sample: anchor %d of the batch has no negative; neg_idx stays 0" % i)
        else:
            neg_idx[i] = cand[rng.randint(len(cand))]
    return neg_idx


def draw_desc_pair_scalars(rng, train, N, M, S, per_point):
    """Scalars of KittiDescriptorLoader.augment (:205-276) for one pair, in the reference's order ->
    (params (2, 32) f64 per cloud, scale, jitter (pc (2,N,3), sn (2,N,S), node (2,M,3)) or None).
    per_point=False skips the O(N) jitter draws (the device draws its own)."""
    p = np.zeros((2, ops.DESC_PARAM_STRIDE), dtype=np.float64)
    if not train:
        return p, 0.0, None
    scale = rng.uniform(low=0.9, high=1.1)
    jit = ([], [], [])
    for side in range(2):
        y_angle = rng.uniform() * 2 * np.pi
        angles_3d = rng.rand(3) * np.pi * 2
        angles_pertb = np.clip(0.06 * rng.randn(3), -0.18, 0.18)
        if per_point:
            jit[0].append(np.clip(0.04 * rng.randn(N, 3), -0.12, 0.12))
            jit[1].append(np.clip(0.01 * rng.randn(N, S), -0.05, 0.05))
            jit[2].append(np.clip(0.04 * rng.randn(M, 3), -0.12, 0.12))
        shift = rng.uniform(-1, 1, (1, 3))
        p[side, 0:9] = angles2rotation_matrix([0, y_angle, 0]).ravel()
        p[side, 9:18] = angles2rotation_matrix(angles_3d).ravel()
        p[side, 18:27] = angles2rotation_matrix(angles_pertb).ravel()
        p[side, 27] = scale
        p[side, 28:31] = shift.ravel()
    return p, scale, (tuple(np.stack(a) for a in jit) if per_point else None)


# ----------------------------------------------------------------------------------------------- the builder
class DescriptorPairBuilder(_PairBuilder):
    """Builds the six cloud tensors (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node) of a batch of KITTI
    descriptor pairs on the device.

    `build(scans, offsets, anc_items, pos_items, step=None)`: scans [T, C] f32 (device, or host -- then the items'
    scans are uploaded), offsets (n_scans+1,) int64 row offsets (host), anc_items / pos_items the scan index of every
    anchor and positive.  Every scan needs at least input_pc_num rows: the reference draws them without replacement.

    See `_PairBuilder` for the two rng modes; rng="numpy" replays KittiDescriptorLoader.__getitem__.  The positive
    search draws from Python's `random` only, so choosing pos_items beforehand with `nearby_index` changes no numpy
    draw.  `last` keeps the index lists of the last build, and the pairs' scales.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device"):
        super().__init__(opt, mode, device, seed, rng, DESC_DIVISOR)
        if not 1 <= self.S <= 8:
            raise ValueError("surface_normal_len %d: the augment kernel takes 1..8" % self.S)

    def _clouds(self, anc_items, pos_items):
        anc = np.asarray(anc_items, dtype=np.int64).ravel()
        pos = np.asarray(pos_items, dtype=np.int64).ravel()
        if anc.size == 0:
            raise ValueError("no items")
        if anc.shape != pos.shape:
            raise ValueError("%d anchors but %d positives" % (anc.size, pos.size))
        return np.stack([anc, pos], 1).ravel()                # cloud 2b = anchor b, 2b+1 = its positive

    def _check_rows(self, clouds, lengths):
        k = int(np.argmin(lengths))
        if lengths[k] < self.N:
            raise ValueError("scan %d has %d rows; input_pc_num = %d rows are drawn without replacement"
                             % (int(clouds[k]), int(lengths[k]), self.N))

    def _draw(self, rng, per_point):
        p, _, jit = draw_desc_pair_scalars(rng, self.mode == "train", self.N, self.M, self.S, per_point)
        return p, jit

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.desc_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.S, self.flags, self.seed,
                                     step, *jit)

    def build(self, scans, offsets, anc_items, pos_items, step=None):
        out = self._build(scans, offsets, step, anc_items, pos_items)
        self.last["scale"] = self.last["params"][0::2, 27]    # a pair's scale is in both of its clouds' blocks
        return out


# ----------------------------------------------------------------------------------------------- KITTI tree
def kitti_pose_path(root, seq, index_in_seq):
    """kitti_descriptor_loader.py:115."""
    return os.path.join(root, "poses", "%02d" % seq, "%06d.npz" % index_in_seq)


def load_kitti_poses(root, mode):
    """(seq (n,) int64, poses (n, 4, 4)) of every scan of make_dataset_kitti(root, mode), in dataset order: the sequence
    number and the pose file of each scan (get_seq_pose_by_index, :137-152), loaded once."""
    seqs, _, nums, _ = make_dataset_kitti(root, mode)
    seq = np.array([seqs[s] for s in range(len(seqs)) for _ in range(nums[s])], dtype=np.int64)
    poses = [np.load(kitti_pose_path(root, seqs[s], i))["pose"] for s in range(len(seqs)) for i in range(nums[s])]
    return seq, (np.stack(poses) if poses else np.zeros((0, 4, 4)))


class KittiDescriptorPairSource(_KittiSource):
    """Shuffled batches of KITTI descriptor training inputs, built on the device, for `ModelDescriptor`.

    Scans and hand-over as in `_KittiSource`; the poses are loaded once into a host array.  For every batch, on the
    build stream: pick each anchor's positive with `nearby_index` (host, Python's random), build the clouds
    (`DescriptorPairBuilder`), run the frozen `detector.run_model_siamese` on the built nodes for keypoints and sigmas,
    and mine the negatives (host, float32 poses).

        src = KittiDescriptorPairSource(root, "train", opt, detector)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, detector, device=None, seed=0, resident="host", rng="device",
                 batch_size=None, drop_last=True):
        super().__init__(root, mode, opt, DescriptorPairBuilder, device, seed, resident, rng, batch_size, drop_last)
        self.detector = detector
        self.pos_threshold = float(getattr(opt, "positive_radius_threshold", 5.0))
        self.neg_threshold = float(getattr(opt, "negative_radius_threshold", 50.0))
        self.seq, self.poses = load_kitti_poses(root, mode)
        self.pos_rng = random.Random(seed)
        self.neg_rng = np.random.RandomState(seed + 1)

    def _build(self, anchors):
        pos = [nearby_index(int(a), self.poses, self.accs, self.nums, self.pos_threshold, self.pos_rng)
               for a in anchors]
        neg = mine_negative_sample(self.seq[anchors], self.poses[anchors].astype(np.float32), self.neg_threshold,
                                   self.neg_rng)
        anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node = self.builder.build(self.scans, self.offsets, anchors, pos,
                                                                                step=self.step)
        (anc_kp, pos_kp), (anc_sig, pos_sig) = self.detector.run_model_siamese((anc_pc, pos_pc), (anc_sn, pos_sn),
                                                                               (anc_node, pos_node))
        neg_d = neg.pin_memory().to(self.device, non_blocking=True)
        info = {"anchors": np.asarray(anchors), "positives": np.asarray(pos), "neg_idx": neg,
                "clouds": (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node)}
        return (anc_pc, anc_sn, anc_kp, anc_sig, pos_pc, pos_sn, pos_kp, pos_sig, neg_d), info
