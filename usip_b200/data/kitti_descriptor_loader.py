"""The KITTI descriptor loader on the GPU: data/kitti_descriptor_loader.py (KittiDescriptorLoader) and the batch
preparation of kitti/train_descriptor.py:94-132.

The descriptor is trained on keypoints of the frozen detector.  Each item is an anchor scan and a positive scan
within `positive_radius_threshold` of it, both subsampled, given FPS nodes and augmented; the frozen detector turns
every cloud into keypoints and sigmas, and the negatives are other anchors of the batch more than
`negative_radius_threshold` away.  `DescriptorPairBuilder` builds the clouds on the device (csrc/pairgen.cu: the
subset and candidate kernels of the detector builder with one scan per cloud, and `usip_desc_pair_augment`);
`KittiDescriptorPairSource` adds the positive search, the frozen detector pass and negative mining, and hands the nine
`ModelDescriptor.set_input` tensors over without a host synchronise.
"""
import os
import random
import warnings

import numpy as np
import torch

from usip_b200 import ops

from .kitti_detector_loader import (FPS_MAX_CANDIDATES, _step_rng, angles2rotation_matrix, draw_subsample,
                                    kitti_scan_path, load_scan_npy, make_dataset_kitti)

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
class DescriptorPairBuilder:
    """Builds the six cloud tensors (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node) of a batch of KITTI
    descriptor pairs on the device.

    `build(scans, offsets, anc_items, pos_items, step=None)`: scans [T, C] f32 (device, or host -- then the items'
    scans are uploaded), offsets (n_scans+1,) int64 row offsets (host), anc_items / pos_items the scan index of every
    anchor and positive.  Every scan needs at least input_pc_num rows: the reference draws them without replacement.

    rng="device": per-point randomness is Philox keyed by (seed, step, cloud, point, purpose), per-pair scalars come
    from a numpy RandomState seeded by (seed, step): a batch is a pure function of (seed, step), with O(B) host work.
    Selected rows ascend (see usip_cloud_subsample in include/usip_b200.h).
    rng="numpy": parity mode.  Consumes the global np.random exactly as KittiDescriptorLoader.__getitem__ does, item by
    item (anchor rows, candidates, FPS start; positive the same; then the augmentation), and uploads the index lists and
    jitter arrays.  The positive search draws from Python's `random` only, so choosing pos_items beforehand with
    `nearby_index` changes no numpy draw.

    The outputs are fresh tensors allocated on the current stream.  `last` keeps the index lists of the last build.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device"):
        if mode not in ("train", "test"):
            raise ValueError("mode must be 'train' or 'test'")
        if rng not in ("device", "numpy"):
            raise ValueError("rng must be 'device' or 'numpy'")
        self.opt, self.mode, self.rng, self.seed = opt, mode, rng, int(seed)
        self.device = torch.device(device if device is not None else "cuda")
        self.N, self.M, self.S = int(opt.input_pc_num), int(opt.node_num), int(opt.surface_normal_len)
        self.n_cand = int(self.N / DESC_DIVISOR)
        if self.n_cand > FPS_MAX_CANDIDATES:
            raise ValueError("input_pc_num / %d = %d FPS candidates; usip_fps_f32 takes at most %d"
                             % (DESC_DIVISOR, self.n_cand, FPS_MAX_CANDIDATES))
        if self.n_cand < 1 or self.M > self.n_cand:
            raise ValueError("node_num %d needs at least as many FPS candidates (%d)" % (self.M, self.n_cand))
        if not 1 <= self.S <= 8:
            raise ValueError("surface_normal_len %d: the augment kernel takes 1..8" % self.S)
        self.flags = ((ops.PAIR_TRAIN if mode == "train" else 0)
                      | (ops.PAIR_ROT_HORIZONTAL if getattr(opt, "rot_horizontal", False) else 0)
                      | (ops.PAIR_ROT_3D if getattr(opt, "rot_3d", False) else 0)
                      | (ops.PAIR_ROT_PERTURBATION if getattr(opt, "rot_perturbation", False) else 0)
                      | (ops.PAIR_TRANSLATION if getattr(opt, "translation_perturbation", False) else 0))
        self.step = 0
        self.last = None

    def _check(self, scans, offsets, anc_items, pos_items):
        offsets = np.asarray(offsets, dtype=np.int64)
        if offsets.ndim != 1 or offsets.shape[0] < 2:
            raise ValueError("no scans")
        anc = np.asarray(anc_items, dtype=np.int64).ravel()
        pos = np.asarray(pos_items, dtype=np.int64).ravel()
        if anc.size == 0:
            raise ValueError("no items")
        if anc.shape != pos.shape:
            raise ValueError("%d anchors but %d positives" % (anc.size, pos.size))
        clouds = np.stack([anc, pos], 1).ravel()              # cloud 2b = anchor b, 2b+1 = its positive
        if clouds.min() < 0 or clouds.max() >= offsets.shape[0] - 1:
            raise IndexError("item out of range")
        lengths = offsets[clouds + 1] - offsets[clouds]
        k = int(np.argmin(lengths))
        if lengths[k] <= 0:
            raise ValueError("scan %d has no points" % int(clouds[k]))
        if lengths[k] < self.N:
            raise ValueError("scan %d has %d rows; input_pc_num = %d rows are drawn without replacement"
                             % (int(clouds[k]), int(lengths[k]), self.N))
        C = scans.shape[1]
        if scans.dim() != 2 or C < 3 + self.S:
            raise ValueError("scans have %d columns, surface_normal_len %d needs %d" % (C, self.S, 3 + self.S))
        max_rows = int(lengths.max())
        if max_rows > ops.pair_max_scan_rows():
            raise ValueError("a scan of %d rows exceeds the %d the subsample kernel holds"
                             % (max_rows, ops.pair_max_scan_rows()))
        return offsets, clouds, lengths, max_rows

    def build(self, scans, offsets, anc_items, pos_items, step=None):
        offsets, clouds, lengths, max_rows = self._check(scans, offsets, anc_items, pos_items)
        if step is None:
            step = self.step
        self.step = int(step) + 1
        B, N, M, S, dev = len(clouds) // 2, self.N, self.M, self.S, self.device
        train = self.mode == "train"

        host_scans = None
        if self.rng == "numpy":
            host_scans = [scans[offsets[i]:offsets[i + 1]].cpu().numpy() for i in clouds]
        if scans.device != dev:                        # upload only the scans this batch uses, each once
            uniq, inv = np.unique(clouds, return_inverse=True)
            parts = [scans[offsets[i]:offsets[i + 1]] for i in uniq]
            scans = torch.cat(parts).pin_memory().to(dev, non_blocking=True)
            offsets = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
            clouds = inv.astype(np.int64).ravel()
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)
        offsets_d = up(offsets)
        scan_of_cloud = up(clouds.astype(np.int32))

        jit = (None, None, None)
        with torch.cuda.device(dev):
            if self.rng == "device":
                rows, cand, start = ops.cloud_subsample(scans, offsets_d, scan_of_cloud, max_rows, N, self.n_cand,
                                                        self.seed, step)
                hrng = _step_rng(self.seed, step)
                drawn = [draw_desc_pair_scalars(hrng, train, N, M, S, False) for _ in range(B)]
            else:
                rows_h = np.empty((2 * B, N), np.int32)
                cand_h = np.empty((2 * B, self.n_cand), np.int32)
                start_h = np.empty((2 * B,), np.int32)
                drawn = []
                for b in range(B):                     # KittiDescriptorLoader.__getitem__, item by item
                    for side in range(2):              # anchor, then positive (:321-323)
                        c = 2 * b + side
                        rows_h[c], cand_h[c], start_h[c] = draw_subsample(np.random, len(host_scans[c]), N,
                                                                          DESC_DIVISOR)
                    drawn.append(draw_desc_pair_scalars(np.random, train, N, M, S, True))
                rows, cand, start = up(rows_h), up(cand_h), up(start_h)
                if train:
                    jit = tuple(up(np.stack([d[2][k] for d in drawn]).reshape((2 * B,) + drawn[0][2][k].shape[1:]))
                                for k in range(3))
            params = up(np.concatenate([d[0] for d in drawn]))
            scale = up(np.array([d[1] for d in drawn], dtype=np.float64))
            pts = ops.cloud_gather_candidates(scans, offsets_d, scan_of_cloud, rows, cand)
            _, nodes = ops.fps(pts, start, M, want_nodes=True)
            out = ops.desc_pair_augment(scans, offsets_d, scan_of_cloud, rows, nodes, params, scale, S, self.flags,
                                        self.seed, step, *jit)
        self.last = {"rows": rows, "cand": cand, "start": start, "candidates": pts, "params": params, "scale": scale}
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


class KittiDescriptorPairSource:
    """Shuffled batches of KITTI descriptor training inputs, built on the device, for `ModelDescriptor`.

    Scans are indexed like make_dataset_kitti and loaded once into pinned host memory (or onto the device with
    resident="device"), the poses once into a host array.  For every batch, on a stream of its own: shuffle the
    anchors, pick each positive with `nearby_index` (host, Python's random), build the clouds (`DescriptorPairBuilder`),
    run the frozen `detector.run_model_siamese` on the built nodes for keypoints and sigmas, and mine the negatives
    (host, float32 poses).  Batch i+1 is built while the caller runs step i; `feed()` hands each batch over with
    `model.prefetch_input(..., after=event)` + `set_input()`, so the host never synchronises.

        src = KittiDescriptorPairSource(root, "train", opt, detector)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, detector, device=None, seed=0, resident="host", rng="device",
                 batch_size=None, drop_last=True):
        self.opt, self.mode, self.detector = opt, mode, detector
        self.device = torch.device(device if device is not None else "cuda")
        self.batch_size = int(batch_size or opt.batch_size)
        self.drop_last = drop_last
        self.pos_threshold = float(getattr(opt, "positive_radius_threshold", 5.0))
        self.neg_threshold = float(getattr(opt, "negative_radius_threshold", 50.0))
        _, _, self.nums, self.accs = make_dataset_kitti(root, mode)
        n = self.accs[-1] if self.accs else 0
        if n == 0:
            raise ValueError("no scans under %s" % root)
        arrs = [load_scan_npy(kitti_scan_path(root, mode, i), opt.surface_normal_len) for i in range(n)]
        if len({a.shape[1] for a in arrs}) != 1:
            raise ValueError("scans differ in column count")
        self.seq, self.poses = load_kitti_poses(root, mode)
        self.offsets = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
        scans = torch.from_numpy(np.concatenate(arrs))
        self.scans = scans.to(self.device) if resident == "device" else scans.pin_memory()
        self.builder = DescriptorPairBuilder(opt, mode, self.device, seed, rng)
        self.order_rng = np.random.RandomState(seed)
        self.pos_rng = random.Random(seed)
        self.neg_rng = np.random.RandomState(seed + 1)
        self.stream = torch.cuda.Stream(device=self.device)
        self.step = 0
        self.last = None                        # what the batch last yielded was built from, for inspection

    def __len__(self):
        n = len(self.offsets) - 1
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _build(self, anchors):
        pos = [nearby_index(int(a), self.poses, self.accs, self.nums, self.pos_threshold, self.pos_rng)
               for a in anchors]
        neg = mine_negative_sample(self.seq[anchors], self.poses[anchors].astype(np.float32), self.neg_threshold,
                                   self.neg_rng)
        with torch.cuda.stream(self.stream):
            anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node = self.builder.build(self.scans, self.offsets, anchors,
                                                                                    pos, step=self.step)
            (anc_kp, pos_kp), (anc_sig, pos_sig) = self.detector.run_model_siamese((anc_pc, pos_pc), (anc_sn, pos_sn),
                                                                                   (anc_node, pos_node))
            neg_d = neg.pin_memory().to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.step += 1
        info = {"anchors": np.asarray(anchors), "positives": np.asarray(pos), "neg_idx": neg,
                "clouds": (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node)}
        return (anc_pc, anc_sn, anc_kp, anc_sig, pos_pc, pos_sn, pos_kp, pos_sig, neg_d), ev, info

    def batches(self):
        """One shuffled epoch of (nine set_input tensors, ready event); batch i+1 is enqueued before batch i is
        yielded."""
        perm = self.order_rng.permutation(len(self.offsets) - 1)
        chunks = [perm[i:i + self.batch_size] for i in range(0, len(perm), self.batch_size)]
        if self.drop_last and chunks and len(chunks[-1]) < self.batch_size:
            chunks.pop()
        nxt = self._build(chunks[0]) if chunks else None
        for k in range(len(chunks)):
            out, ev, self.last = nxt
            nxt = self._build(chunks[k + 1]) if k + 1 < len(chunks) else None
            yield out, ev

    def feed(self, model):
        """One epoch; before each yield the batch is the model's input (prefetch_input + set_input)."""
        for out, ev in self.batches():
            model.prefetch_input(*out, after=ev)
            model.set_input(*out)
            yield out
