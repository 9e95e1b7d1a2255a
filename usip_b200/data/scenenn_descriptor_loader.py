"""The SceneNN descriptor loader on the GPU: data/scenenn_descriptor_loader.py (SceneNNDescriptorLoader) and the
training set of scenenn/train_descriptor.py, `SceneNNDescriptorLoader('train') + SceneNNDescriptorLoader('val')`.

Item i of a split is the frame pair pairs_np[i] = (anchor, positive) of info_<split>.pkl, both frames of
frames_<split>/; the test split keeps every third pair (`pairs_np[::3]`, icp_np alike).  Per item, in this draw order:
the anchor's N rows, the positive's (a fragment shorter than N is tiled, as draw_rows); the anchor is aligned to the
positive by hom2cart(icp_np[i] @ [x y z 1]) in float64 (its sn[:, 0:3] too, translation included, rounded to fp32);
FPS over N/2 candidates, candidates and start of the anchor (on its float64 ICP'd cloud), then of the positive; then one
augmentation shared by the pair's two clouds -- augment() for the train split (rotations, scale U(0.9, 1.1), shift; the
jitter is drawn but never applied), augment_rot_only() for val (the three rotations only), none for test -- and
transform_pc_pytorch on the positive (scale_thre 0.2, shift_thre 0.5).

`SceneNNDescriptorPairBuilder` builds the clouds on the device (csrc/pairgen.cu: the shared subset kernel, the float64
ICP'd candidate gather, usip_fps_f64 and usip_scenenn_desc_pair_augment).  `SceneNNDescriptorPairSource` feeds
`ModelDescriptorIndoor` from a SceneNN tree, keypoints and sigmas from a frozen `ModelDetector`, as the train script does.
"""
import os
import pickle

import numpy as np

from usip_b200 import ops

from .kitti_detector_loader import (_PairBuilder, _ScanSource, angles2rotation_matrix, draw_candidates,
                                    draw_pair_scalars, draw_rows)
from .scenenn_detector_loader import SCENENN_MODES

SCENENN_DESC_DIVISOR = 2                         # scenenn_descriptor_loader.py __getitem__: FPS over N/2 candidates
DESC_SCALE = (0.9, 1.1)                          # augment(): scale
DESC_PERTURBATION = (0.12, 0.36)                 # augment() / augment_rot_only(): perturbation angles
DESC_JITTER = ((0.01, 0.03), (0.01, 0.03), (0.015, 0.03))   # augment(): pc, sn, node -- drawn, never applied
DESC_SCALE_THRE = 0.2                            # transform_pc_pytorch's default scale_thre
MAX_S = 8                                        # usip_scenenn_desc_pair_augment
KIND_OF_SPLIT = {"train": ops.SCENENN_KIND_FULL, "val": ops.SCENENN_KIND_ROT, "test": ops.SCENENN_KIND_NONE}


def draw_rotations(rng):
    """The rotation draws of augment() and augment_rot_only(), in order -> (horizontal, 3-d, perturbation) matrices."""
    y_angle = rng.uniform() * 2 * np.pi
    angles_3d = rng.rand(3) * np.pi * 2
    angles_pertb = np.clip(DESC_PERTURBATION[0] * rng.randn(3), -DESC_PERTURBATION[1], DESC_PERTURBATION[1])
    return tuple(angles2rotation_matrix(a) for a in ([0, y_angle, 0], angles_3d, angles_pertb))


class SceneNNDescriptorPairBuilder(_PairBuilder):
    """Builds the nine cloud tensors of a batch of SceneNN descriptor pairs on the device: (anc_pc, anc_sn, anc_node,
    pos_pc, pos_sn, pos_node, R (B,3,3), scale (B,), shift (B,3,1)), all f32.

    `build(scans, offsets, anc_items, pos_items, icp, kinds, step=None)`: scans [T, C] f32 (device, or host -- then the
    items' scans are uploaded), offsets (n_scans+1,) int64 row offsets (host), anc_items / pos_items the scan index of
    every pair's two frames, icp (B, 4, 4) the matrix that aligns each anchor to its positive, kinds (B,) each pair's
    augmentation: ops.SCENENN_KIND_FULL (train split), _ROT (val) or _NONE (test).  See `_PairBuilder` for the two rng
    modes; rng="numpy" replays SceneNNDescriptorLoader.__getitem__ item by item, including the jitter draws augment()
    discards, and rng="device" draws no jitter at all.  `last` adds the FPS selection ("node_idx").
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device", divisor=SCENENN_DESC_DIVISOR):
        super().__init__(opt, mode, device, seed, rng, divisor)
        if not 3 <= self.S <= MAX_S:
            raise ValueError("surface_normal_len %d: the SceneNN descriptor loader ICPs sn[:, 0:3], so it takes 3 to %d"
                             " sn columns" % (self.S, MAX_S))
        self.flags &= ~ops.PAIR_TRAIN            # each pair's kind decides what it gets
        self._pending = None                     # kinds of the pairs still to be drawn in this build
        self._icp_h = self._icp = None           # this build's (B, 4, 4) f64 matrices, on the host and the device
        self._node_idx = None

    def _clouds(self, anc_items, pos_items):
        anc = np.asarray(anc_items, dtype=np.int64).ravel()
        pos = np.asarray(pos_items, dtype=np.int64).ravel()
        if anc.size == 0:
            raise ValueError("no items")
        if anc.shape != pos.shape:
            raise ValueError("%d anchors but %d positives" % (anc.size, pos.size))
        return np.stack([anc, pos], 1).ravel()                # cloud 2b = anchor b, 2b+1 = its positive

    def _draw(self, rng, per_point):
        # called once per pair, in pair order, in both rng modes
        kind = next(self._pending)
        rots = draw_rotations(rng) if kind == ops.SCENENN_KIND_ROT else None
        p, _ = draw_pair_scalars(rng, self.opt, kind == ops.SCENENN_KIND_FULL, self.N, self.M, self.S, per_point,
                                 DESC_SCALE, DESC_PERTURBATION, DESC_JITTER, DESC_SCALE_THRE)
        if rots is not None:
            for r, R in enumerate(rots):
                p[9 * r:9 * r + 9] = R.ravel()
        p[ops.PAIR_AUGMENT_SLOT] = float(kind)
        return p, None                           # the jitter is never applied: nothing to upload

    def _draw_item(self, rng, n_valid):
        """__getitem__: rows of the anchor and of the positive, then candidates and start of the anchor and of the
        positive, then the pair's augmentation and the transform."""
        rows = [draw_rows(rng, n, self.N) for n in n_valid]
        cands = [draw_candidates(rng, self.N, self.divisor) for _ in n_valid]
        return [(r,) + c for r, c in zip(rows, cands)], self._draw(rng, True)

    def _nodes(self, scans, offsets, scan_of_cloud, rows, cand, start, params_h, up):
        self._icp = up(self._icp_h)
        pts = ops.cloud_gather_candidates_icp_f64(scans, offsets, scan_of_cloud, rows, cand, self._icp)
        self._node_idx, _ = ops.fps_f64(pts, start, self.M)
        return pts, (pts, self._node_idx)

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        pts, idx = nodes
        return ops.scenenn_desc_pair_augment(scans, offsets, scan_of_cloud, rows, self._icp, pts, idx, params, self.S,
                                             self.flags)

    def build(self, scans, offsets, anc_items, pos_items, icp, kinds, step=None):
        n = np.asarray(anc_items).size
        icp = np.ascontiguousarray(icp, dtype=np.float64)
        if icp.shape != (n, 4, 4):
            raise ValueError("icp must be (%d, 4, 4), one matrix per pair; got %s" % (n, icp.shape))
        kinds = np.asarray(kinds).ravel()
        if kinds.shape != (n,):
            raise ValueError("kinds needs one entry per pair: %d for %d pairs" % (kinds.size, n))
        if not np.isin(kinds, list(KIND_OF_SPLIT.values())).all():
            raise ValueError("kinds must be SCENENN_KIND_NONE, _ROT or _FULL (0, 1, 2)")
        self._pending = iter(kinds.astype(np.int64).tolist())
        self._icp_h = icp
        try:
            out = self._build(scans, offsets, step, anc_items, pos_items)
            self.last["node_idx"] = self._node_idx
            return out
        finally:
            self._pending = self._icp_h = self._icp = self._node_idx = None


# ----------------------------------------------------------------------------------------------- SceneNN tree
def scenenn_pairs(root, split):
    """(pairs (n, 2) int64 frame indices, icp (n, 4, 4) f64) of one split, as SceneNNDescriptorLoader keeps them: the
    test split every third pair."""
    if split not in KIND_OF_SPLIT:
        raise ValueError("split must be 'train', 'val' or 'test'")
    with open(os.path.join(root, "info_%s.pkl" % split), "rb") as f:
        info = pickle.load(f)
    pairs = np.asarray(info["pairs_np"], dtype=np.int64).reshape(-1, 2)
    icp = np.asarray(info["icp_np"], dtype=np.float64).reshape(-1, 4, 4)
    if pairs.shape[0] != icp.shape[0]:
        raise ValueError("info_%s.pkl: %d pairs but %d ICP matrices" % (split, pairs.shape[0], icp.shape[0]))
    if split == "test":
        pairs, icp = pairs[::3], icp[::3]
    return pairs, icp


class SceneNNDescriptorPairSource(_ScanSource):
    """Shuffled batches of SceneNN descriptor training inputs, built on the device, for `ModelDescriptorIndoor`.

    mode: "train" (augmented), "val" (rotations only), "test" (pairs [::3], no augmentation) or "train+val", the train
    script's concatenation: train pairs first, then val pairs, each built with its own split's augmentation.  Only the
    frames the pairs name are loaded, from each split's folder.  resident: "host" (pinned), "device", or "disk" (each
    batch's frames are read when it is built).  For every batch, on the build stream: build the clouds
    (`SceneNNDescriptorPairBuilder`) and run the frozen `detector.run_model_siamese` on them and their nodes for the
    keypoints and sigmas.  The batch is the eleven `ModelDescriptorIndoor.set_input` tensors.

        src = SceneNNDescriptorPairSource(root, "train+val", opt, detector)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    disk_resident = True

    def __init__(self, root, mode, opt, detector, device=None, seed=0, resident="host", rng="device",
                 batch_size=None, drop_last=True):
        if mode not in SCENENN_MODES:
            raise ValueError("mode must be one of %s" % (SCENENN_MODES,))
        splits = ("train", "val") if mode == "train+val" else (mode,)
        self.split = mode
        paths, anc, pos, icp, kinds = [], [], [], [], []
        for split in splits:
            pairs, m = scenenn_pairs(root, split)
            frames = np.unique(pairs)
            local = np.searchsorted(frames, pairs) + len(paths)
            paths += [os.path.join(root, "frames_" + split, "%d.npy" % f) for f in frames]
            anc.append(local[:, 0]); pos.append(local[:, 1]); icp.append(m)
            kinds.append(np.full(len(pairs), KIND_OF_SPLIT[split], dtype=np.int64))
        self.anc, self.pos = np.concatenate(anc), np.concatenate(pos)
        self.icp, self.kinds = np.concatenate(icp), np.concatenate(kinds)
        if self.anc.size == 0:
            raise ValueError("no pairs under %s for %s" % (root, mode))
        super().__init__(paths, "test" if mode == "test" else "train", opt, SceneNNDescriptorPairBuilder, device, seed,
                         resident, rng, batch_size, drop_last, n_items=self.anc.size)
        self.detector = detector

    def _build(self, items):
        items = np.asarray(items, dtype=np.int64)
        scans, offsets, idx = self._batch_scans(np.stack([self.anc[items], self.pos[items]], 1))
        anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node, R, scale, shift = self.builder.build(
            scans, offsets, idx[:, 0], idx[:, 1], self.icp[items], self.kinds[items], step=self.step)
        (anc_kp, pos_kp), (anc_sig, pos_sig) = self.detector.run_model_siamese((anc_pc, pos_pc), (anc_sn, pos_sn),
                                                                               (anc_node, pos_node))
        info = {"items": items, "kinds": self.kinds[items], "clouds": (anc_pc, anc_sn, anc_node, pos_pc, pos_sn, pos_node),
                "rows": self.builder.last["rows"]}
        return (anc_pc, anc_sn, anc_kp, anc_sig, pos_pc, pos_sn, pos_kp, pos_sig, R, scale, shift), info
