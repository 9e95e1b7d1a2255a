"""The SceneNN detector loader on the GPU: data/scenenn_detector_loader.py (SceneNNDetectorLoader) and the training set
of scenenn/train_detector.py:54-61, `SceneNNDetectorLoader('train') + SceneNNDetectorLoader('val')`.

The loader is the 3DMatch detector loader (match3d_detector_loader.py) with its own listing -- item i of a split is
frames_<split>/<i>.npy for i < sample_num of info_<split>.pkl (:58-73) -- and FPS over N/4 candidates (:166-171).  It
augments only when mode == 'train' (:173), so the train script's shuffled batches mix augmented train items with val
items that get only the dst transform and make no augmentation draws.  `SceneNNPairSource(root, "train+val", opt)`
builds exactly those batches, through the shared `IndoorPairBuilder`'s per-pair switch.
"""
import os
import pickle

import numpy as np

from .match3d_detector_loader import _IndoorSource

SCENENN_DIVISOR = 4                              # scenenn_detector_loader.py:166-171: FPS over N/4 candidates
SCENENN_MODES = ("train", "val", "test", "train+val")


def scenenn_sample_num(root, split):
    """sample_num of info_<split>.pkl (scenenn_detector_loader.py:61-67), the dataset's own pickle."""
    with open(os.path.join(root, "info_%s.pkl" % split), "rb") as f:
        return int(pickle.load(f)["sample_num"])


def make_scenenn_dataset(root, split):
    """The fragment paths of one split: frames_<split>/<i>.npy for i < sample_num (:58-73)."""
    if split not in ("train", "val", "test"):
        raise ValueError("split must be 'train', 'val' or 'test'")
    return [os.path.join(root, "frames_" + split, "%d.npy" % i) for i in range(scenenn_sample_num(root, split))]


def write_synthetic_scenenn(root, counts, rows, seed=0, pairs=None):
    """A SceneNN tree for tests and benchmarks: for every split of counts {split: n}, frames_<split>/<i>.npy for i < n,
    synthetic_fragment of rows(split, i) rows (rows may also be an int), and info_<split>.pkl with the keys the
    reference reads (sample_num = n; pairs_np, icp_np and positive_list empty).

    pairs {split: [(anchor, positive), ...]} (optional) fills pairs_np and icp_np of those splits for the descriptor
    loader.  Each positive frame is then rewritten as the rigid image of its anchor frame, row for row: xyz =
    fl32(R x + t), sn[0:3] = fl32(R n), the other columns copied, with (R, t) drawn from the split's seed, and icp_np[k] =
    [[R, t], [0, 0, 0, 1]], the transform that aligns the anchor to the positive.  A positive may not be an anchor or
    the positive of another pair."""
    from usip_b200.evaluation.indoor_test_loader import synthetic_fragment
    from .kitti_detector_loader import angles2rotation_matrix
    pairs = pairs or {}
    for s, (split, n) in enumerate(counts.items()):
        folder = os.path.join(root, "frames_" + split)
        os.makedirs(folder, exist_ok=True)
        for i in range(n):
            k = rows if np.isscalar(rows) else rows(split, i)
            np.save(os.path.join(folder, "%d.npy" % i), synthetic_fragment(seed + 1000 * s + i, k))
        pairs_np = np.asarray(pairs.get(split, []), dtype=np.int64).reshape(-1, 2)
        if len(np.unique(pairs_np[:, 1])) != len(pairs_np) or np.isin(pairs_np[:, 1], pairs_np[:, 0]).any():
            raise ValueError("%s: a positive frame may be the positive of one pair only, and no anchor" % split)
        icp_np = np.zeros((len(pairs_np), 4, 4))
        r = np.random.RandomState(seed + 7919 * (s + 1))
        for k, (a, p) in enumerate(pairs_np):
            T = np.eye(4)
            T[0:3, 0:3] = angles2rotation_matrix(r.uniform(0, 2 * np.pi, 3))
            T[0:3, 3] = r.uniform(-1, 1, 3)
            frag = np.load(os.path.join(folder, "%d.npy" % a))
            img = frag.copy()
            img[:, 0:3] = (frag[:, 0:3].astype(np.float64) @ T[0:3, 0:3].T + T[0:3, 3]).astype(np.float32)
            img[:, 3:6] = (frag[:, 3:6].astype(np.float64) @ T[0:3, 0:3].T).astype(np.float32)
            np.save(os.path.join(folder, "%d.npy" % p), img)
            icp_np[k] = T
        info = {"pairs_np": pairs_np, "icp_np": icp_np, "positive_list": [], "sample_num": n}
        with open(os.path.join(root, "info_%s.pkl" % split), "wb") as f:
            pickle.dump(info, f)


class SceneNNPairSource(_IndoorSource):
    """Shuffled batches of SceneNN detector pairs, built on the device and handed to `ModelDetector` (see
    `_ScanSource`).  mode: "train" (augmented), "val" (dst transform only), "test", or "train+val", the train script's
    concatenation: train items first, then val items, which are built without augmentation (`augment_mask`).
    resident: "host" (pinned), "device", or "disk".

        src = SceneNNPairSource(root, "train+val", opt)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, device=None, seed=0, resident="host", rng="device", batch_size=None,
                 drop_last=True):
        if mode not in SCENENN_MODES:
            raise ValueError("mode must be one of %s" % (SCENENN_MODES,))
        splits = ("train", "val") if mode == "train+val" else (mode,)
        self.split = mode
        self.dataset, augment = [], []
        for split in splits:
            paths = make_scenenn_dataset(root, split)
            self.dataset += paths
            augment += [split == "train"] * len(paths)
        super().__init__(self.dataset, "test" if mode == "test" else "train", opt, SCENENN_DIVISOR, device, seed,
                         resident, rng, batch_size, drop_last, augment=augment)
