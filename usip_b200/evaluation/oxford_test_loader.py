"""The Oxford test-set loader on the GPU: evaluation/oxford_test_loader.py (OxfordTestLoader).

Item i is the ENU scan test_models_20k_np_nofilter/<number>.npy, number = i by default (the reference's 828 test
scans).  Its draws are the KITTI test loader's with FPS over int(input_pc_num / 3) candidates; then pc, sn columns 0:3
and the nodes go to the camera frame, (x, y, z) -> (x, -z, y).  The frame change comes after FPS, so FPS runs on the
ENU candidates, as in the reference; it is exact, so the nodes are the same points either way.  See
kitti_test_loader._TestCloudSource for the batches and the rng modes.
"""
import os

import numpy as np

from usip_b200 import ops
from usip_b200.data.oxford_detector_loader import OXFORD_TEST_FOLDER, oxford_test_path, synthetic_enu_scan

from .kitti_test_loader import _TestCloudSource, random_rigid

OXFORD_TEST_SCANS = 828                           # oxford_test_loader.py:43-44


class OxfordTestLoader(_TestCloudSource):
    """evaluation/oxford_test_loader.py OxfordTestLoader over root; `numbers` the scan numbers of the items
    (default 0 .. 827)."""

    divisor = 3                                   # oxford_test_loader.py:85
    flags = ops.PAIR_ENU_TO_CAM

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=8, numbers=None):
        self.numbers = list(range(OXFORD_TEST_SCANS)) if numbers is None else [int(n) for n in numbers]
        if not self.numbers:
            raise ValueError("no test scans")
        super().__init__([oxford_test_path(root, n) for n in self.numbers], opt, device, seed, rng, batch_size)

    def key(self, i):
        return self.numbers[i]

    def keypoint_path(self, out_dir, i):
        """save_keypoints.py:371-374."""
        return os.path.join(out_dir, "%d.bin" % self.numbers[i])


def write_synthetic_oxford_test(root, numbers, rows, pairs, gt_path, seed=0):
    """An Oxford-shaped test tree for tests and benchmarks: root/test_models_20k_np_nofilter/%d.npy for every number,
    (rows, 8) float32 ENU from synthetic_enu_scan, and gt_path (groundtruths.txt: a header, then anc, pos, two file
    names, t and q (w, x, y, z) tab-separated) for the (anc, pos) pairs, T_gt random and rigid (identity when
    anc == pos)."""
    os.makedirs(os.path.join(root, OXFORD_TEST_FOLDER), exist_ok=True)
    for i, n in enumerate(numbers):
        np.save(oxford_test_path(root, n), synthetic_enu_scan(seed + i, rows))
    rng = np.random.RandomState(seed)
    lines = ["anc\tpos\tanc_file\tpos_file\tt1\tt2\tt3\tqw\tqx\tqy\tqz\n"]
    for a, p in pairs:
        t, q = (np.zeros(3), np.array([1.0, 0, 0, 0])) if a == p else random_rigid(rng)
        lines.append("\t".join([str(a), str(p), "%d.bin" % a, "%d.bin" % p] + ["%.6f" % v for v in np.concatenate([t, q])])
                     + "\n")
    with open(gt_path, "w") as f:
        f.write("".join(lines))
