"""The KITTI test-set loader on the GPU: evaluation/kitti_test_loader.py (KittiTestLoader, make_kitti_test_dataset).

Each item is one scan of the test list, as the detector sees it at evaluation time: input_pc_num rows drawn without
replacement, FPS nodes over int(input_pc_num / 4) of them, no augmentation and no pair.  `_TestCloudSource` builds a
batch of such clouds on the device with the per-cloud steps of the pair builders (usip_cloud_subsample,
usip_cloud_gather_candidates, usip_fps_f32) and usip_test_cloud_gather, which also adds save_keypoints.py:275's noise.
The Oxford loader (oxford_test_loader.py) builds on the same base.

Two rng modes, as the pair builders have:
  rng="device": rows, FPS candidates and start, and the noise are Philox keyed by (seed, step, cloud, point, purpose),
    step = the batch's number; the same seed gives the same bits.
  rng="numpy": parity mode.  Consumes the global np.random item by item in the reference's order (rows, FPS candidates,
    FPS start) and, for the noise, torch's CPU generator once per batch (torch.randn of the batch's pc shape): with the
    reference's batch size it reproduces save_keypoints.py's clouds.  Slow by design.
"""
import os

import numpy as np
import torch

from usip_b200 import ops
from usip_b200.data.kitti_detector_loader import FPS_MAX_CANDIDATES, KITTI_NP_FOLDER, draw_subsample, load_scan_npy

TEST_SN_LEN = 4                                   # kitti_test_loader.py:120, oxford_test_loader.py:76


def load_kitti_test_gt_txt(txt_root, seq):
    """kitti_test_loader.py:24-58: the scans of <txt_root>/<seq>/groundtruths.txt (one header line), in file order.
    A line adds its anc unless an entry already has anc_idx == anc, and its pos as an entry of its own unless an entry
    has anc_idx == pos.  -> [{'seq', 'anc_idx', 'pos_idx'}]"""
    dataset = []
    with open(os.path.join(txt_root, "%02d" % seq, "groundtruths.txt")) as f:
        lines = f.readlines()
    for line in lines[1:]:
        parts = line.split()
        if not parts:
            continue
        anc, pos = int(parts[0]), int(parts[1])
        have = {d["anc_idx"] for d in dataset}
        if anc not in have:
            dataset.append({"seq": seq, "anc_idx": anc, "pos_idx": pos})
        if pos not in have:
            dataset.append({"seq": seq, "anc_idx": pos, "pos_idx": anc})
    return dataset


def make_kitti_test_dataset(txt_root):
    """kitti_test_loader.py:61-71: every sequence folder of txt_root in sorted order."""
    dataset = []
    for seq in sorted(int(x) for x in sorted(os.listdir(txt_root))):
        dataset += load_kitti_test_gt_txt(txt_root, seq)
    return dataset


class _TestCloudSource:
    """Batches of test clouds built on the device.  A subclass lists the scan files (`paths`), names each item's
    keypoint file (`keypoint_path`) and the key its ground truth uses (`key`), and sets the FPS candidate divisor, the
    frame flags, the surface-normal length sn_len (columns 3:3+sn_len) and whether a scan may be shorter than
    input_pc_num (allow_short: every row is taken t times, then a random remainder, as usip_cloud_subsample and
    draw_subsample do).  `build(items)` -> (pc (B,3,N), sn (B,sn_len,N), node (B,3,M)) f32, fresh tensors on the
    current stream; nothing synchronises with the host."""

    divisor = 4
    flags = 0
    sn_len = TEST_SN_LEN
    allow_short = False

    def __init__(self, paths, opt, device, seed, rng, batch_size):
        if int(opt.surface_normal_len) != self.sn_len:
            raise ValueError("surface_normal_len must be %d for this test loader, got %d"
                             % (self.sn_len, int(opt.surface_normal_len)))
        if rng not in ("device", "numpy"):
            raise ValueError("rng must be 'device' or 'numpy'")
        self.opt, self.paths, self.rng, self.seed = opt, list(paths), rng, int(seed)
        self.device = torch.device(device if device is not None else "cuda")
        self.N, self.M, self.S = int(opt.input_pc_num), int(opt.node_num), self.sn_len
        self.n_cand = int(self.N / self.divisor)
        if self.n_cand > FPS_MAX_CANDIDATES:
            raise ValueError("input_pc_num / %d = %d FPS candidates; usip_fps_f32 takes at most %d"
                             % (self.divisor, self.n_cand, FPS_MAX_CANDIDATES))
        if self.n_cand < 1 or self.M > self.n_cand:
            raise ValueError("node_num %d needs at least as many FPS candidates (%d)" % (self.M, self.n_cand))
        self.batch_size = int(batch_size)
        if self.batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        self.step = 0
        self.last = None                      # index lists of the last build, for inspection

    def __len__(self):
        return len(self.paths)

    def key(self, i):
        raise NotImplementedError

    def keypoint_path(self, out_dir, i):
        raise NotImplementedError

    def load(self, items):
        """The items' scans as (Ns, C) float32 arrays.  Unless allow_short, a scan shorter than input_pc_num raises
        ValueError (the reference draws its rows without replacement and has no fill); an empty scan always does."""
        arrs = [load_scan_npy(self.paths[i], self.S) for i in items]
        for i, a in zip(items, arrs):
            if len(a) == 0 or (len(a) < self.N and not self.allow_short):
                raise ValueError("scan %s (%s) has %d rows; input_pc_num = %d rows are drawn without replacement"
                                 % (self.key(i), self.paths[i], len(a), self.N))
        if len({a.shape[1] for a in arrs}) != 1:
            raise ValueError("scans differ in column count")
        return arrs

    def draw_item(self, rng, n_rows):
        """Parity mode: one item's draws in the reference's order -> (rows, FPS candidates, FPS start)."""
        return draw_subsample(rng, n_rows, self.N, self.divisor)

    def build(self, items, noise_sigma=0.0, step=None):
        items = [int(i) for i in np.asarray(items, dtype=np.int64).ravel()]
        if not items:
            raise ValueError("no items")
        if min(items) < 0 or max(items) >= len(self):
            raise IndexError("item out of range")
        if step is None:
            step = self.step
        self.step = int(step) + 1
        arrs = self.load(items)
        B, N, dev = len(items), self.N, self.device
        # the per-cloud steps take clouds in pairs: an odd batch repeats its last scan, whose outputs are dropped
        soc = np.arange(B, dtype=np.int32)
        if B % 2:
            soc = np.concatenate([soc, soc[-1:]])
        offsets = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)
        with torch.cuda.device(dev):
            scans = up(np.concatenate(arrs))
            offsets_d, soc_d = up(offsets), up(soc)
            noise = None
            if self.rng == "device":
                rows, cand, start, _ = ops.cloud_subsample(scans, offsets_d, soc_d, int(np.diff(offsets).max()), N,
                                                           self.n_cand, None, self.seed, step)
            else:
                drawn = [self.draw_item(np.random, len(a)) for a in arrs]
                drawn += drawn[-1:] * (len(soc) - B)
                rows = up(np.stack([d[0] for d in drawn]).astype(np.int32))
                cand = up(np.stack([d[1] for d in drawn]).astype(np.int32))
                start = up(np.array([d[2] for d in drawn], dtype=np.int32))
                if noise_sigma:
                    noise = torch.randn((B, 3, N)).pin_memory().to(dev, non_blocking=True)   # save_keypoints.py:275
            pts = ops.cloud_gather_candidates(scans, offsets_d, soc_d, rows, cand)
            _, nodes = ops.fps(pts, start, self.M, want_nodes=True)
            out = ops.test_cloud_gather(scans, offsets_d, soc_d[:B], rows[:B], nodes[:B], self.S, self.flags,
                                        noise_sigma, noise, self.seed, step)
        self.last = {"rows": rows[:B], "cand": cand[:B], "start": start[:B], "candidates": pts[:B]}
        return out

    def batches(self, noise_sigma=0.0):
        """The test set in order, batch_size items at a time: (items, (pc, sn, node)); the step is the batch number."""
        for b, i in enumerate(range(0, len(self), self.batch_size)):
            items = list(range(i, min(i + self.batch_size, len(self))))
            yield items, self.build(items, noise_sigma, step=b)


class KittiTestLoader(_TestCloudSource):
    """evaluation/kitti_test_loader.py KittiTestLoader: the scans of make_kitti_test_dataset(txt_root), read from
    numpy_root/%02d/np_0.20_20480_r90_sn/%06d.npy; sn = columns 3:7.  See `_TestCloudSource` for the rng modes."""

    divisor = 4                                   # kitti_test_loader.py:130

    def __init__(self, txt_root, numpy_root, opt, device=None, seed=0, rng="device", batch_size=8):
        self.dataset = make_kitti_test_dataset(txt_root)
        if not self.dataset:
            raise ValueError("no scans listed under %s" % txt_root)
        paths = [os.path.join(numpy_root, "%02d" % d["seq"], KITTI_NP_FOLDER, "%06d.npy" % d["anc_idx"])
                 for d in self.dataset]
        super().__init__(paths, opt, device, seed, rng, batch_size)

    def key(self, i):
        return (self.dataset[i]["seq"], self.dataset[i]["anc_idx"])

    def keypoint_path(self, out_dir, i):
        """save_keypoints.py:367-370."""
        return os.path.join(out_dir, "%02d" % self.dataset[i]["seq"], "%06d.bin" % self.dataset[i]["anc_idx"])


def random_rigid(rng):
    """A random rigid motion for synthetic ground truth: t (3,) within +-5, q (w, x, y, z) unit, w > 0."""
    q = rng.normal(size=4)
    q = q / np.linalg.norm(q) * np.sign(q[0])
    return rng.uniform(-5, 5, 3), q


def write_synthetic_kitti_test(txt_root, numpy_root, calib_root, counts, rows, pairs, seed=0):
    """A KITTI-shaped test tree for tests and benchmarks.  Sequence s has counts[s] scans numpy_root/%02d/
    np_0.20_20480_r90_sn/%06d.npy, (rows, 8) float32 from synthetic_scan; pairs[s] lists its (idx1, idx2) ground-truth
    pairs, written to txt_root/%02d/groundtruths.txt (the test list) and correct_gt.txt with a random rigid T_gt (the
    identity when idx1 == idx2); calib_root/%02d/calib.txt holds P0..P3 and a random rigid Tr."""
    from usip_b200.data.kitti_detector_loader import synthetic_scan
    from .repeatability import quat2rotm
    rng = np.random.RandomState(seed)
    for s, n in enumerate(counts):
        folder = os.path.join(numpy_root, "%02d" % s, KITTI_NP_FOLDER)
        os.makedirs(folder, exist_ok=True)
        for i in range(n):
            np.save(os.path.join(folder, "%06d.npy" % i), synthetic_scan(seed + 1000 * s + i, rows))
        os.makedirs(os.path.join(txt_root, "%02d" % s), exist_ok=True)
        lines, correct = ["idx1 idx2 t1 t2 t3 qw qx qy qz\n"], ["idx1,idx2,t1,t2,t3,qw,qx,qy,qz\n"]
        for a, p in pairs[s]:
            t, q = (np.zeros(3), np.array([1.0, 0, 0, 0])) if a == p else random_rigid(rng)
            vals = [a, p] + ["%.6f" % v for v in np.concatenate([t, q])]
            lines.append(" ".join(map(str, vals)) + "\n")
            correct.append(",".join(map(str, vals)) + "\n")
        with open(os.path.join(txt_root, "%02d" % s, "groundtruths.txt"), "w") as f:
            f.write("".join(lines))
        with open(os.path.join(txt_root, "%02d" % s, "correct_gt.txt"), "w") as f:
            f.write("".join(correct))
        t, q = random_rigid(rng)
        Tr = np.concatenate([quat2rotm(q), t.reshape(3, 1)], axis=1)
        os.makedirs(os.path.join(calib_root, "%02d" % s), exist_ok=True)
        with open(os.path.join(calib_root, "%02d" % s, "calib.txt"), "w") as f:
            P = " ".join(["%.12e" % v for v in np.eye(3, 4).ravel()])
            f.write("".join("P%d: %s\n" % (k, P) for k in range(4)))
            f.write("Tr: %s\n" % " ".join("%.12e" % v for v in Tr.ravel()))
