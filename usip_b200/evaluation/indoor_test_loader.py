"""The Redwood and 3DMatch test sets on the GPU: evaluation/redwood_loader.py (RedwoodLoader) and
data/match3d_eval_loader.py (Match3DEvalLoader, make_dataset_3dmatch_eval).

Both draw input_pc_num rows of a fragment, sn = columns 3:7, and FPS nodes over int(input_pc_num / 2) of the rows; both
name an item by (scene, frame) and write its keypoints to <out>/<scene>/<frame>.bin (save_keypoints.py:379-382).
Redwood: <root>/<scene>/%d.npy for the scenes livingroom1, livingroom2, office1 and office2 with 57, 47, 53 and 50
frames, in that order; a fragment shorter than input_pc_num is taken whole t times, then a random remainder
(redwood_loader.py:76-83).  3DMatch: <root>/<scene>/cloud_bin_<k>.npy for the reference's eight scenes, frame =
int(name[10:-4]); a shorter fragment is refused.  Fragments may be longer than usip_cloud_subsample's one-CTA limit: the
cluster kernel then draws their rows.

The reference lists a 3DMatch scene with os.listdir, whose order is arbitrary.  Here a scene's files are sorted by frame
number unless an explicit listing is given (`files`), which parity mode needs to replay the reference's draws.  See
kitti_test_loader._TestCloudSource for the batches and the rng modes.
"""
import os

import numpy as np

from .kitti_test_loader import _TestCloudSource

REDWOOD_SCENES = (("livingroom1", 57), ("livingroom2", 47), ("office1", 53), ("office2", 50))   # redwood_loader.py:62-64
MATCH3D_SCENES = ("7-scenes-redkitchen", "sun3d-home_at-home_at_scan1_2013_jan_1",
                  "sun3d-home_md-home_md_scan9_2012_sep_30", "sun3d-hotel_uc-scan3",
                  "sun3d-hotel_umd-maryland_hotel1", "sun3d-hotel_umd-maryland_hotel3",
                  "sun3d-mit_76_studyroom-76-1studyroom2", "sun3d-mit_lab_hj-lab_hj_tea_nov_2_2012_scan1_erika")


class _SceneFrameSource(_TestCloudSource):
    """Items (scene, frame) with paths; keypoints under <out>/<scene>/<frame>.bin."""

    divisor = 2                                   # redwood_loader.py:101, match3d_eval_loader.py:89

    def __init__(self, items, paths, opt, device, seed, rng, batch_size):
        self.items = list(items)
        if not self.items:
            raise ValueError("no test fragments")
        super().__init__(paths, opt, device, seed, rng, batch_size)

    def key(self, i):
        return self.items[i]

    def keypoint_path(self, out_dir, i):
        scene, frame = self.items[i]
        return os.path.join(out_dir, scene, "%d.bin" % frame)


class RedwoodTestLoader(_SceneFrameSource):
    """RedwoodLoader over root (numpy_gt_normal); `scenes` [(name, frame count)] overrides the reference's four for
    other trees.  Item i is frame i - (frames of the earlier scenes) of its scene."""

    allow_short = True

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=8, scenes=REDWOOD_SCENES):
        self.scenes = [(str(s), int(n)) for s, n in scenes]
        items = [(s, f) for s, n in self.scenes for f in range(n)]
        paths = [os.path.join(root, s, "%d.npy" % f) for s, f in items]
        super().__init__(items, paths, opt, device, seed, rng, batch_size)


def match3d_frame(name):
    """make_dataset_3dmatch_eval's frame number: int(name[10:-4]) of `cloud_bin_<k>.npy`."""
    if not (name.startswith("cloud_bin_") and name.endswith(".npy")):
        raise ValueError("not a 3DMatch fragment name: %r" % name)
    return int(name[10:-4])


class Match3DTestLoader(_SceneFrameSource):
    """Match3DEvalLoader over root (3DMatch_eval_npy).  `files` {scene: [file names in order]} gives each scene's
    listing (parity mode replays the reference's os.listdir order); by default every cloud_bin_*.npy of a scene folder,
    sorted by frame number.  `scenes` overrides the reference's eight."""

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=8, files=None, scenes=MATCH3D_SCENES):
        self.scenes = list(scenes)
        items, paths = [], []
        for s in self.scenes:
            if files is not None:
                names = list(files[s])
            else:
                names = sorted((n for n in os.listdir(os.path.join(root, s))
                                if n.startswith("cloud_bin_") and n.endswith(".npy")), key=match3d_frame)
            for n in names:
                items.append((s, match3d_frame(n)))
                paths.append(os.path.join(root, s, n))
        super().__init__(items, paths, opt, device, seed, rng, batch_size)


def synthetic_fragment(seed, rows):
    """(rows, 7) float32 [x, y, z, nx, ny, nz, curvature]: points in a 4 m room with unit normals."""
    r = np.random.RandomState(seed)
    a = np.empty((rows, 7), np.float32)
    a[:, 0:3] = r.uniform(-2, 2, (rows, 3))
    n = r.normal(size=(rows, 3))
    a[:, 3:6] = n / np.linalg.norm(n, axis=1, keepdims=True)
    a[:, 6] = r.uniform(0, 0.3, rows)
    return a


def write_gt_log(path, entries):
    """A gt.log (mrWriteLog.m's layout): per entry `anc pos count` and the 4x4, row by row."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        for anc, pos, count, T in entries:
            f.write("%d\t%d\t%d\n" % (anc, pos, count))
            f.write("".join(" ".join("%.12e" % v for v in row) + "\n" for row in np.asarray(T).reshape(4, 4)))


def write_gt_info(path, entries):
    """A gt.info (mrWriteInfo.m's layout): per entry `anc pos count` and the 6x6, row by row."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        for anc, pos, count, M in entries:
            f.write("%d\t%d\t%d\n" % (anc, pos, count))
            f.write("".join(" ".join("%.12e" % v for v in row) + "\n" for row in np.asarray(M).reshape(6, 6)))


def info_matrix(points):
    """getGtInfoLog.m's covariance of correspondences q: sum over the points of G^T G, G = [I3, -[q]_x] -> (6, 6)."""
    q = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    M = np.zeros((6, 6))
    for x, y, z in q:
        G = np.array([[1, 0, 0, 0, z, -y], [0, 1, 0, -z, 0, x], [0, 0, 1, y, -x, 0]], dtype=np.float64)
        M += G.T @ G
    return M


def _gt_entries(rng, pairs, count):
    from .kitti_test_loader import random_rigid
    from .repeatability import gt_transform
    out = []
    for a, p in pairs:
        T = np.eye(4)
        if a != p:
            T[:3] = gt_transform(*random_rigid(rng))
        out.append((a, p, count, T))
    return out


def write_synthetic_redwood(npy_root, gt_root, rows, pairs, seed=0, scenes=REDWOOD_SCENES):
    """A Redwood-shaped tree for tests and benchmarks: <npy_root>/<scene>/%d.npy, rows(scene index, frame) rows of
    synthetic_fragment each (rows may also be an int), and <gt_root>/original/<scene>-evaluation/gt.log listing
    pairs[scene] [(anc, pos)] with random rigid transforms (the identity when anc == pos), and next to it a gt.info with
    one info_matrix of 64 random room points per entry (drawn from their own stream, so the gt.log transforms do not
    depend on it)."""
    rng = np.random.RandomState(seed)
    info_rng = np.random.RandomState(seed + 7)
    for s, (scene, n) in enumerate(scenes):
        os.makedirs(os.path.join(npy_root, scene), exist_ok=True)
        for f in range(n):
            k = rows if np.isscalar(rows) else rows(s, f)
            np.save(os.path.join(npy_root, scene, "%d.npy" % f), synthetic_fragment(seed + 1000 * s + f, k))
        entries = _gt_entries(rng, pairs.get(scene, []), n)
        evaluation = os.path.join(gt_root, "original", "%s-evaluation" % scene)
        write_gt_log(os.path.join(evaluation, "gt.log"), entries)
        write_gt_info(os.path.join(evaluation, "gt.info"),
                      [(a, p, c, info_matrix(info_rng.uniform(-2, 2, (64, 3)))) for a, p, c, _ in entries])


def write_synthetic_3dmatch(root, frames, rows, pairs, seed=0):
    """A 3DMatch-shaped tree for tests and benchmarks: <root>/<scene>/cloud_bin_<k>.npy for k in frames[scene],
    rows(scene index, k) rows of synthetic_fragment each (rows may also be an int), and <root>/<scene>-evaluation/gt.log
    listing pairs[scene] with random rigid transforms."""
    rng = np.random.RandomState(seed)
    for s, scene in enumerate(frames):
        os.makedirs(os.path.join(root, scene), exist_ok=True)
        for k in frames[scene]:
            n = rows if np.isscalar(rows) else rows(s, k)
            np.save(os.path.join(root, scene, "cloud_bin_%d.npy" % k), synthetic_fragment(seed + 1000 * s + k, n))
        write_gt_log(os.path.join(root, "%s-evaluation" % scene, "gt.log"),
                     _gt_entries(rng, pairs.get(scene, []), len(frames[scene])))
