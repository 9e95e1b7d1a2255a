"""The rotated ModelNet40 test set on the GPU: data/modelnet_rotated_loader.py (ModelNet_Rotated_Loader,
make_dataset_modelnet40), and the tree it reads (evaluation/matlab/eval_repeatability/rotate_modelnet_dateset.m).

Items 0..n-1 are <root>/original/%d.npy and items n..2n-1 <root>/rotated/%d.npy, n = 2468 (the reference's count) or
the row count of the tree's modelnet_info.mat.  Each item is input_pc_num rows drawn without replacement (a shorter
object is refused), sn = columns 3:6, and FPS nodes over int(input_pc_num / 4) of the rows.  See
kitti_test_loader._TestCloudSource for the batches and the rng modes.

`write_rotated_modelnet` builds the tree from a ModelNet40 normal-resampled tree.  Its angles come from a numpy
RandomState, the authors' from MATLAB's `rand`: without their rotated tree their published numbers cannot be
reproduced bit for bit.
"""
import os

import numpy as np

from .kitti_test_loader import _TestCloudSource

MODELNET_TEST_OBJECTS = 2468                      # modelnet_rotated_loader.py:20, :24
MODELNET_FOLDERS = ("original", "rotated")        # pc_type_id 0 and 1


class ModelNetRotatedTestLoader(_TestCloudSource):
    """ModelNet_Rotated_Loader over root with n objects (default 2468): key(i) = ("original" | "rotated", object)."""

    divisor = 4                                   # modelnet_rotated_loader.py:71
    sn_len = 3                                    # modelnet_rotated_loader.py:67, columns 3:6

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=4, n=None):
        self.n = MODELNET_TEST_OBJECTS if n is None else int(n)
        if self.n < 1:
            raise ValueError("no test objects")
        paths = [os.path.join(root, f, "%d.npy" % i) for f in MODELNET_FOLDERS for i in range(self.n)]
        super().__init__(paths, opt, device, seed, rng, batch_size)

    def key(self, i):
        return (MODELNET_FOLDERS[i // self.n], i % self.n)

    def keypoint_path(self, out_dir, i):
        """save_keypoints.py:383-391."""
        return os.path.join(out_dir, MODELNET_FOLDERS[i // self.n], "%d.bin" % (i % self.n))


def eul2rotm(angles):
    """MATLAB eul2rotm in its default ZYX order: angles (a, b, c) -> Rz(a) @ Ry(b) @ Rx(c), (3, 3) float64."""
    a, b, c = np.asarray(angles, dtype=np.float64)
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rz = np.array([[ca, -sa, 0], [sa, ca, 0], [0, 0, 1.0]])
    Ry = np.array([[cb, 0, sb], [0, 1.0, 0], [-sb, 0, cb]])
    Rx = np.array([[1.0, 0, 0], [0, cc, -sc], [0, sc, cc]])
    return Rz @ Ry @ Rx


def write_rotated_modelnet(normal_root, out_root, seed=0):
    """rotate_modelnet_dateset.m: for the objects of <normal_root>/modelnet40_test.txt in file order, object i (read
    from <normal_root>/<label>/<name>.npy, label = name[:-5]) is written unchanged to <out_root>/original/%d.npy and as
    [xyz @ R, n @ R] (float64 product, stored float32) to <out_root>/rotated/%d.npy, R = eul2rotm(angles) with angles
    U(-pi, pi) from RandomState(seed).  <out_root>/modelnet_info.mat holds the cell array {original path, rotated path,
    [R, 0]} per object, as eval_rep.m and read_modelnet_info read it.  -> the (n, 3, 3) rotations."""
    import scipy.io
    with open(os.path.join(normal_root, "modelnet40_test.txt")) as f:
        names = f.read().split()
    rng = np.random.RandomState(seed)
    for folder in MODELNET_FOLDERS:
        os.makedirs(os.path.join(out_root, folder), exist_ok=True)
    info = np.empty((len(names), 3), dtype=object)
    Rs = np.empty((len(names), 3, 3))
    for i, name in enumerate(names):
        obj = np.load(os.path.join(normal_root, name[:-5], "%s.npy" % name))
        R = eul2rotm((rng.rand(3) - 0.5) * 2 * np.pi)
        o64 = obj[:, 0:6].astype(np.float64)
        rotated = np.concatenate([o64[:, 0:3] @ R, o64[:, 3:6] @ R], axis=1).astype(np.float32)
        paths = [os.path.join(out_root, f, "%d.npy" % i) for f in MODELNET_FOLDERS]
        np.save(paths[0], obj)
        np.save(paths[1], rotated)
        info[i, 0], info[i, 1] = paths
        info[i, 2] = np.concatenate([R, np.zeros((3, 1))], axis=1)
        Rs[i] = R
    scipy.io.savemat(os.path.join(out_root, "modelnet_info.mat"), {"modelnet_info": info})
    return Rs


def write_synthetic_modelnet40_normal(root, names, rows, seed=0):
    """A ModelNet40 normal-resampled tree for tests and benchmarks: <root>/modelnet40_test.txt lists names (each
    `<label>_%04d`), <root>/<label>/<name>.npy is (rows, 6) float32 points on a sphere with their unit normals."""
    rng = np.random.RandomState(seed)
    with open(os.path.join(root, "modelnet40_test.txt"), "w") as f:
        f.write("".join(n + "\n" for n in names))
    for name in names:
        os.makedirs(os.path.join(root, name[:-5]), exist_ok=True)
        n = rng.normal(size=(rows, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        pts = n * rng.uniform(0.8, 1.0, (rows, 1))
        np.save(os.path.join(root, name[:-5], "%s.npy" % name), np.concatenate([pts, n], axis=1).astype(np.float32))
