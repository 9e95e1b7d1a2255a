"""The ModelNet detector loader on the GPU: data/modelnet_shrec_loader.py (ModelNet_Shrec_Loader with
opt.dataset == 'modelnet') and the batching of modelnet/train_detector.py:23-29 (shuffled, drop_last).

Each item is one object file: `get_instance_unaugmented_np` (:152-180) runs twice on it, so src and dst are independent
subsamples of the same cloud, with FPS nodes over N/4 candidates.  `augment` (:182-243) differs from KITTI's: one draw of
every jitter array serves both clouds, the laws are sigma 0.01 / clip 0.05 for pc and sn and 0.04 / 0.1 for nodes, sn is
a float64 chain after any rotation and is scaled (never shifted), and the scale is U(0.8, 1.2).  The dst transform has
scale_thre 0.2 and never the rotation perturbation.  `ModelNetPairBuilder` builds the nine `ModelDetector.set_input`
tensors on the device (csrc/pairgen.cu: the detector builder's subset, candidate and FPS kernels, and
`usip_modelnet_pair_augment`); `ModelNetPairSource` feeds them from a ModelNet tree.  The Shrec variant is not covered.
"""
import math
import os

import numpy as np
import torch

from usip_b200 import ops

from .kitti_detector_loader import _PairBuilder, _ScanSource, angles2rotation_matrix

MODELNET_DIVISOR = 4                             # modelnet_shrec_loader.py:177: FPS over N/4 candidates


def _check_dataset(opt):
    dataset = getattr(opt, "dataset", "modelnet")
    if dataset == "shrec":
        raise NotImplementedError("the Shrec variant of ModelNet_Shrec_Loader (make_dataset_shrec2016, "
                                  "modelnet_shrec_loader.py:66-112: .npz files with their own pc / sn) is not built here")
    if dataset != "modelnet":
        raise ValueError("dataset %r: only 'modelnet' is built here" % (dataset,))


# ----------------------------------------------------------------------------------------------- ModelNet tree
def make_dataset_modelnet40_10k(root, mode, opt):
    """modelnet_shrec_loader.py:27-63 -> [(npy path, label, SOM-node path)] in the order of the split's list file.
    Item `name` is root/<name[0:-5]>/<name>.npy, labelled with the index of that folder among the shape names."""
    rows = round(math.sqrt(opt.node_num))
    classes = getattr(opt, "classes", 40)                          # modelnet/options_detector.py: ModelNet40
    with open(os.path.join(root, "modelnet%d_shape_names.txt" % classes)) as f:
        shape_list = [s.rstrip() for s in f.readlines()]
    if mode not in ("train", "test"):
        raise ValueError("mode must be 'train' or 'test'")
    with open(os.path.join(root, "modelnet%d_%s.txt" % (classes, mode))) as f:
        lines = [s.rstrip() for s in f.readlines()]
    som_folder = "%dx%d_som_nodes" % (rows, rows)
    return [(os.path.join(root, name[0:-5], name + ".npy"), shape_list.index(name[0:-5]),
             os.path.join(root, som_folder, name[0:-5], name + ".npy")) for name in lines]


def write_synthetic_modelnet(root, shapes, n_train, n_test, rows, seed=0, classes=40):
    """A ModelNet-shaped tree of seeded objects for tests and benchmarks: for every shape name, n_train + n_test files
    <shape>/<shape>_%04d.npy of (rows, 6) float32 [x, y, z, nx, ny, nz] -- points in the unit cube, unit normals -- drawn
    from RandomState(seed + 1000 * shape + i), and the list files, one split interleaving the shapes.  The shape-name
    file lists the shapes in reverse, so a label is not the shape's position in `shapes`."""
    with open(os.path.join(root, "modelnet%d_shape_names.txt" % classes), "w") as f:
        f.write("".join(s + "\n" for s in reversed(shapes)))
    splits = {"train": [], "test": []}
    for k, shape in enumerate(shapes):
        os.makedirs(os.path.join(root, shape), exist_ok=True)
        for i in range(n_train + n_test):
            name = "%s_%04d" % (shape, i + 1)
            np.save(os.path.join(root, shape, name + ".npy"), synthetic_object(seed + 1000 * k + i, rows))
            splits["train" if i < n_train else "test"].append((i, k, name))
    for split, items in splits.items():
        with open(os.path.join(root, "modelnet%d_%s.txt" % (classes, split)), "w") as f:
            f.write("".join(name + "\n" for _, _, name in sorted(items)))


def synthetic_object(seed, rows):
    r = np.random.RandomState(seed)
    a = np.empty((rows, 6), np.float32)
    a[:, 0:3] = r.uniform(-1, 1, (rows, 3))
    n = r.normal(size=(rows, 3))
    a[:, 3:6] = n / np.linalg.norm(n, axis=1, keepdims=True)
    return a


# ----------------------------------------------------------------------------------------------- host-side draws
def draw_modelnet_pair_scalars(rng, opt, train, N, M, per_point):
    """Scalars of augment() (:188-205, train only) and transform_pc_pytorch (augmentation.py:210-243, called with
    shift_thre=0.5 at :270) for one pair, in the reference's order -> (params (48,) f64, jitter (pc (N,3), sn (N,3),
    node (M,3)) shared by both clouds, or None).  per_point=False skips the O(N) jitter draws (the device draws its
    own)."""
    p = np.zeros(ops.PAIR_PARAM_STRIDE, dtype=np.float64)
    jit = None
    if train:
        y_angle = rng.uniform() * 2 * np.pi
        angles_2d = [0, y_angle, 0]
        angles_3d = rng.rand(3) * np.pi * 2
        angles_pertb = np.clip(0.06 * rng.randn(3), -0.18, 0.18)
        if per_point:
            sigma, clip = 0.01, 0.05
            jitter_pc = np.clip(sigma * rng.randn(N, 3), -1 * clip, clip)
            jitter_sn = np.clip(sigma * rng.randn(N, 3), -1 * clip, clip)
            sigma, clip = 0.04, 0.1
            jitter_node = np.clip(sigma * rng.randn(M, 3), -1 * clip, clip)
            jit = (jitter_pc, jitter_sn, jitter_node)
        scale = rng.uniform(low=0.8, high=1.2)
        shift = rng.uniform(-0.1, 0.1, (1, 3))
        p[0:9] = angles2rotation_matrix(angles_2d).ravel()
        p[9:18] = angles2rotation_matrix(angles_3d).ravel()
        p[18:27] = angles2rotation_matrix(angles_pertb).ravel()
        p[27] = scale
        p[28:31] = shift.ravel()
    rot_type = "3d" if opt.rot_3d else ("2d" if opt.rot_horizontal else None)
    if rot_type == "2d":
        x_angle, z_angle = 0, 0
        y_angle = rng.uniform() * 2 * np.pi
    elif rot_type == "3d":
        x_angle = rng.uniform() * 2 * np.pi
        y_angle = rng.uniform() * 2 * np.pi
        z_angle = rng.uniform() * 2 * np.pi
    else:
        x_angle, y_angle, z_angle = 0, 0, 0
    # rot_perturbation is not passed to transform_pc_pytorch here: it stays False whatever opt says
    p[31:40] = angles2rotation_matrix([x_angle, y_angle, z_angle]).astype(np.float32).ravel()
    scale_t = rng.uniform(low=1 - 0.2, high=1 + 0.2)               # scale_thre keeps its default 0.2
    p[40:43] = rng.uniform(-1 * 0.5, 0.5, (3, 1)).astype(np.float32).ravel()
    p[43] = np.float32(scale_t)                                     # float32 tensor * Python float, see pairgen.cu
    return p, jit


# ----------------------------------------------------------------------------------------------- the builder
class ModelNetPairBuilder(_PairBuilder):
    """Builds the nine `ModelDetector.set_input` tensors of a batch of ModelNet pairs on the device.

    `build(scans, offsets, items, step=None)`: scans [T, C >= 6] f32 (device, or host -- then the items' scans are
    uploaded), offsets (n_scans+1,) int64 row offsets (host), items the scan index of every pair.  Both clouds of a pair
    are independent subsamples of the same scan (modelnet_shrec_loader.py:246-247) and share one jitter draw.  Every
    scan needs at least input_pc_num rows: the reference draws them without replacement.  sn is columns 3:6, so
    surface_normal_len must be 3.  See `_PairBuilder` for the two rng modes; rng="numpy" replays
    ModelNet_Shrec_Loader.__getitem__.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device"):
        _check_dataset(opt)
        super().__init__(opt, mode, device, seed, rng, MODELNET_DIVISOR)
        if self.S != 3:
            raise ValueError("surface_normal_len %d: ModelNet's sn is columns 3:6, surface_normal_len must be 3"
                             % self.S)

    def _clouds(self, items):
        items = np.asarray(items, dtype=np.int64).ravel()
        if items.size == 0:
            raise ValueError("no items")
        return np.repeat(items, 2)

    def _check_rows(self, clouds, lengths):
        k = int(np.argmin(lengths))
        if lengths[k] < self.N:
            raise ValueError("scan %d has %d rows; input_pc_num = %d rows are drawn without replacement"
                             % (int(clouds[k]), int(lengths[k]), self.N))

    def _draw(self, rng, per_point):
        return draw_modelnet_pair_scalars(rng, self.opt, self.mode == "train", self.N, self.M, per_point)

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.modelnet_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.flags, self.seed,
                                         step, *jit)

    def build(self, scans, offsets, items, step=None):
        return self._build(scans, offsets, step, items)


class ModelNetPairSource(_ScanSource):
    """Shuffled batches of ModelNet detector pairs, built on the device and handed to `ModelDetector` (see
    `_ScanSource`).  The items are those of make_dataset_modelnet40_10k(root, mode, opt); `labels` holds their class
    indices.

        src = ModelNetPairSource(root, "train", opt)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, device=None, seed=0, resident="host", rng="device", batch_size=None,
                 drop_last=True):
        _check_dataset(opt)
        self.dataset = make_dataset_modelnet40_10k(root, mode, opt)
        if not self.dataset:
            raise ValueError("no items in the %s split under %s" % (mode, root))
        self.labels = np.array([label for _, label, _ in self.dataset], dtype=np.int64)
        super().__init__([path for path, _, _ in self.dataset], mode, opt, ModelNetPairBuilder, device, seed, resident,
                         rng, batch_size, drop_last)

    def _build(self, items):
        return self.builder.build(self.scans, self.offsets, items, step=self.step), None
