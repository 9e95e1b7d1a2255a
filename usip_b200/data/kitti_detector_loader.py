"""The KITTI detector loader on the GPU (SURVEY section 8 f-2).

`FarthestSampler` mirrors the node generation of data/kitti_detector_loader.py:68-83.  `DetectorPairBuilder` builds the
whole training batch of `KittiLoader.__getitem__` (:218-259) on the device -- random subsampling, FPS nodes,
augmentation and the dst transform -- and `KittiPairSource` feeds such batches to `ModelDetector` from a KITTI tree.
The reference runs all of this per pair in DataLoader workers: serial numpy, more host time per pair than a whole
training step of this repository.  Only the KITTI loaders are covered (the descriptor's builds on the bases here); the
Oxford / ModelNet / SceneNN / Match3D loaders differ in the candidate divisor (a parameter here) and in using two scans.
"""
import os

import numpy as np
import torch

from usip_b200 import ops

FPS_MAX_CANDIDATES = 8192                        # usip_fps_f32
KITTI_NP_FOLDER = "np_0.20_20480_r90_sn"


class FarthestSampler:
    """Drop-in for the reference class: `sample(pts, k)` with pts an (Ns, 3) float array returns the (k, 3) float64
    array the numpy code returns -- bit-identical, including which random number it consumes (one
    np.random.randint(len(pts)) for the first node)."""

    def __init__(self, device=None):
        self.device = torch.device(device if device is not None else "cuda")

    def sample(self, pts, k):
        pts32 = np.ascontiguousarray(pts, dtype=np.float32)
        if pts32.shape[1] != 3:
            raise ValueError("pts must be (Ns, 3)")
        start = np.random.randint(len(pts32))                      # kitti_detector_loader.py:78
        idx = self.sample_indices(torch.from_numpy(pts32).to(self.device)[None], torch.tensor([start], dtype=torch.int32), k)[0]
        return pts32[idx[0].cpu().numpy()].astype(np.float64)

    def sample_indices(self, pts, start, k, want_nodes=False):
        """Batched form for a GPU-resident pipeline: pts (B, Ns, 3) f32 CUDA, start (B,) int -> (idx (B,k) i32,
        nodes (B,3,k) f32 in the detector's node layout or None)."""
        pts = pts.to(self.device, torch.float32).contiguous()
        start = torch.as_tensor(start).to(self.device, torch.int32).contiguous()
        if int(start.min()) < 0 or int(start.max()) >= pts.shape[1]:
            raise IndexError("start index out of range")
        return ops.fps(pts, start, k, want_nodes=want_nodes)


# ----------------------------------------------------------------------------------------------- host-side draws
def angles2rotation_matrix(angles):
    """data/augmentation.py:15-26: Rz . (Ry . Rx), float64."""
    cx, sx = np.cos(angles[0]), np.sin(angles[0])
    cy, sy = np.cos(angles[1]), np.sin(angles[1])
    cz, sz = np.cos(angles[2]), np.sin(angles[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return np.dot(Rz, np.dot(Ry, Rx))


def radius_mask(pc, radius):
    """kitti_detector_loader.py:121-122."""
    return np.linalg.norm(pc[:, [0, 2]], axis=1) <= radius


def draw_subsample(rng, n_valid, N, divisor=3):
    """The index draws of get_instance_unaugmented_np (:126-145) for one cloud, in the reference's order:
    rows into the n_valid (masked) points, FPS candidate positions into the N rows, FPS start."""
    if n_valid >= N:
        choice = rng.choice(n_valid, N, replace=False)
    else:
        fix = np.arange(n_valid)
        while n_valid + fix.shape[0] < N:
            fix = np.concatenate((fix, np.arange(n_valid)), axis=0)
        choice = np.concatenate((fix, rng.choice(n_valid, N - fix.shape[0], replace=False)), axis=0)
    cand = rng.choice(N, int(N / divisor), replace=False)
    start = rng.randint(len(cand))                                  # FarthestSampler.sample, :78
    return choice, cand, start


def draw_pair_scalars(rng, opt, train, N, M, S, per_point):
    """Scalars of augment() (:157-175, train only) and transform_pc_pytorch (augmentation.py:210-243) for one pair,
    in the reference's order -> (params (48,) f64, jitter (pc (2,N,3), sn (2,N,S), node (2,M,3)) or None).
    per_point=False skips the O(N) jitter draws (the device draws its own)."""
    p = np.zeros(ops.PAIR_PARAM_STRIDE, dtype=np.float64)
    jit = None
    if train:
        y_angle = rng.uniform() * 2 * np.pi
        angles_2d = [0, y_angle, 0]
        angles_3d = rng.rand(3) * np.pi * 2
        angles_pertb = np.clip(0.06 * rng.randn(3), -0.18, 0.18)
        if per_point:
            jit = (np.clip(0.04 * rng.randn(2, N, 3), -0.12, 0.12), np.clip(0.01 * rng.randn(2, N, S), -0.05, 0.05),
                   np.clip(0.04 * rng.randn(2, M, 3), -0.12, 0.12))
        scale = rng.uniform(low=0.9, high=1.1)
        shift = rng.uniform(-1, 1, (1, 3))
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
    if getattr(opt, "rot_perturbation", False):
        angle_sigma = 0.06
        angle_clip = 3 * angle_sigma
        x_angle += np.clip(angle_sigma * rng.randn(), -angle_clip, angle_clip)
        y_angle += np.clip(angle_sigma * rng.randn(), -angle_clip, angle_clip)
        z_angle += np.clip(angle_sigma * rng.randn(), -angle_clip, angle_clip)
    p[31:40] = angles2rotation_matrix([x_angle, y_angle, z_angle]).astype(np.float32).ravel()
    scale_t = rng.uniform(low=1 - 0, high=1 + 0)                   # scale_thre = 0
    p[40:43] = rng.uniform(-0.5, 0.5, (3, 1)).astype(np.float32).ravel()
    p[43] = np.float32(scale_t)
    return p, jit


def _step_rng(seed, step):
    w = [(seed >> s) & 0xffffffff for s in (0, 32)] + [(step >> s) & 0xffffffff for s in (0, 32)]
    return np.random.RandomState(np.array(w, dtype=np.uint32))


# ----------------------------------------------------------------------------------------------- the builders
class _PairBuilder:
    """What the detector's and the descriptor's pair builders share.  A batch of B pairs is 2B clouds, cloud 2b + side
    (side 0 = src / anchor, 1 = dst / positive) a subsample of one scan: subsets, FPS candidates and nodes are built per
    cloud, whichever scans a pair's two clouds come from.  A subclass names the scan of every cloud (`_clouds`), draws
    one pair's scalars (`_draw`) and runs its augment kernel (`_augment`).

    rng="device": per-point randomness (subsets, jitter, FPS start) is Philox keyed by (seed, step, cloud, point,
    purpose); per-pair scalars come from a numpy RandomState seeded by (seed, step).  Host work is O(B) and a given
    (seed, step) always gives the same batch, bit for bit.  Selected rows ascend within each part (see
    usip_cloud_subsample in include/usip_b200.h); the reference's order is numpy's permutation order.
    rng="numpy": parity mode.  Consumes the global np.random exactly as the reference's __getitem__ does, item by item
    (side 0's rows, candidates and FPS start, side 1's, then the pair's augmentation), and uploads the index lists and
    jitter arrays: slow by design, it reproduces the reference's batch.

    The outputs are fresh tensors allocated on the current stream; nothing is overwritten by a later build.
    """

    radius = None                                # only rows within this xz distance of the sensor are drawable

    def __init__(self, opt, mode, device, seed, rng, divisor):
        if mode not in ("train", "test"):
            raise ValueError("mode must be 'train' or 'test'")
        if rng not in ("device", "numpy"):
            raise ValueError("rng must be 'device' or 'numpy'")
        self.opt, self.mode, self.rng, self.seed = opt, mode, rng, int(seed)
        self.device = torch.device(device if device is not None else "cuda")
        self.N, self.M, self.S = int(opt.input_pc_num), int(opt.node_num), int(opt.surface_normal_len)
        self.n_cand = int(self.N / divisor)
        self.divisor = divisor
        if self.n_cand > FPS_MAX_CANDIDATES:
            raise ValueError("input_pc_num / %s = %d FPS candidates; usip_fps_f32 takes at most %d"
                             % (divisor, self.n_cand, FPS_MAX_CANDIDATES))
        if self.n_cand < 1 or self.M > self.n_cand:
            raise ValueError("node_num %d needs at least as many FPS candidates (%d)" % (self.M, self.n_cand))
        self.flags = ((ops.PAIR_TRAIN if mode == "train" else 0)
                      | (ops.PAIR_ROT_HORIZONTAL if getattr(opt, "rot_horizontal", False) else 0)
                      | (ops.PAIR_ROT_3D if getattr(opt, "rot_3d", False) else 0)
                      | (ops.PAIR_ROT_PERTURBATION if getattr(opt, "rot_perturbation", False) else 0)
                      | (ops.PAIR_TRANSLATION if getattr(opt, "translation_perturbation", False) else 0))
        self.step = 0
        self.last = None                      # index lists of the last build (rows, cand, start), for inspection

    def _clouds(self, *items):
        """(2B,) int64: the scan of every cloud."""
        raise NotImplementedError

    def _check_rows(self, clouds, lengths):
        """Reject scans too short for the subclass's loader (every scan here has at least one row)."""

    def _draw(self, rng, per_point):
        """One pair's scalars -> (params block, jitter (pc (2,N,3), sn (2,N,S), node (2,M,3)) or None)."""
        raise NotImplementedError

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        raise NotImplementedError

    def _build(self, scans, offsets, step, *items):
        offsets = np.asarray(offsets, dtype=np.int64)
        if offsets.ndim != 1 or offsets.shape[0] < 2:
            raise ValueError("no scans")
        clouds = self._clouds(*items)
        if clouds.min() < 0 or clouds.max() >= offsets.shape[0] - 1:
            raise IndexError("item out of range")
        lengths = offsets[clouds + 1] - offsets[clouds]
        k = int(np.argmin(lengths))
        if lengths[k] <= 0:
            raise ValueError("scan %d has no points" % int(clouds[k]))
        self._check_rows(clouds, lengths)
        B, N, M, S, dev = len(clouds) // 2, self.N, self.M, self.S, self.device
        C = scans.shape[1]
        if scans.dim() != 2 or C < 3 + max(S, 1):
            raise ValueError("scans have %d columns, surface_normal_len %d needs %d" % (C, S, 3 + S))
        max_rows = int(max(lengths.max(), N))
        if max_rows > ops.pair_max_scan_rows():
            raise ValueError("a scan of %d rows exceeds the %d the subsample kernel holds"
                             % (max_rows, ops.pair_max_scan_rows()))
        if step is None:
            step = self.step
        self.step = int(step) + 1

        used = np.unique(clouds)
        drawable = None                                # parity mode with a radius: the rows inside it, per cloud
        if self.rng == "numpy" and self.radius is not None:
            inside = {i: np.nonzero(radius_mask(scans[offsets[i]:offsets[i + 1]].cpu().numpy(), self.radius))[0]
                      for i in used}
            drawable = [inside[i] for i in clouds]
        if scans.device != dev:                        # upload only the scans this batch uses, each once
            parts = [scans[offsets[i]:offsets[i + 1]] for i in used]
            scans = torch.cat(parts).pin_memory().to(dev, non_blocking=True)
            offsets = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
            clouds = np.searchsorted(used, clouds)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)
        offsets_d = up(offsets)
        scan_of_cloud = up(clouds.astype(np.int32))

        jit = (None, None, None)
        with torch.cuda.device(dev):
            if self.rng == "device":
                rows, cand, start, _ = ops.cloud_subsample(scans, offsets_d, scan_of_cloud, max_rows, N, self.n_cand,
                                                           self.radius, self.seed, step)
                hrng = _step_rng(self.seed, step)
                drawn = [self._draw(hrng, False) for _ in range(B)]
            else:
                rows_h = np.empty((2 * B, N), np.int32)
                cand_h = np.empty((2 * B, self.n_cand), np.int32)
                start_h = np.empty((2 * B,), np.int32)
                drawn = []
                for b in range(B):                     # the reference's __getitem__, item by item
                    for c in (2 * b, 2 * b + 1):
                        n_valid = int(lengths[c]) if drawable is None else len(drawable[c])
                        choice, cand_h[c], start_h[c] = draw_subsample(np.random, n_valid, N, self.divisor)
                        rows_h[c] = choice if drawable is None else drawable[c][choice]
                    drawn.append(self._draw(np.random, True))
                rows, cand, start = up(rows_h), up(cand_h), up(start_h)
                if drawn[0][1] is not None:
                    jit = tuple(up(np.stack([d[1][k] for d in drawn]).reshape((2 * B,) + drawn[0][1][k].shape[1:]))
                                for k in range(3))
            params = np.stack([d[0] for d in drawn])
            params = up(params.reshape(-1, params.shape[-1]))
            pts = ops.cloud_gather_candidates(scans, offsets_d, scan_of_cloud, rows, cand)
            _, nodes = ops.fps(pts, start, M, want_nodes=True)
            out = self._augment(scans, offsets_d, scan_of_cloud, rows, nodes, params, step, jit)
        self.last = {"rows": rows, "cand": cand, "start": start, "candidates": pts, "params": params}
        return out


class DetectorPairBuilder(_PairBuilder):
    """Builds the nine `ModelDetector.set_input` tensors of a batch of KITTI pairs on the device.

    `build(scans, offsets, items, step=None)`: scans [T, C] f32 (device, or host -- then the items' scans are uploaded),
    offsets (n_scans+1,) int64 row offsets (host), items the scan index of every pair.  Both clouds of a pair are
    independent subsamples of the same scan (kitti_detector_loader.py:219-220); rng="numpy" replays
    KittiLoader.__getitem__.  See `_PairBuilder` for the two rng modes.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device", divisor=3):
        super().__init__(opt, mode, device, seed, rng, divisor)
        r = getattr(opt, "radius_threshold", 100.0)
        self.radius = float(r) if r < 90 else None

    def _clouds(self, items):
        items = np.asarray(items, dtype=np.int64).ravel()
        if items.size == 0:
            raise ValueError("no items")
        return np.repeat(items, 2)

    def _draw(self, rng, per_point):
        return draw_pair_scalars(rng, self.opt, self.mode == "train", self.N, self.M, self.S, per_point)

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.S, self.flags, self.seed, step,
                                *jit)

    def build(self, scans, offsets, items, step=None):
        return self._build(scans, offsets, step, items)


# ----------------------------------------------------------------------------------------------- KITTI tree
def make_dataset_kitti(root, mode):
    """kitti_detector_loader.py:23-47 -> (seq_list, folder_list, sample_num_list, accumulated_sample_num_list)."""
    if mode == "train":
        seq_list = list(range(9))
    elif mode == "test":
        seq_list = [9, 10]
    else:
        raise ValueError("Invalid mode.")
    acc, nums, accs, folders = 0, [], [], []
    for seq in seq_list:
        folder = os.path.join(root, "data_odometry_velodyne", "numpy", "%02d" % seq, KITTI_NP_FOLDER)
        folders.append(folder)
        n = len(os.listdir(folder))
        acc += n
        nums.append(n)
        accs.append(acc)
    return seq_list, folders, nums, accs


def kitti_scan_path(root, mode, index):
    """The file `KittiLoader(root, mode).get_instance_unaugmented_np(index)` reads (:103-113)."""
    seqs, folders, _, accs = make_dataset_kitti(root, mode)
    if not 0 <= index < accs[-1]:
        raise IndexError(index)
    i = next(i for i, a in enumerate(accs) if index < a)
    return os.path.join(folders[i], "%06d.npy" % (index - (accs[i - 1] if i else 0)))


def load_scan_npy(path, surface_normal_len):
    """(Ns, C) float32 scan, checked like evaluation.save_keypoints.read_pointcloud_npy."""
    a = np.load(path)
    if a.ndim != 2 or a.shape[1] < 3 + max(surface_normal_len, 1):
        raise ValueError("expected an (N, >=%d) array, got %r" % (3 + surface_normal_len, a.shape))
    return np.ascontiguousarray(a, dtype=np.float32)


def write_synthetic_kitti(root, counts, Ns, seed=0, C=8, poses=None):
    """A KITTI-shaped tree of seeded scans for tests and benchmarks: counts[seq] scans in sequence seq (0..10), each
    (Ns or Ns[seq][i], C) float32 [x, y, z, nx, ny, nz, curvature, reflectance] drawn from RandomState(seed + 1000*seq +
    i), plus poses: poses[seq][i] (4, 4) when given (a trajectory, for the descriptor's positives and negatives),
    identity otherwise."""
    for seq, n in enumerate(counts):
        folder = os.path.join(root, "data_odometry_velodyne", "numpy", "%02d" % seq, KITTI_NP_FOLDER)
        os.makedirs(folder, exist_ok=True)
        os.makedirs(os.path.join(root, "poses", "%02d" % seq), exist_ok=True)
        for i in range(n):
            ns = Ns if np.isscalar(Ns) else Ns[seq][i]
            np.save(os.path.join(folder, "%06d.npy" % i), synthetic_scan(seed + 1000 * seq + i, ns, C))
            pose = np.eye(4) if poses is None else np.asarray(poses[seq][i])
            np.savez(os.path.join(root, "poses", "%02d" % seq, "%06d.npz" % i), pose=pose)


def synthetic_scan(seed, Ns, C=8):
    r = np.random.RandomState(seed)
    a = np.empty((Ns, C), np.float32)
    a[:, 0] = r.uniform(-40, 40, Ns)
    a[:, 1] = r.normal(0, 1.5, Ns)
    a[:, 2] = r.uniform(-40, 40, Ns)
    n = r.normal(size=(Ns, 3))
    a[:, 3:6] = n / np.linalg.norm(n, axis=1, keepdims=True)
    a[:, 6:C] = r.uniform(0, 1, (Ns, C - 6))
    return a


class _KittiSource:
    """What the KITTI detector and descriptor sources share: the scans of a tree, indexed like make_dataset_kitti (so
    `index` names the reference's sample) and loaded once into pinned host memory, or onto the device with
    resident="device"; shuffled epochs; and the hand-over.  Iteration builds batch i+1 on a stream of its own while the
    caller runs step i, and hands each batch over with `model.prefetch_input(..., after=event)` + `set_input()`: the
    model's stream waits on the build's event, the host never synchronises.  Every batch is a fresh set of tensors, so
    a batch still in use is never overwritten.  A subclass turns the scan indices of one batch into the model's inputs
    (`_build`, called with the build stream current)."""

    def __init__(self, root, mode, opt, builder, device, seed, resident, rng, batch_size, drop_last):
        self.opt, self.mode = opt, mode
        self.device = torch.device(device if device is not None else "cuda")
        self.batch_size = int(batch_size or opt.batch_size)
        self.drop_last = drop_last
        _, _, self.nums, self.accs = make_dataset_kitti(root, mode)
        n = self.accs[-1] if self.accs else 0
        if n == 0:
            raise ValueError("no scans under %s" % root)
        arrs = [load_scan_npy(kitti_scan_path(root, mode, i), opt.surface_normal_len) for i in range(n)]
        if len({a.shape[1] for a in arrs}) != 1:
            raise ValueError("scans differ in column count")
        self.offsets = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
        scans = torch.from_numpy(np.concatenate(arrs))
        self.scans = scans.to(self.device) if resident == "device" else scans.pin_memory()
        self.builder = builder(opt, mode, self.device, seed, rng)
        self.order_rng = np.random.RandomState(seed)
        self.stream = torch.cuda.Stream(device=self.device)
        self.step = 0
        self.last = None                        # what the batch last yielded was built from, for inspection

    def __len__(self):
        n = len(self.offsets) - 1
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _build(self, items):
        """-> (the model's input tensors, what `last` will say about them)."""
        raise NotImplementedError

    def _enqueue(self, items):
        with torch.cuda.stream(self.stream):
            out, info = self._build(items)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.step += 1
        return out, ev, info

    def batches(self):
        """One shuffled epoch of (input tensors, ready event); batch i+1 is enqueued before batch i is yielded."""
        perm = self.order_rng.permutation(len(self.offsets) - 1)
        chunks = [perm[i:i + self.batch_size] for i in range(0, len(perm), self.batch_size)]
        if self.drop_last and chunks and len(chunks[-1]) < self.batch_size:
            chunks.pop()
        nxt = self._enqueue(chunks[0]) if chunks else None
        for k in range(len(chunks)):
            out, ev, self.last = nxt
            nxt = self._enqueue(chunks[k + 1]) if k + 1 < len(chunks) else None
            yield out, ev

    def feed(self, model):
        """One epoch; before each yield the batch is the model's input (prefetch_input + set_input)."""
        for out, ev in self.batches():
            model.prefetch_input(*out, after=ev)
            model.set_input(*out)
            yield out


class KittiPairSource(_KittiSource):
    """Shuffled batches of KITTI detector pairs, built on the device and handed to `ModelDetector` (see `_KittiSource`).

        src = KittiPairSource(root, "train", opt)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, device=None, seed=0, resident="host", rng="device", batch_size=None,
                 drop_last=True):
        super().__init__(root, mode, opt, DetectorPairBuilder, device, seed, resident, rng, batch_size, drop_last)

    def _build(self, items):
        return self.builder.build(self.scans, self.offsets, items, step=self.step), None
