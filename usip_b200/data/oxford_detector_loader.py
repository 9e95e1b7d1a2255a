"""The Oxford detector loader on the GPU: data/oxford_detector_loader.py (OxfordLoader) and the batching of
oxford/train_detector.py (shuffled, drop_last).

An Oxford tree holds ENU scans (z up), (Ns, 8) float32 [x y z nx ny nz curvature reflectance]:
train_np_nofilter/<file[0:-3]>npy for the lines of train_relative.txt, test_models_20k_np_nofilter/%d.npy in test mode.
Each item subsamples one scan twice (src and dst, N rows each without replacement), draws one height scale
U(0.25, 1.2) that multiplies both clouds' z in train mode (when opt.is_height_scaling, the default), builds FPS nodes
over N/8 candidates of the scaled clouds, maps everything to the camera frame (x, -z, y), and then augments like KITTI
with a scale law of U(0.7, 1.3).  `OxfordPairBuilder` builds the nine `ModelDetector.set_input` tensors on the device
(csrc/pairgen.cu: the shared subset kernel, the z-scaled candidate gather, FPS and `usip_pair_augment` with the
USIP_PAIR_ENU_TO_CAM / USIP_PAIR_HEIGHT_SCALE steps); `OxfordPairSource` feeds them from an Oxford tree.
"""
import os
import pickle
import warnings

import numpy as np

from usip_b200 import ops

from .kitti_detector_loader import _PairBuilder, _ScanSource, draw_pair_scalars, synthetic_scan

OXFORD_DET_DIVISOR = 8                           # oxford_detector_loader.py:196: FPS over N/8 candidates
OXFORD_TRAIN_FOLDER = "train_np_nofilter"
OXFORD_TEST_FOLDER = "test_models_20k_np_nofilter"
HEIGHT_SCALE_RANGE = (0.25, 1.2)                 # :189, and oxford/train_descriptor.py:124
OXFORD_SCALE_RANGE = (0.7, 1.3)                  # OxfordLoader.augment, :139


# ----------------------------------------------------------------------------------------------- Oxford tree
def parse_train_relative(root):
    """train_relative.txt, one line per scan: `file | positive line numbers | non-negative line numbers` ->
    [(file, positives, non-negatives)].  A line that does not split into three parts is skipped with a warning, as the
    reference skips it with a print; the line numbers index this parsed list, so they keep the reference's meaning."""
    out = []
    with open(os.path.join(root, "train_relative.txt")) as f:
        for i, line in enumerate(f.readlines()):
            parts = line.split("|")
            if len(parts) != 3:
                warnings.warn("train_relative.txt line %d is invalid and skipped: %r" % (i, line))
                continue
            out.append((parts[0].strip(), list(map(int, parts[1].split())), list(map(int, parts[2].split()))))
    return out


def make_dataset_oxford_train(root):
    """oxford_detector_loader.py:43-71 -> [{'file', 'pos_list', 'nonneg_list'}]."""
    return [{"file": f, "pos_list": p, "nonneg_list": n} for f, p, n in parse_train_relative(root)]


def make_dataset_oxford_test(root):
    """oxford_detector_loader.py:74-76: the list in test_models_20k_np_nofilter/groundtruths.pkl (dicts with at least
    'anc_idx', the file number of the item's scan)."""
    with open(os.path.join(root, OXFORD_TEST_FOLDER, "groundtruths.pkl"), "rb") as f:
        return pickle.load(f)


def oxford_train_path(root, file_name):
    """get_instance_unaugmented_np, :102."""
    return os.path.join(root, OXFORD_TRAIN_FOLDER, file_name[0:-3] + "npy")


def oxford_test_path(root, number):
    """get_instance_unaugmented_np, :105."""
    return os.path.join(root, OXFORD_TEST_FOLDER, "%d.npy" % number)


def synthetic_enu_scan(seed, Ns):
    """(Ns, 8) float32 [x y z nx ny nz curvature reflectance] in ENU: the KITTI synthetic scan with y and z swapped, so
    that z is up (heights N(0, 1.5)) and the frame change and height scaling move something."""
    a = synthetic_scan(seed, Ns, 8)
    a[:, [1, 2]] = a[:, [2, 1]]
    a[:, [4, 5]] = a[:, [5, 4]]
    return a


def write_synthetic_oxford(root, n_train, rows, n_test=0, seed=0, pos_width=2, nonneg_width=4, invalid_at=None,
                           test_numbers=None):
    """An Oxford-shaped tree of seeded ENU scans for tests and benchmarks.

    Train: n_train scans %06d.bin (stored as train_np_nofilter/%06d.npy), (rows or rows[i], 8) float32 from
    synthetic_enu_scan(seed + i), along a line: the positives of scan i are the scans within pos_width of it, its
    non-negatives those within nonneg_width that are not positives (line numbers = parsed indices).  train_relative.txt
    has one invalid line before the scan `invalid_at` (default n_train // 2).
    Test: n_test scans test_models_20k_np_nofilter/%d.npy numbered test_numbers (default 100 + 3 i), from
    synthetic_enu_scan(seed + 5000 + i), and both pickles: groundtruths.pkl [{'anc_idx', 'pos_idx', 'neg_idx', 't',
    'q'}] and gt_descriptor_testing.pkl [{'anc_idx', 'pos_idx_list'}], the positives being the test scans within
    pos_width in order."""
    rows_of = (lambda i: rows) if np.isscalar(rows) else (lambda i: rows[i])
    os.makedirs(os.path.join(root, OXFORD_TRAIN_FOLDER), exist_ok=True)
    os.makedirs(os.path.join(root, OXFORD_TEST_FOLDER), exist_ok=True)
    invalid_at = n_train // 2 if invalid_at is None else invalid_at
    lines = []
    for i in range(n_train):
        np.save(oxford_train_path(root, "%06d.bin" % i), synthetic_enu_scan(seed + i, rows_of(i)))
        pos = [j for j in range(n_train) if 0 < abs(i - j) <= pos_width]
        nonneg = [j for j in range(n_train) if pos_width < abs(i - j) <= nonneg_width]
        if i == invalid_at:
            lines.append("an invalid line without separators\n")
        lines.append("%06d.bin | %s | %s\n" % (i, " ".join(map(str, pos)), " ".join(map(str, nonneg))))
    with open(os.path.join(root, "train_relative.txt"), "w") as f:
        f.write("".join(lines))
    numbers = [100 + 3 * i for i in range(n_test)] if test_numbers is None else list(test_numbers)
    gt, gt_desc = [], []
    for i, num in enumerate(numbers):
        np.save(oxford_test_path(root, num), synthetic_enu_scan(seed + 5000 + i, rows_of(0)))
        pos = [numbers[j] for j in range(len(numbers)) if 0 < abs(i - j) <= pos_width]
        far = [numbers[j] for j in range(len(numbers)) if abs(i - j) > nonneg_width]
        gt.append({"anc_idx": num, "pos_idx": pos[0] if pos else num, "neg_idx": far[0] if far else num,
                   "t": np.zeros(3), "q": np.array([1.0, 0, 0, 0])})
        gt_desc.append({"anc_idx": num, "pos_idx_list": pos})
    with open(os.path.join(root, OXFORD_TEST_FOLDER, "groundtruths.pkl"), "wb") as f:
        pickle.dump(gt, f)
    with open(os.path.join(root, OXFORD_TEST_FOLDER, "gt_descriptor_testing.pkl"), "wb") as f:
        pickle.dump(gt_desc, f)


# ----------------------------------------------------------------------------------------------- the builder
def check_oxford_opt(builder):
    if not 3 <= builder.S <= 8:
        raise ValueError("surface_normal_len %d: the Oxford loaders move sn columns 0:3 to the camera frame, so it must "
                         "be 3..8" % builder.S)


class _OxfordRows:
    """Both Oxford loaders draw input_pc_num rows without replacement and raise on a shorter scan."""

    def _check_rows(self, clouds, lengths):
        k = int(np.argmin(lengths))
        if lengths[k] < self.N:
            raise ValueError("scan %d has %d rows; input_pc_num = %d rows are drawn without replacement"
                             % (int(clouds[k]), int(lengths[k]), self.N))

    def _draw_rows_then_nodes(self, rng, n_valid, between=None):
        """Parity mode's draws of one Oxford item: rows of both clouds, `between(rng)` (or nothing), then the FPS
        candidates and start of each cloud -> ([(rows, cand, start)] * 2, what `between` returned)."""
        rows = [rng.choice(n, self.N, replace=False) for n in n_valid]
        mid = between(rng) if between is not None else None
        sides = []
        for r in rows:
            cand = rng.choice(self.N, self.n_cand, replace=False)
            sides.append((r, cand, rng.randint(len(cand))))
        return sides, mid


class OxfordPairBuilder(_OxfordRows, _PairBuilder):
    """Builds the nine `ModelDetector.set_input` tensors of a batch of Oxford pairs on the device.

    `build(scans, offsets, items, step=None)`: scans [T, C] f32 ENU (device, or host -- then the items' scans are
    uploaded), offsets (n_scans+1,) int64 row offsets (host), items the scan index of every pair.  Both clouds of a
    pair are independent subsamples of the same scan (oxford_detector_loader.py:185-186) and share the pair's height
    scale, params[:, 44].  Every scan needs input_pc_num rows; sn is columns 3:3+S with 3 <= S <= 8.

    See `_PairBuilder` for the two rng modes; rng="numpy" replays OxfordLoader.__getitem__, whose draws come in the
    order rows, rows, height scale, candidates and start of src, of dst, then the augmentation.
    """

    def __init__(self, opt, mode="train", device=None, seed=0, rng="device"):
        super().__init__(opt, mode, device, seed, rng, OXFORD_DET_DIVISOR)
        check_oxford_opt(self)
        self.height_scaling = mode == "train" and bool(getattr(opt, "is_height_scaling", True))
        self.flags |= ops.PAIR_ENU_TO_CAM | (ops.PAIR_HEIGHT_SCALE if self.height_scaling else 0)

    def _clouds(self, items):
        items = np.asarray(items, dtype=np.int64).ravel()
        if items.size == 0:
            raise ValueError("no items")
        return np.repeat(items, 2)

    def _scalars(self, rng, per_point):
        return draw_pair_scalars(rng, self.opt, self.mode == "train", self.N, self.M, self.S, per_point,
                                 scale_range=OXFORD_SCALE_RANGE)

    def _draw(self, rng, per_point):
        hs = rng.uniform(low=HEIGHT_SCALE_RANGE[0], high=HEIGHT_SCALE_RANGE[1])
        p, jit = self._scalars(rng, per_point)
        p[44] = hs
        return p, jit

    def _draw_item(self, rng, n_valid):
        sides, hs = self._draw_rows_then_nodes(
            rng, n_valid, lambda r: r.uniform(low=HEIGHT_SCALE_RANGE[0], high=HEIGHT_SCALE_RANGE[1]))
        p, jit = self._scalars(rng, True)
        p[44] = hs
        return sides, (p, jit)

    def _z_scale(self, params):
        if not self.height_scaling:
            return None
        return np.repeat(params[:, 44].astype(np.float32), 2)       # float32 array *= Python float

    def _augment(self, scans, offsets, scan_of_cloud, rows, nodes, params, step, jit):
        return ops.pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, self.S, self.flags, self.seed, step,
                                *jit)

    def build(self, scans, offsets, items, step=None):
        return self._build(scans, offsets, step, items)


class OxfordPairSource(_ScanSource):
    """Shuffled batches of Oxford detector pairs, built on the device and handed to `ModelDetector` (see
    `_ScanSource`).  The items are those of make_dataset_oxford_train(root) (train) or make_dataset_oxford_test(root)
    (test, item i reading the scan numbered dataset[i]['anc_idx']); `dataset` holds them.

        src = OxfordPairSource(root, "train", opt)
        for epoch in range(E):
            for _ in src.feed(model):
                model.optimize(epoch)
    """

    def __init__(self, root, mode, opt, device=None, seed=0, resident="host", rng="device", batch_size=None,
                 drop_last=True):
        if mode == "train":
            self.dataset = make_dataset_oxford_train(root)
            paths = [oxford_train_path(root, d["file"]) for d in self.dataset]
        elif mode == "test":
            self.dataset = make_dataset_oxford_test(root)
            paths = [oxford_test_path(root, int(d["anc_idx"])) for d in self.dataset]
        else:
            raise ValueError("mode must be 'train' or 'test'")
        if not paths:
            raise ValueError("no items under %s" % root)
        super().__init__(paths, mode, opt, OxfordPairBuilder, device, seed, resident, rng, batch_size, drop_last)

    def _build(self, items):
        return self.builder.build(self.scans, self.offsets, items, step=self.step), None
