"""Keypoint repeatability on the GPU: evaluation/save_keypoints.py (detection, NMS, sigma-sorted top K) followed by
evaluation/matlab/eval_repeatability/eval_rep.m (the score), for the KITTI, Oxford, rotated ModelNet40, Redwood and
3DMatch test sets.

One pass of the detector over the test set gives the whole keypoint-count sweep: every scan's keypoints, sigmas and
selection order stay on the device, each K reads a prefix of that order, and one launch of usip_repeatability_f64
scores every ground-truth pair for every K.  No keypoint files and no MATLAB are needed; `write_keypoint_tree` still
writes the reference's `.bin` layout for the reference's registration scripts.

    ev = KittiRepeatability(txt_root, numpy_root, calib_root, opt)
    res = ev.run(model)                  # model: a ModelDetector with trained weights
    print("\\n".join(res.lines()))

Per pair (anc, pos) and K, as eval_rep.m:142-146: the anchor's first min(K, count) keypoints and the positive's, both
mapped to the ground-truth frame (anchor: F_a; positive: T_gt after F_p, applied one after the other), and
inliers = #{anchor keypoints whose nearest positive keypoint is closer than inlier_radius}, a strict `<`;
repeatability = inliers / n_anc.  KITTI: keypoints leave the camera frame with inv(Tr) (cam2velodyne.m), Tr from
<calib_root>/<seq>/calib.txt; pairs from <txt_root>/<seq>/correct_gt.txt.  Oxford: coord_cam2enu.m, (x, y, z) ->
(x, z, -y); pairs from groundtruths.txt.  T_gt = [quat2rotm(q), t] with q normalised first, as MATLAB does.
ModelNet, Redwood and 3DMatch (eval_rep.m:87-126): F_a = F_p = I.  ModelNet pairs object i of original/ with object i
of rotated/, T_gt = [R, 0] from modelnet_info.mat; Redwood and 3DMatch pair the fragments of every gt.log line, T_gt =
the top three rows of its 4x4.  eval_rep.m's apply_transform(x, T) = [x 1] * T' is exactly the map applied here.

Deliberate deviations from the reference:
  * save_keypoints.py:348-349 overwrites desired_keypoint_num with the keypoint count of the first scan that has fewer
    after NMS, and that smaller K then applies to every later scan.  Here each scan keeps min(K, its own count).
  * With NMS off the reference's np.argsort is not stable; the sort here is, so keypoints with EQUAL sigma may come out
    in another order (as in save_keypoints.select_keypoints).
  * Every run draws its subsamples from a seed (or replays np.random in parity mode) instead of a fresh random state.
  * The homogeneous step of cam2velodyne.m is dropped: the keypoints go through the top three rows of inv(Tr).
  * 3DMatch fragments are taken in frame order, not os.listdir's (indoor_test_loader.py).
"""
import argparse
import json
import os
import types

import numpy as np
import torch

from usip_b200 import ops

from .indoor_test_loader import MATCH3D_SCENES, REDWOOD_SCENES, Match3DTestLoader, RedwoodTestLoader
from .kitti_test_loader import KittiTestLoader
from .modelnet_test_loader import ModelNetRotatedTestLoader, eul2rotm, write_rotated_modelnet  # noqa: F401
from .oxford_test_loader import OxfordTestLoader
from .save_keypoints import write_keypoints_bin

DEFAULT_KEYPOINT_NUMS = (4, 8, 16, 32, 64, 128, 256, 512)
DEFAULT_INLIER_RADIUS = 0.5                       # eval_rep.m:7
CAM_TO_ENU = np.array([[1.0, 0, 0, 0], [0, 0, 1.0, 0], [0, -1.0, 0, 0]])     # coord_cam2enu.m, as a 3x4 map


# ----------------------------------------------------------------------------------------------- ground truth
def quat2rotm(q):
    """MATLAB quat2rotm: q = (w, x, y, z), normalised first -> (3, 3) float64."""
    q = np.asarray(q, dtype=np.float64)
    w, x, y, z = q / np.sqrt(np.sum(q * q))
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def gt_transform(t, q):
    """eval_rep.m:58-60: T_gt = [quat2rotm(q), t'] -> (3, 4) float64."""
    return np.concatenate([quat2rotm(q), np.asarray(t, dtype=np.float64).reshape(3, 1)], axis=1)


def read_correct_gt_kitti(txt_path):
    """read_txts_correct_kitti.m for one sequence: correct_gt.txt, comma-separated, one header line; columns idx1, idx2,
    t1..t3, qw, qx, qy, qz -> (n, 9) float64."""
    rows = []
    with open(txt_path) as f:
        for line in f.readlines()[1:]:
            if line.strip():
                rows.append([float(v) for v in line.split(",")[:9]])
    return np.array(rows, dtype=np.float64).reshape(-1, 9)


def read_gt_oxford(txt_path):
    """read_txt_oxford.m: groundtruths.txt, tab-separated, one header line; columns 1, 2 and 5-11 (anc, pos, t, q wxyz)
    -> (n, 9) float64."""
    rows = []
    with open(txt_path) as f:
        for line in f.readlines()[1:]:
            parts = line.rstrip("\r\n").split("\t")
            if len(parts) < 11:
                continue
            rows.append([float(parts[k]) for k in (0, 1, 4, 5, 6, 7, 8, 9, 10)])
    return np.array(rows, dtype=np.float64).reshape(-1, 9)


def read_kitti_calib(path):
    """read_kitti_calib.m: the first five lines `<name>: 12 values`, each a row-major 3x4 plus [0 0 0 1] -> {name:
    (4, 4) float64}."""
    out = {}
    with open(path) as f:
        for line in f.readlines()[:5]:
            parts = line.split()
            if len(parts) < 13:
                continue
            out[parts[0].rstrip(":")] = np.concatenate([np.array(parts[1:13], dtype=np.float64).reshape(3, 4),
                                                        [[0, 0, 0, 1.0]]])
    return out


def read_gt_log(path):
    """mrLoadLog.m: a stream of whitespace-separated numbers, three integers (anc, pos, and a count) then 16 numbers
    forming a row-major 4x4, repeated until fewer than three integers remain -> (anc (n,) int64, pos (n,) int64,
    T (n, 3, 4) float64, the top three rows)."""
    with open(path) as f:
        tok = f.read().split()
    anc, pos, T = [], [], []
    at = 0
    while at + 3 <= len(tok):
        try:
            head = [int(t) for t in tok[at:at + 3]]
        except ValueError:
            break
        m = tok[at + 3:at + 19]
        if len(m) != 16:
            raise ValueError("%s: the entry for (%d, %d) has %d of its 16 matrix values" % (path, head[0], head[1],
                                                                                             len(m)))
        anc.append(head[0]); pos.append(head[1])
        T.append(np.array(m, dtype=np.float64).reshape(4, 4)[:3])
        at += 19
    return (np.array(anc, dtype=np.int64), np.array(pos, dtype=np.int64),
            np.array(T, dtype=np.float64).reshape(-1, 3, 4))


def read_modelnet_info(path):
    """modelnet_info.mat (rotate_modelnet_dateset.m): the cell array modelnet_info, one row per object; column 3 is
    T = [R, 0] -> (n, 3, 4) float64.  scipy reads MATLAB files up to v7; a v7.3 (HDF5) file raises ValueError."""
    import scipy.io
    try:
        info = scipy.io.loadmat(path)["modelnet_info"]
    except NotImplementedError as e:
        raise ValueError("%s is a MATLAB v7.3 (HDF5) file, which scipy.io cannot read; re-save it with "
                         "save(..., '-v7')" % path) from e
    return np.stack([np.asarray(info[i, 2], dtype=np.float64).reshape(3, 4) for i in range(info.shape[0])])


def cam_to_velodyne(Tr):
    """cam2velodyne.m without the homogeneous division: the top three rows of inv(Tr)."""
    return np.linalg.inv(np.asarray(Tr, dtype=np.float64))[:3]


def check_sweep(keypoint_nums, inlier_radius):
    ks = [int(k) for k in keypoint_nums]
    if not ks or any(k <= 0 for k in ks) or any(b <= a for a, b in zip(ks, ks[1:])):
        raise ValueError("keypoint_nums must be positive and ascending, got %r" % (list(keypoint_nums),))
    if len(ks) > 32:
        raise ValueError("at most 32 keypoint numbers per sweep")
    if not inlier_radius > 0:
        raise ValueError("inlier_radius must be > 0, got %r" % inlier_radius)
    return ks


# ----------------------------------------------------------------------------------------------- selection
def select_order(keypoints, sigmas, nms_radius):
    """save_keypoints.py:336-351 for every scan at once -> (order (S, M) i32, count (S,) i32): the first count[s]
    entries of order[s] are scan s's keypoints in ascending sigma, after NMS when nms_radius >= 0.01."""
    if nms_radius < 0.01:
        order = torch.sort(sigmas, dim=1, stable=True).indices.to(torch.int32)
        count = torch.full((sigmas.shape[0],), sigmas.shape[1], dtype=torch.int32, device=sigmas.device)
        return order, count
    return ops.nms(keypoints, sigmas, nms_radius)


# ----------------------------------------------------------------------------------------------- result
class RepeatabilityResult:
    """Per pair and K: inliers and n_anc (P, nK) int; per K (eval_rep.m:152-154): mean_repeatability,
    mean_keypoint_num, min_repeatability, max_repeatability."""

    def __init__(self, dataset, keypoint_nums, inlier_radius, inliers, n_anc):
        self.dataset, self.keypoint_nums, self.inlier_radius = dataset, list(keypoint_nums), float(inlier_radius)
        self.inliers, self.n_anc = inliers, n_anc
        rep = inliers / np.maximum(n_anc, 1)
        self.repeatability = rep
        self.mean_repeatability = rep.mean(axis=0)
        self.mean_keypoint_num = n_anc.mean(axis=0)
        self.min_repeatability = rep.min(axis=0)
        self.max_repeatability = rep.max(axis=0)

    def lines(self):
        """eval_rep.m:153-154's two lines per K."""
        out = []
        for k, K in enumerate(self.keypoint_nums):
            out.append("K=%d %s: average keypoint number: %d, repeatability: %f"
                       % (K, self.dataset, round(self.mean_keypoint_num[k]), self.mean_repeatability[k]))
            out.append("K=%d %s: min repeatability: %f, max repeatability: %f"
                       % (K, self.dataset, self.min_repeatability[k], self.max_repeatability[k]))
        return out

    def to_dict(self):
        return {"dataset": self.dataset, "keypoint_nums": self.keypoint_nums, "inlier_radius": self.inlier_radius,
                "pairs": int(self.inliers.shape[0]),
                "mean_repeatability": self.mean_repeatability.tolist(),
                "mean_keypoint_num": self.mean_keypoint_num.tolist(),
                "min_repeatability": self.min_repeatability.tolist(),
                "max_repeatability": self.max_repeatability.tolist()}


# ----------------------------------------------------------------------------------------------- the evaluator
class Repeatability:
    """A test source (KittiTestLoader / OxfordTestLoader) and its ground truth: pair_keys [(anc key, pos key)] in the
    source's `key` naming, frames (P, 3, 3, 4) float64 (F_a, F_p, T_gt).  A pair naming a scan the source does not list
    raises KeyError."""

    dataset = "dataset"

    def __init__(self, source, pair_keys, frames):
        self.source = source
        index = {source.key(i): i for i in range(len(source))}
        pairs = []
        for a, p in pair_keys:
            for k in (a, p):
                if k not in index:
                    raise KeyError("ground truth names scan %r, which the test list does not detect" % (k,))
            pairs.append((index[a], index[p]))
        self.pairs = np.array(pairs, dtype=np.int32).reshape(-1, 2)
        self.frames = np.ascontiguousarray(frames, dtype=np.float64).reshape(-1, 3, 3, 4)
        if len(self.pairs) == 0 or len(self.pairs) != len(self.frames):
            raise ValueError("need one frame triple per ground-truth pair, and at least one pair")
        self.keypoints = self.sigmas = self.order = self.count = self.descriptors = None

    def detect(self, model, nms_radius=0.0, noise_sigma=0.0, descriptor=None):
        """Runs the detector over the whole test set and keeps every scan's keypoints (S, 3, M), sigmas (S, M) and
        selection order / count on the device.  With a ModelDescriptor `descriptor`, every batch is also described at
        its keypoints, on the clouds the detector saw (noise included), and descriptors (S, D, M) are kept too."""
        src = self.source
        dev = src.device
        S, M = len(src), src.M
        kp = torch.empty((S, 3, M), dtype=torch.float32, device=dev)
        sg = torch.empty((S, M), dtype=torch.float32, device=dev)
        desc = None
        for items, (pc, sn, node) in src.batches(noise_sigma):
            k, s = model.run_model(pc, sn, node)
            kp[items[0]:items[-1] + 1] = k
            sg[items[0]:items[-1] + 1] = s
            if descriptor is not None:
                d = descriptor.run_model(pc, sn, k)
                if desc is None:
                    desc = torch.empty((S, d.shape[1], M), dtype=torch.float32, device=dev)
                desc[items[0]:items[-1] + 1] = d
        self.keypoints, self.sigmas, self.descriptors = kp, sg, desc
        self.order, self.count = select_order(kp, sg, nms_radius)

    def score(self, keypoint_nums=DEFAULT_KEYPOINT_NUMS, inlier_radius=DEFAULT_INLIER_RADIUS):
        """Scores the last detection -> RepeatabilityResult."""
        ks = check_sweep(keypoint_nums, inlier_radius)
        if self.keypoints is None:
            raise RuntimeError("detect() first")
        dev = self.keypoints.device
        pairs = torch.from_numpy(self.pairs).to(dev)
        frames = torch.from_numpy(self.frames).to(dev)
        inl, n_anc = ops.repeatability(self.keypoints, self.order, self.count, pairs, frames, ks, inlier_radius)
        return RepeatabilityResult(self.dataset, ks, inlier_radius, inl.cpu().numpy(), n_anc.cpu().numpy())

    def run(self, model, keypoint_nums=DEFAULT_KEYPOINT_NUMS, nms_radius=0.0, inlier_radius=DEFAULT_INLIER_RADIUS,
            noise_sigma=0.0):
        check_sweep(keypoint_nums, inlier_radius)
        self.detect(model, nms_radius, noise_sigma)
        return self.score(keypoint_nums, inlier_radius)

    def selected(self, i, K):
        """Scan i's first min(K, count) keypoints in selection order, (n, 3) float32 CUDA."""
        n = min(int(K), int(self.count[i]))
        return self.keypoints[i][:, self.order[i, :n].long()].t().contiguous()

    def write_keypoint_tree(self, out_dir, K):
        """The reference's keypoint files for K (save_keypoints.py:367-393): KITTI %02d/%06d.bin, Oxford %d.bin,
        ModelNet original|rotated/%d.bin, Redwood and 3DMatch <scene>/%d.bin."""
        if self.keypoints is None:
            raise RuntimeError("detect() first")
        for i in range(len(self.source)):
            path = self.source.keypoint_path(out_dir, i)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            write_keypoints_bin(path, self.selected(i, K))


class KittiRepeatability(Repeatability):
    """The KITTI test set: scans from KittiTestLoader(txt_root, numpy_root, opt), pairs from every sequence's
    <txt_root>/<seq>/correct_gt.txt, frames inv(Tr) of <calib_root>/<seq>/calib.txt."""

    dataset = "kitti"

    def __init__(self, txt_root, numpy_root, calib_root, opt, device=None, seed=0, rng="device", batch_size=8):
        source = KittiTestLoader(txt_root, numpy_root, opt, device, seed, rng, batch_size)
        keys, frames = [], []
        for seq in sorted({d["seq"] for d in source.dataset}):
            gt = read_correct_gt_kitti(os.path.join(txt_root, "%02d" % seq, "correct_gt.txt"))
            F = cam_to_velodyne(read_kitti_calib(os.path.join(calib_root, "%02d" % seq, "calib.txt"))["Tr"])
            for row in gt:
                keys.append(((seq, int(row[0])), (seq, int(row[1]))))
                frames.append(np.stack([F, F, gt_transform(row[2:5], row[5:9])]))
        super().__init__(source, keys, np.array(frames).reshape(-1, 3, 3, 4))


class OxfordRepeatability(Repeatability):
    """The Oxford test set: scans from OxfordTestLoader(root, opt), pairs from gt_path (groundtruths.txt), frames
    coord_cam2enu."""

    dataset = "oxford"

    def __init__(self, root, gt_path, opt, device=None, seed=0, rng="device", batch_size=8, numbers=None):
        source = OxfordTestLoader(root, opt, device, seed, rng, batch_size, numbers)
        gt = read_gt_oxford(gt_path)
        keys = [(int(r[0]), int(r[1])) for r in gt]
        frames = [np.stack([CAM_TO_ENU, CAM_TO_ENU, gt_transform(r[2:5], r[5:9])]) for r in gt]
        super().__init__(source, keys, np.array(frames).reshape(-1, 3, 3, 4))


class _IdentityFrameRepeatability(Repeatability):
    """Pairs whose keypoints are already in one frame up to T_gt: F_a = F_p = I (eval_rep.m:87-126)."""

    def __init__(self, source, pair_keys, T_gt):
        T_gt = np.asarray(T_gt, dtype=np.float64).reshape(-1, 3, 4)
        I = np.broadcast_to(np.eye(3, 4), T_gt.shape)
        super().__init__(source, pair_keys, np.stack([I, I, T_gt], axis=1))


class ModelNetRepeatability(_IdentityFrameRepeatability):
    """Rotated ModelNet40: scans from ModelNetRotatedTestLoader(root, opt), one pair (original i, rotated i) per row of
    <root>/modelnet_info.mat (or info_path), T_gt = its [R, 0]."""

    dataset = "modelnet"

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=4, info_path=None):
        T = read_modelnet_info(info_path or os.path.join(root, "modelnet_info.mat"))
        source = ModelNetRotatedTestLoader(root, opt, device, seed, rng, batch_size, n=len(T))
        keys = [(("original", i), ("rotated", i)) for i in range(len(T))]
        super().__init__(source, keys, T)


def _gt_log_pairs(scenes, log_path):
    keys, T = [], []
    for scene in scenes:
        anc, pos, t = read_gt_log(log_path(scene))
        keys += [((scene, int(a)), (scene, int(p))) for a, p in zip(anc, pos)]
        T.append(t)
    return keys, np.concatenate(T) if T else np.zeros((0, 3, 4))


class RedwoodRepeatability(_IdentityFrameRepeatability):
    """Redwood: scans from RedwoodTestLoader(npy_root, opt) (numpy_gt_normal), pairs and T_gt from every scene's
    <gt_root>/original/<scene>-evaluation/gt.log (build_redwood_dataset.m)."""

    dataset = "redwood"

    def __init__(self, npy_root, gt_root, opt, device=None, seed=0, rng="device", batch_size=8,
                 scenes=REDWOOD_SCENES):
        source = RedwoodTestLoader(npy_root, opt, device, seed, rng, batch_size, scenes)
        keys, T = _gt_log_pairs([s for s, _ in source.scenes],
                                lambda s: os.path.join(gt_root, "original", "%s-evaluation" % s, "gt.log"))
        super().__init__(source, keys, T)


class Match3DRepeatability(_IdentityFrameRepeatability):
    """3DMatch: scans from Match3DTestLoader(root, opt) (3DMatch_eval_npy), pairs and T_gt from every scene's
    <gt_root>/<scene>-evaluation/gt.log, gt_root = root by default (build_3dmatch_dataset.m)."""

    dataset = "3dmatch"

    def __init__(self, root, opt, device=None, seed=0, rng="device", batch_size=8, gt_root=None, files=None,
                 scenes=MATCH3D_SCENES):
        source = Match3DTestLoader(root, opt, device, seed, rng, batch_size, files, scenes)
        keys, T = _gt_log_pairs(source.scenes,
                                lambda s: os.path.join(gt_root or root, "%s-evaluation" % s, "gt.log"))
        super().__init__(source, keys, T)


# ----------------------------------------------------------------------------------------------- command line
DATASETS = ("kitti", "oxford", "modelnet", "redwood", "3dmatch")
DEFAULT_BATCH_SIZE = {"modelnet": 4}              # 8 for the others


def detector_opt(dataset, **over):
    """The reference's detector options for evaluation on cuda:0: kitti/ and oxford/options_detector.py; modelnet/
    (modelnet), scenenn/ (redwood) and match3d/options_detector.py (3dmatch).  loss_sigma_lower_bound enters the
    sigmas, and so the keypoint order."""
    if dataset not in DATASETS:
        raise ValueError("dataset must be one of %s, got %r" % (", ".join(DATASETS), dataset))
    o = types.SimpleNamespace(
        gpu_ids=[0], device=torch.device("cuda:0"), scene="outdoor", batch_size=8, input_pc_num=16384,
        surface_normal_len=4, node_num=512, k=1, node_knn_k_1=16, activation="relu", normalization="batch",
        bn_momentum=0.1, bn_momentum_decay_step=None, bn_momentum_decay=0.6, lr=0.001, loss_sigma_lower_bound=0.001,
        random_pc_dropout_lower_limit=1.0, keypoint_on_pc_type="point_to_point",
        keypoint_on_pc_alpha=0.01 if dataset == "kitti" else 1.0, rot_3d=False, rot_horizontal=True,
        rot_perturbation=False, translation_perturbation=False, checkpoints_dir="./checkpoints")
    if dataset == "modelnet":
        o.__dict__.update(scene="object", batch_size=4, input_pc_num=5000, surface_normal_len=3, node_knn_k_1=32,
                          loss_sigma_lower_bound=1e-4, keypoint_on_pc_alpha=1.0, rot_3d=True, rot_horizontal=False)
    elif dataset in ("redwood", "3dmatch"):
        o.__dict__.update(input_pc_num=10240, node_knn_k_1=32, loss_sigma_lower_bound=1e-4,
                          keypoint_on_pc_alpha=100.0 if dataset == "redwood" else 10.0, rot_3d=True,
                          rot_horizontal=False)
    o.__dict__.update(over)
    return o


def load_checkpoint(net, path):
    """torch.load + model_state_dict_convert_auto for one GPU (save_keypoints.py:168-177) into `net`: a `module.`
    prefix is stripped."""
    sd = torch.load(path, map_location="cpu")
    if any(k.startswith("module.") for k in sd):
        sd = {k[7:]: v for k, v in sd.items()}
    net.load_state_dict(sd)


def load_detector_checkpoint(model, path):
    load_checkpoint(model.detector, path)
    model.freeze_model()


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m usip_b200.evaluation.repeatability",
                                 description="Keypoint repeatability of a trained detector (save_keypoints.py + "
                                             "eval_rep.m) on the KITTI, Oxford, rotated ModelNet40, Redwood or 3DMatch "
                                             "test set.")
    ap.add_argument("dataset", choices=DATASETS)
    ap.add_argument("--checkpoint", required=True, help="detector state dict (the reference's *_net_detector.pth)")
    ap.add_argument("--txt-root", help="kitti: the folder of <seq>/groundtruths.txt and <seq>/correct_gt.txt")
    ap.add_argument("--numpy-root", help="kitti: the folder of <seq>/np_0.20_20480_r90_sn/%%06d.npy")
    ap.add_argument("--calib-root", help="kitti: the folder of <seq>/calib.txt")
    ap.add_argument("--root", help="oxford: the folder of test_models_20k_np_nofilter/; modelnet: the rotated tree "
                                   "(original/, rotated/, modelnet_info.mat); redwood: numpy_gt_normal/; 3dmatch: "
                                   "3DMatch_eval_npy/")
    ap.add_argument("--gt", help="oxford: groundtruths.txt; modelnet: modelnet_info.mat (default <root>/...)")
    ap.add_argument("--gt-root", help="redwood: the folder of original/<scene>-evaluation/gt.log; 3dmatch: the folder "
                                      "of <scene>-evaluation/gt.log (default --root)")
    ap.add_argument("--keypoint-nums", type=int, nargs="+", default=list(DEFAULT_KEYPOINT_NUMS))
    ap.add_argument("--nms-radius", type=float, default=0.0)
    ap.add_argument("--inlier-radius", type=float, default=DEFAULT_INLIER_RADIUS)
    ap.add_argument("--noise-sigma", type=float, default=0.0)
    ap.add_argument("--batch-size", type=int, help="default 4 for modelnet, 8 otherwise")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--input-pc-num", type=int, help="default: the dataset's (16384, 5000 for modelnet, 10240 for "
                                                     "redwood and 3dmatch)")
    ap.add_argument("--node-num", type=int, default=512)
    ap.add_argument("--write-keypoints", metavar="DIR", help="also write the .bin tree of the largest K")
    ap.add_argument("--json", metavar="OUT", help="write the summary as JSON")
    a = ap.parse_args(argv)
    check_sweep(a.keypoint_nums, a.inlier_radius)
    from usip_b200.models.keypoint_detector import ModelDetector
    bs = a.batch_size or DEFAULT_BATCH_SIZE.get(a.dataset, 8)
    over = {"batch_size": bs, "node_num": a.node_num}
    if a.input_pc_num:
        over["input_pc_num"] = a.input_pc_num
    opt = detector_opt(a.dataset, **over)
    kw = {"seed": a.seed, "batch_size": bs}
    if a.dataset == "kitti":
        if not (a.txt_root and a.numpy_root and a.calib_root):
            ap.error("kitti needs --txt-root, --numpy-root and --calib-root")
        ev = KittiRepeatability(a.txt_root, a.numpy_root, a.calib_root, opt, **kw)
    elif a.dataset == "oxford":
        if not (a.root and a.gt):
            ap.error("oxford needs --root and --gt")
        ev = OxfordRepeatability(a.root, a.gt, opt, **kw)
    elif a.dataset == "modelnet":
        if not a.root:
            ap.error("modelnet needs --root")
        ev = ModelNetRepeatability(a.root, opt, info_path=a.gt, **kw)
    elif a.dataset == "redwood":
        if not (a.root and a.gt_root):
            ap.error("redwood needs --root and --gt-root")
        ev = RedwoodRepeatability(a.root, a.gt_root, opt, **kw)
    else:
        if not a.root:
            ap.error("3dmatch needs --root")
        ev = Match3DRepeatability(a.root, opt, gt_root=a.gt_root, **kw)
    model = ModelDetector(opt)
    load_detector_checkpoint(model, a.checkpoint)
    res = ev.run(model, a.keypoint_nums, a.nms_radius, a.inlier_radius, a.noise_sigma)
    print("\n".join(res.lines()))
    if a.write_keypoints:
        ev.write_keypoint_tree(a.write_keypoints, a.keypoint_nums[-1])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res.to_dict(), f, indent=1)
    return res


if __name__ == "__main__":
    main()
