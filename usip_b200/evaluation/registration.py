"""Outdoor registration on the GPU: evaluation/matlab/eval_outdoor/kitti/evaluate_kitti.m and
oxford/evaluate_oxford.m (descriptor matching, RANSAC of ransacfitRt.m, Utils.compareTransform), for the KITTI and
Oxford test sets, every K of a keypoint-count sweep and every maxTrials of automation_kitti.m's sweep at once.

One detector and descriptor pass over the test set (Repeatability.detect with a descriptor) keeps every scan's
keypoints, descriptors and selection order on the device; one launch of usip_desc_match_f64 matches every pair for
every K, and one launch of usip_ransac_rt_f64 runs RANSAC for every (pair, K) and every trial budget.  The score is
computed on the host in float64.

    ev = Registration(KittiRepeatability(txt_root, numpy_root, calib_root, opt))
    res = ev.run(detector, descriptor)          # a ModelDetector and a ModelDescriptor with trained weights
    print("\\n".join(res.lines()))

Per pair and K: each scan's first min(K, count) rows [xyz | descriptor] in selection order; xyz leaves the camera frame
as in repeatability.py (KITTI inv(Tr), Oxford the "my" branch (x, z, -y)).  Matching (Euclidean, float64 on float32
values): KITTI the 1-NN of every anchor among the positives, in anchor order; Oxford the k = 5 nearest positives of
every anchor united with the 5 nearest anchors of every positive, unique rows sorted by (anchor, positive).  RANSAC:
x1 = R x2 + t, inlier threshold 1.0, Horn's quaternion fit; see include/usip_b200.h for the exact rules.  Score:
dt = |t_gt - t|, ddeg = sum |rotm2eul(R_gt^T R)| * 180 / pi (ZYX), a failure when dt > 2 or ddeg > 5; no model counts
as dt = 3, ddeg = 6.  Summary per (K, maxTrials) as the scripts print it, plus registration recall 1 - wrong / P.

`write_descriptor_tree` writes the reference's result layout (float32 rows [xyz in the camera frame | descriptor], one
file per scan) for evaluate_*.m's RESULT_FOLDER; `read_descriptor_tree` scores an existing tree of that layout (for
example 3DFeat-Net's 128-D or SHOT's 352-D features), each file's rows taken in file order.

Deliberate deviations from the reference:
  * The random stream is Philox4x32-10 keyed by the seed, not MATLAB's randsample under rng(0); like rng(0) it is the
    same for every pair.  Trial counts are therefore comparable with the MATLAB numbers statistically, not bitwise.
  * Ties in descriptor distance go to the lowest index; pdist2's order among ties is unspecified.
  * Each scan keeps min(K, its own count) keypoints, as repeatability.py's selection does.
  * The isPrintWrong ground-truth diagnostics are dropped.
  * DescriptorLiteOld draws its point permutation from np.random (networks.py:345, as in the reference); `describe`
    gives it a numpy state seeded from the evaluator's seed, so two runs give the same descriptors.  The global
    np.random stream is left to the test loader (rng="numpy" parity mode replays it).
"""
import argparse
import json
import os

import numpy as np
import torch

from usip_b200 import ops

from .handcrafted import add_method_args, detector_from_args
from .repeatability import (DEFAULT_KEYPOINT_NUMS, KittiRepeatability, OxfordRepeatability, check_sweep,
                            detector_opt, load_checkpoint, load_detector_checkpoint)

DEFAULT_MAX_TRIALS = (50, 100, 250, 500, 1000, 2500, 5000, 10000)     # automation_kitti.m
DEFAULT_INLIER_THRESHOLD = 1.0                                         # evaluate_*.m: ransacfitRt(.., 1.0, ..)
DEFAULT_MATCH_K = {"kitti": 1, "oxford": 5}
MAX_KEYPOINTS = 1024                                                   # USIP_REG_MAX_KEYPOINTS
NO_MODEL = (3.0, 6.0)                                                  # evaluate_*.m's catch


def check_trials(max_trials, inlier_threshold):
    ts = [int(t) for t in max_trials]
    if not ts or any(t < 1 for t in ts) or any(b <= a for a, b in zip(ts, ts[1:])):
        raise ValueError("max_trials must be >= 1 and ascending, got %r" % (list(max_trials),))
    if len(ts) > 16 or ts[-1] > 100000:
        raise ValueError("at most 16 trial budgets, each <= 100000")
    if not inlier_threshold > 0:
        raise ValueError("inlier_threshold must be > 0, got %r" % inlier_threshold)
    return ts


def rotm2eul_zyx(R):
    """MATLAB rotm2eul(R) with its default 'ZYX' sequence: R (..., 3, 3) -> (..., 3) float64 radians."""
    R = np.asarray(R, dtype=np.float64)
    cy = np.sqrt(R[..., 0, 0] * R[..., 0, 0] + R[..., 1, 0] * R[..., 1, 0])
    singular = cy < 10 * np.finfo(np.float64).eps
    return np.stack([np.where(singular, 0.0, np.arctan2(R[..., 1, 0], R[..., 0, 0])),
                     np.arctan2(-R[..., 2, 0], cy),
                     np.where(singular, np.arctan2(-R[..., 1, 2], R[..., 1, 1]), np.arctan2(R[..., 2, 1], R[..., 2, 2]))],
                    axis=-1)


def compare_transforms(T_gt, Rt, has_model):
    """Utils.compareTransform over arrays: T_gt (..., 3, 4) against estimates Rt (..., 3, 4) (broadcast) -> (dt, ddeg)
    float64 arrays; where has_model is False, evaluate_*.m's catch values (3, 6)."""
    T_gt, Rt = np.asarray(T_gt, dtype=np.float64), np.asarray(Rt, dtype=np.float64)
    dt = np.sqrt(np.sum((T_gt[..., :, 3] - Rt[..., :, 3]) ** 2, axis=-1))
    dR = np.matmul(np.swapaxes(T_gt[..., :, :3], -1, -2), Rt[..., :, :3])
    dd = np.abs(rotm2eul_zyx(dR)).sum(axis=-1) * 180 / np.pi
    return np.where(has_model, dt, NO_MODEL[0]), np.where(has_model, dd, NO_MODEL[1])


def compare_transform(T_gt, Rt):
    """Utils.compareTransform: (dt, ddeg) of an estimate Rt (3, 4) against T_gt (3, 4); Rt None -> (3, 6)."""
    if Rt is None:
        return NO_MODEL
    dt, dd = compare_transforms(T_gt, Rt, True)
    return float(dt), float(dd)


def _mean_std(x):
    """MATLAB mean / std (N - 1 normalisation; a single value has std 0; empty -> NaN)."""
    x = np.asarray(x, dtype=np.float64)
    if x.size == 0:
        return float("nan"), float("nan")
    return float(x.mean()), float(x.std(ddof=1)) if x.size > 1 else 0.0


def _f(x):
    return "NaN" if np.isnan(x) else "%f" % x


def _check_keypoint_limit(ks):
    if ks[-1] > MAX_KEYPOINTS:
        raise ValueError("keypoint_nums: at most %d keypoints per scan can be registered, got K = %d"
                         % (MAX_KEYPOINTS, ks[-1]))


class _SeededNumpy:
    """A ModelDescriptor whose run_model draws np.random from its own seeded state (DescriptorLiteOld's point
    permutation, networks.py:345), leaving the global np.random state as it found it."""

    def __init__(self, model, seed):
        self.model, self.state = model, np.random.RandomState(seed).get_state()

    def run_model(self, pc, sn, keypoints):
        outer = np.random.get_state()
        np.random.set_state(self.state)
        try:
            return self.model.run_model(pc, sn, keypoints)
        finally:
            self.state = np.random.get_state()
            np.random.set_state(outer)


class RegistrationResult:
    """Per (pair, K, maxTrials), arrays (P, nK, nT): delta_t, delta_deg, success, inliers, npts, trialcount, status
    (usip_ransac_rt_f64's).  Per (K, maxTrials), arrays (nK, nT): wrong (evaluate_*.m's `wrong counter`), recall
    (1 - wrong / P), and over the successful pairs only inlier_ratio, trial_count, rte / rte_std, rre / rre_std."""

    def __init__(self, dataset, keypoint_nums, max_trials, inlier_threshold, match_k, delta_t, delta_deg, inliers,
                 npts, trialcount, status):
        self.dataset, self.keypoint_nums, self.max_trials = dataset, list(keypoint_nums), list(max_trials)
        self.inlier_threshold, self.match_k = float(inlier_threshold), int(match_k)
        self.delta_t, self.delta_deg = delta_t, delta_deg
        self.inliers, self.npts, self.trialcount, self.status = inliers, npts, trialcount, status
        self.success = ~((delta_t > 2) | (delta_deg > 5))
        P = delta_t.shape[0]
        shape = delta_t.shape[1:]
        self.wrong = (~self.success).sum(axis=0)
        self.recall = 1.0 - self.wrong / P
        stats = {k: np.full(shape, np.nan) for k in ("inlier_ratio", "trial_count", "rte", "rte_std", "rre", "rre_std")}
        for k in range(shape[0]):
            for t in range(shape[1]):
                ok = self.success[:, k, t]
                ratio = inliers[ok, k, t] / np.maximum(npts[ok, k, t], 1)
                stats["inlier_ratio"][k, t] = _mean_std(ratio)[0]
                stats["trial_count"][k, t] = _mean_std(trialcount[ok, k, t])[0]
                stats["rte"][k, t], stats["rte_std"][k, t] = _mean_std(delta_t[ok, k, t])
                stats["rre"][k, t], stats["rre_std"][k, t] = _mean_std(delta_deg[ok, k, t])
        self.__dict__.update(stats)

    def lines(self):
        """evaluate_*.m's two fprintf lines per (K, maxTrials), each on one line."""
        out = []
        for k, K in enumerate(self.keypoint_nums):
            for t, T in enumerate(self.max_trials):
                pre = "K=%d maxTrials=%d %s: " % (K, T, self.dataset)
                out.append(pre + "wrong counter: %d, inlier ratio %s, trial count %s"
                           % (self.wrong[k, t], _f(self.inlier_ratio[k, t]), _f(self.trial_count[k, t])))
                out.append(pre + "successful alignment RTE: %s +- %s, RRE: %s +- %s"
                           % (_f(self.rte[k, t]), _f(self.rte_std[k, t]), _f(self.rre[k, t]), _f(self.rre_std[k, t])))
        return out

    def to_dict(self):
        nan = lambda a: [[None if np.isnan(v) else float(v) for v in row] for row in a]
        return {"dataset": self.dataset, "keypoint_nums": self.keypoint_nums, "max_trials": self.max_trials,
                "inlier_threshold": self.inlier_threshold, "match_k": self.match_k,
                "pairs": int(self.delta_t.shape[0]), "wrong": self.wrong.tolist(), "recall": self.recall.tolist(),
                "inlier_ratio": nan(self.inlier_ratio), "trial_count": nan(self.trial_count),
                "rte": nan(self.rte), "rte_std": nan(self.rte_std), "rre": nan(self.rre), "rre_std": nan(self.rre_std)}


class Registration:
    """Registration of a test set: wraps a KittiRepeatability / OxfordRepeatability, whose source, pairs, frames and
    selection order it uses as they are.  After `describe` (or `read_descriptor_tree`) it holds every scan's rows in
    selection order: xyz (S, L, 3) f32 in the camera frame, desc (S, L, D) f32 and count (S,) i32, on the device."""

    def __init__(self, evaluator):
        self.ev = evaluator
        self.dataset = evaluator.dataset
        self.xyz = self.desc = self.count = None

    def describe(self, detector, descriptor, nms_radius=0.0, noise_sigma=0.0, L=MAX_KEYPOINTS):
        """One detector and descriptor pass over the test set, then each scan's first L rows in selection order.  The
        descriptor's np.random draws come from a numpy state seeded with the evaluator's seed and swapped in around
        each descriptor call, so the descriptors repeat from run to run and a source in rng="numpy" parity mode still
        sees the global np.random stream alone."""
        ev = self.ev
        ev.detect(detector, nms_radius, noise_sigma, descriptor=_SeededNumpy(descriptor, ev.source.seed))
        L = min(int(L), ev.keypoints.shape[2])
        idx = ev.order[:, :L].long().clamp(min=0)              # NMS pads the order with -1 past count
        self.xyz = torch.gather(ev.keypoints, 2, idx[:, None, :].expand(-1, 3, -1)).transpose(1, 2).contiguous()
        D = ev.descriptors.shape[1]
        self.desc = torch.gather(ev.descriptors, 2, idx[:, None, :].expand(-1, D, -1)).transpose(1, 2).contiguous()
        self.count = torch.clamp(ev.count, max=L).to(torch.int32).contiguous()

    def score(self, keypoint_nums=DEFAULT_KEYPOINT_NUMS, max_trials=DEFAULT_MAX_TRIALS,
              inlier_threshold=DEFAULT_INLIER_THRESHOLD, match_k=None, seed=0, uniforms=None, raw=False):
        """Matches, RANSAC and the score of the held rows -> RegistrationResult (and the kernels' raw outputs as
        numpy arrays when raw).  uniforms: None (Philox from seed) or (max(max_trials) + 1, 3) float64."""
        ks = check_sweep(keypoint_nums, 1.0)
        ts = check_trials(max_trials, inlier_threshold)
        k = DEFAULT_MATCH_K[self.dataset] if match_k is None else int(match_k)
        if self.xyz is None:
            raise RuntimeError("describe() or read_descriptor_tree() first")
        _check_keypoint_limit(ks)
        L = min(self.xyz.shape[1], ks[-1])
        dev = self.xyz.device
        xyz, desc = self.xyz[:, :L].contiguous(), self.desc[:, :L].contiguous()
        count = torch.clamp(self.count, max=L).to(torch.int32).contiguous()
        pairs = torch.from_numpy(self.ev.pairs).to(dev)
        frames = torch.from_numpy(self.ev.frames).to(dev)
        if uniforms is not None:
            uniforms = torch.as_tensor(np.ascontiguousarray(uniforms, dtype=np.float64)).to(dev)
        matches, n = ops.desc_match(desc, count, pairs, ks, k)
        out = ops.ransac_rt(xyz, count, pairs, frames, matches, n, ts, inlier_threshold, seed, uniforms)
        out = {key: v.cpu().numpy() for key, v in out.items()}
        npts = np.repeat(n.cpu().numpy()[:, :, None], len(ts), axis=2)
        dt, dd = compare_transforms(self.ev.frames[:, None, None, 2], out["Rt"], out["status"] == 0)
        res = RegistrationResult(self.dataset, ks, ts, inlier_threshold, k, dt, dd, out["n_inliers"], npts,
                                 out["trialcount"], out["status"])
        if raw:
            out["matches"], out["n_matches"] = matches.cpu().numpy(), n.cpu().numpy()
            return res, out
        return res

    def run(self, detector, descriptor, keypoint_nums=DEFAULT_KEYPOINT_NUMS, nms_radius=0.0, noise_sigma=0.0,
            max_trials=DEFAULT_MAX_TRIALS, inlier_threshold=DEFAULT_INLIER_THRESHOLD, match_k=None, seed=0):
        ks = check_sweep(keypoint_nums, 1.0)
        check_trials(max_trials, inlier_threshold)
        _check_keypoint_limit(ks)
        self.describe(detector, descriptor, nms_radius, noise_sigma, L=ks[-1])
        return self.score(ks, max_trials, inlier_threshold, match_k, seed)

    def write_descriptor_tree(self, out_dir, K):
        """evaluate_*.m's RESULT_FOLDER for K: one file per scan at source.keypoint_path, float32 rows
        [x y z (camera frame) | descriptor], the scan's first min(K, count) rows in selection order."""
        if self.xyz is None:
            raise RuntimeError("describe() first")
        xyz, desc, count = self.xyz.cpu().numpy(), self.desc.cpu().numpy(), self.count.cpu().numpy()
        for i in range(len(self.ev.source)):
            n = min(int(K), int(count[i]))
            path = self.ev.source.keypoint_path(out_dir, i)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.concatenate([xyz[i, :n], desc[i, :n]], axis=1).astype(np.float32).tofile(path)

    def read_descriptor_tree(self, tree_dir, feature_dim):
        """Holds the rows of an existing result tree (Utils.load_descriptors: float32 rows of 3 + feature_dim values,
        xyz in the camera frame), each file's rows in file order.  A file may hold more than MAX_KEYPOINTS rows: only
        its first K rows are ever scored, and `score` refuses K > MAX_KEYPOINTS."""
        rows = []
        for i in range(len(self.ev.source)):
            path = self.ev.source.keypoint_path(tree_dir, i)
            a = np.fromfile(path, dtype=np.float32)
            if a.size % (3 + int(feature_dim)):
                raise ValueError("%s: %d floats is not a whole number of %d-column rows"
                                 % (path, a.size, 3 + int(feature_dim)))
            rows.append(a.reshape(-1, 3 + int(feature_dim)))
        L = max(1, min(max(len(r) for r in rows), MAX_KEYPOINTS))
        S, D = len(rows), int(feature_dim)
        xyz = np.zeros((S, L, 3), np.float32)
        desc = np.zeros((S, L, D), np.float32)
        for i, r in enumerate(rows):
            n = min(len(r), L)
            xyz[i, :n], desc[i, :n] = r[:n, :3], r[:n, 3:]
        dev = self.ev.source.device
        self.xyz, self.desc = torch.from_numpy(xyz).to(dev), torch.from_numpy(desc).to(dev)
        self.count = torch.tensor([min(len(r), L) for r in rows], dtype=torch.int32, device=dev)


def descriptor_opt(dataset, **over):
    """The reference's descriptor options: KITTI / Oxford (kitti/ and oxford/options_descriptor.py) the detector's
    options plus ball_radius 2, ball_nsamples 64, descriptor_len 128, surface_normal_len 4; Redwood and 3DMatch
    (scenenn/options_descriptor.py) ball_radius 0.75, ball_nsamples 448, descriptor_len 128, sigma_max 0.5: the options
    of ModelDescriptorIndoor (DescriptorLiteOldGlobal, 64-row sub-groups of the 448-sample balls combined on the device).
    ModelDescriptor (DescriptorLiteOld) refuses balls above 128 samples."""
    if dataset in ("redwood", "3dmatch"):
        o = detector_opt(dataset, ball_radius=0.75, ball_nsamples=448, descriptor_len=128, surface_normal_len=4,
                         sigma_max=0.5, triple_loss_gamma=0.3)
        o.__dict__.update(over)
        return o
    o = detector_opt(dataset, ball_radius=2.0, ball_nsamples=64, descriptor_len=128, surface_normal_len=4,
                     sigma_max=3.0, triple_loss_gamma=0.5)
    o.__dict__.update(over)
    return o


def load_descriptor_checkpoint(model, path):
    """load_detector_checkpoint for a ModelDescriptor: a `module.` prefix is stripped."""
    load_checkpoint(model.descriptor, path)
    model.freeze_model()


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m usip_b200.evaluation.registration",
                                 description="Registration of a trained detector and descriptor (evaluate_kitti.m / "
                                             "evaluate_oxford.m) on the KITTI or Oxford test set.")
    ap.add_argument("dataset", choices=("kitti", "oxford"))
    ap.add_argument("--detector", help="detector state dict (the reference's *_net_detector.pth); --method tsf only")
    ap.add_argument("--descriptor", help="descriptor state dict (the reference's *_net_descriptor.pth)")
    ap.add_argument("--descriptor-tree", metavar="DIR", help="score an existing result tree instead")
    ap.add_argument("--feature-dim", type=int, default=128, help="descriptor length of --descriptor-tree")
    ap.add_argument("--txt-root", help="kitti: the folder of <seq>/groundtruths.txt and <seq>/correct_gt.txt")
    ap.add_argument("--numpy-root", help="kitti: the folder of <seq>/np_0.20_20480_r90_sn/%%06d.npy")
    ap.add_argument("--calib-root", help="kitti: the folder of <seq>/calib.txt")
    ap.add_argument("--root", help="oxford: the folder of test_models_20k_np_nofilter/")
    ap.add_argument("--gt", help="oxford: groundtruths.txt")
    ap.add_argument("--keypoint-nums", type=int, nargs="+", default=list(DEFAULT_KEYPOINT_NUMS))
    ap.add_argument("--max-trials", type=int, nargs="+", default=list(DEFAULT_MAX_TRIALS))
    ap.add_argument("--inlier-threshold", type=float, default=DEFAULT_INLIER_THRESHOLD)
    ap.add_argument("--match-k", type=int, default=None, help="1: one-way 1-NN (kitti default); 2..8: k-NN union "
                                                              "(oxford default 5)")
    ap.add_argument("--nms-radius", type=float, default=0.0)
    ap.add_argument("--noise-sigma", type=float, default=0.0)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--input-pc-num", type=int, default=16384)
    ap.add_argument("--node-num", type=int, default=512)
    ap.add_argument("--write-descriptors", metavar="DIR", help="also write the result tree of the largest K")
    ap.add_argument("--json", metavar="OUT", help="write the summary as JSON")
    add_method_args(ap)
    a = ap.parse_args(argv)
    _check_keypoint_limit(check_sweep(a.keypoint_nums, 1.0))
    check_trials(a.max_trials, a.inlier_threshold)
    hc = detector_from_args(a, ap)
    if not a.descriptor_tree and not ((a.detector or hc is not None) and a.descriptor):
        ap.error("give --detector (--method tsf) and --descriptor, or --descriptor-tree")
    if hc is not None and a.nms_radius >= 0.01:
        ap.error("--nms-radius applies to --method tsf only")
    opt = descriptor_opt(a.dataset, batch_size=a.batch_size, input_pc_num=a.input_pc_num, node_num=a.node_num)
    if a.dataset == "kitti":
        if not (a.txt_root and a.numpy_root and a.calib_root):
            ap.error("kitti needs --txt-root, --numpy-root and --calib-root")
        rep = KittiRepeatability(a.txt_root, a.numpy_root, a.calib_root, opt, seed=a.seed, batch_size=a.batch_size)
    else:
        if not (a.root and a.gt):
            ap.error("oxford needs --root and --gt")
        rep = OxfordRepeatability(a.root, a.gt, opt, seed=a.seed, batch_size=a.batch_size)
    ev = Registration(rep)
    if a.descriptor_tree:
        ev.read_descriptor_tree(a.descriptor_tree, a.feature_dim)
        res = ev.score(a.keypoint_nums, a.max_trials, a.inlier_threshold, a.match_k, a.seed)
    else:
        from usip_b200.models.keypoint_descriptor import ModelDescriptor
        from usip_b200.models.keypoint_detector import ModelDetector
        det = ModelDetector(opt) if hc is None else hc
        des = ModelDescriptor(opt)
        if hc is None:
            load_detector_checkpoint(det, a.detector)
        load_descriptor_checkpoint(des, a.descriptor)
        res = ev.run(det, des, a.keypoint_nums, a.nms_radius, a.noise_sigma, a.max_trials, a.inlier_threshold,
                     a.match_k, a.seed)
    print("\n".join(res.lines()))
    if hc is not None and not a.descriptor_tree:
        print(hc.count_summary())
    if a.write_descriptors:
        ev.write_descriptor_tree(a.write_descriptors, a.keypoint_nums[-1])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res.to_dict(), f, indent=1)
    return res


if __name__ == "__main__":
    main()
