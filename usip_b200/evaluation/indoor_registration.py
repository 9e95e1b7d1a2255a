"""Indoor registration on the GPU: the geometric-registration benchmark of Choi et al. as
evaluation/matlab/eval_indoor/3dmatch/ runs it (runFragmentRegistration.m -> clusterCallback.m -> register2Fragments.m,
writeLog.m, evaluate.m -> mrEvaluateRegistrationMy.m), for the Redwood and 3DMatch test sets, every K of a keypoint-count
sweep and every maxTrials of a sweep at once.

    ev = IndoorRegistration.redwood(npy_root, gt_root, descriptor_opt("redwood"))
    ev.read_descriptor_tree(tree, 128)            # or ev.describe(detector, ModelDescriptorIndoor)
    res = ev.score()
    print("\\n".join(res.lines()))
    ev.write_registration_logs(out_dir, K=512, max_trials=30000)
    res = ev.score(solver="fgr")                   # Fast Global Registration instead of RANSAC
    ev.write_registration_logs(out_dir, K=512)

Per scene, the fragment pairs are every i < j by frame number (pairs="all", runFragmentRegistration.m) or the gt.log
pairs only (pairs="gt", the overlapped-pairs variant).  Frames are the identity.  Per pair and K, on the device:
matches (k = 5 nearest both ways, united: usip_desc_match_f64), RANSAC with inlier threshold 0.2 for the whole maxTrials
sweep in one stream (usip_ransac_rt_f64), the information matrix sum A^T A over the best model's inliers
(usip_ransac_info_f64), and, for the (pair, K, maxTrials) entries whose inlierRatio = inliers / matches exceeds 0.025,
the share of fragment 1's points within 0.2 of the mapped fragment 2 over the full fragments (usip_fragment_overlap_f32,
ratioAligned(1)).  An entry enters the scene's log iff ratioAligned(1) > 0.23 and inlierRatio > 0.025 (writeLog.m).
The score (mrEvaluateRegistrationMy.m) counts only pairs with j - i > 1: p = er' info er / info(1, 1) with er = [t;
-q(2:4)] of inv(T_gt) T and dcm2quat as written there; a pair is good iff p <= 0.04; recall = good / gt_num, precision =
good / rs_num, and the mean inlierNum and inlierRatio over the good pairs.  The summary is evaluate.m's mean over scenes.

Deliberate deviations from the reference:
  * The random stream is Philox4x32-10 keyed by the seed (see registration.py), not randsample under rng(0).
  * MATLAB maps fragment 2 in single precision with its BLAS's order; here every point is mapped in fp64 and rounded
    once to fp32.  Only points within rounding distance of the 0.2 m shell can come out differently.
  * A pair whose RANSAC has no model (fewer than 3 matches, or a best set under 3 inliers) gets the identity and no
    inliers, which is register2Fragments.m's catch; MATLAB reaches that catch for the first case and errors on the
    empty Rt of the second.
  * The .log is written straight from the kernels' fp64 results (%.10f), not re-read from the %15.8e of a per-pair
    .rt.txt.
  * 3DMatch fragments are taken in frame order (indoor_test_loader.py).

solver="fgr" registers with Fast Global Registration instead (evaluation/matlab/eval_indoor/fgr/,
register2FragmentsFGR.m; usip_desc_match_mutual_f64 and usip_fgr_f64, see include/usip_b200.h): mutual nearest
descriptor matches, FGR's tuple test and its 640 graduated non-convexity iterations, for every pair and K in one launch.
The trial axis then has length 1 and no maxTrials.  Its further deviations:
  * register2FragmentsFGR.m writes constant statistics (numInliers 1, inlierRatio 0.99, ratioAligned 0.8) and no
    information matrix.  Here they are measured under the final T: the mutual matches within 0.2 (the RANSAC inlier
    test), inlierRatio = inliers / mutual matches, info = sum A^T A over them as for RANSAC, and the overlap test and
    writeLog.m's filters run as for RANSAC (overlap_threshold None keeps ratioAligned = 0.8).
  * The library seeds rand() with time(NULL); here the tuple draws are Philox4x32-10 keyed by the seed, the same stream
    for every pair and K.
  * The library matches with FLANN and moves the points in float; here everything is fp64.
  * The library divides by zero with no correspondences; here that, like any pair with fewer than 10 tuple
    correspondences, gets no iterations (status 1).  A fragment whose centred points all coincide (scale 0) is status
    4.  Only status 0 counts as a model, as for RANSAC.

Descriptors (describe, with a ModelDescriptorIndoor): DescriptorLiteOldGlobal's global context is the max over the
keypoints the descriptor is given.  describe() gives it all M keypoints of the detector pass, before NMS and before the
top-K selection -- the keypoint set scenenn/train_descriptor.py:116-119 feeds it in training -- so one descriptor pass
serves the whole K sweep.  The reference's save_keypoints.py computes no descriptors, so there is no reference policy for
this.
"""
import argparse
import json
import math
import os

import numpy as np
import torch

from usip_b200 import ops

from .handcrafted import add_method_args, detector_from_args
from .indoor_test_loader import MATCH3D_SCENES, REDWOOD_SCENES
from .registration import Registration, _check_keypoint_limit, check_trials, descriptor_opt
from .repeatability import (DEFAULT_KEYPOINT_NUMS, Match3DRepeatability, RedwoodRepeatability, check_sweep,
                            read_gt_log)

DEFAULT_MAX_TRIALS = (1000, 30000)        # the overlapped-pairs note of fullEvaluation.m; ransac.m's default
INLIER_THRESHOLD = 0.2                    # register2Fragments.m:14
MATCH_K = 5                               # register2Fragments.m:49
OVERLAP_RADIUS = 0.2                      # register2Fragments.m:135
DEFAULT_OVERLAP_THRESHOLD = 0.23          # writeLog.m: resultAlignRatio(1) > 0.23
INLIER_RATIO_THRESHOLD = 0.025            # writeLog.m: resultInlierRatio > 0.025
ERR2 = 0.04                               # mrEvaluateRegistrationMy.m
MATCH_BUFFER_BYTES = 1 << 28              # pairs per launch: the match list of one chunk stays under 256 MB
SOLVERS = ("ransac", "fgr")
FGR_MAX_DIM = 512                         # USIP_REG_MAX_DIM
FGR_MAX_ROWS = 1024                       # USIP_REG_MAX_KEYPOINTS


# ----------------------------------------------------------------------------------------------- files
def _numbers(path):
    with open(path) as f:
        return f.read().split()


def _head(tok, at):
    try:
        return [int(t) for t in tok[at:at + 3]]
    except ValueError:
        return None


def read_gt_info(path):
    """mrLoadInfo.m: three integers (i, j, count), then a 6x6 read row by row, repeated until fewer than three integers
    remain -> (head (n, 3) int64, info (n, 6, 6) float64), in the file's order (the order of gt.log)."""
    tok, heads, mats, at = _numbers(path), [], [], 0
    while at + 3 <= len(tok):
        head = _head(tok, at)
        if head is None:
            break
        m = tok[at + 3:at + 39]
        if len(m) != 36:
            raise ValueError("%s: the entry for (%d, %d) has %d of its 36 values" % (path, head[0], head[1], len(m)))
        heads.append(head)
        mats.append(np.array(m, dtype=np.float64).reshape(6, 6))
        at += 39
    return np.array(heads, dtype=np.int64).reshape(-1, 3), np.array(mats, dtype=np.float64).reshape(-1, 6, 6)


def read_gt_log4(path):
    """mrLoadLog.m -> (head (n, 3) int64, T (n, 4, 4) float64)."""
    anc, pos, T = read_gt_log(path)
    with open(path) as f:
        tok = f.read().split()
    count = [int(tok[19 * e + 2]) for e in range(len(anc))]
    T4 = np.zeros((len(anc), 4, 4))
    T4[:, :3] = T
    for e in range(len(anc)):
        T4[e, 3] = np.array(tok[19 * e + 15:19 * e + 19], dtype=np.float64)
    return np.stack([anc, pos, np.array(count, dtype=np.int64)], axis=1).reshape(-1, 3), T4


def read_registration_log(path):
    """mrLoadLogMy.m: per entry (i, j, count), a 4x4 read row by row, inlierNum and inlierRatio, and a 6x6 read column
    by column (fscanf's [6 6] without the transpose) -> dict of head (n, 3) int64, T (n, 4, 4), inlier_num (n,),
    inlier_ratio (n,), info (n, 6, 6)."""
    tok, at = _numbers(path), 0
    out = {"head": [], "T": [], "inlier_num": [], "inlier_ratio": [], "info": []}
    while at + 3 <= len(tok):
        head = _head(tok, at)
        if head is None:
            break
        body = tok[at + 3:at + 3 + 16 + 2 + 36]
        if len(body) != 54:
            raise ValueError("%s: the entry for (%d, %d) is cut short" % (path, head[0], head[1]))
        out["head"].append(head)
        out["T"].append(np.array(body[:16], dtype=np.float64).reshape(4, 4))
        out["inlier_num"].append(float(body[16]))
        out["inlier_ratio"].append(float(body[17]))
        out["info"].append(np.array(body[18:], dtype=np.float64).reshape(6, 6).T)
        at += 57
    return {"head": np.array(out["head"], dtype=np.int64).reshape(-1, 3),
            "T": np.array(out["T"], dtype=np.float64).reshape(-1, 4, 4),
            "inlier_num": np.array(out["inlier_num"], dtype=np.float64),
            "inlier_ratio": np.array(out["inlier_ratio"], dtype=np.float64),
            "info": np.array(out["info"], dtype=np.float64).reshape(-1, 6, 6)}


def format_log_entry(i, j, n_fragments, T, inlier_num, inlier_ratio, info):
    """One entry of writeLog.m's .log: the head, the 4x4 row by row (%.10f), `inlierNum\\tinlierRatio` and the 6x6 as
    fprintf prints a matrix, column by column."""
    T, info = np.asarray(T, dtype=np.float64).reshape(4, 4), np.asarray(info, dtype=np.float64).reshape(6, 6)
    s = "%d\t %d\t %d\t\n" % (i, j, n_fragments)
    s += "".join("%.10f\t%.10f\t%.10f\t%.10f\n" % tuple(row) for row in T)
    s += "%d\t%f\n" % (inlier_num, inlier_ratio)
    s += "".join("%.10f\t%.10f\t%.10f\t%.10f\t%.10f\t%.10f\n" % tuple(col) for col in info.T)
    return s


# ----------------------------------------------------------------------------------------------- the score
def dcm2quat(R):
    """mrEvaluateRegistrationMy.m's dcm2quat, as written there (the Aerospace Toolbox's sign convention)."""
    R = np.asarray(R, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        q0 = 0.5 * np.sqrt(1 + R[0, 0] + R[1, 1] + R[2, 2])
        return np.array([q0, -(R[2, 1] - R[1, 2]) / (4 * q0), -(R[0, 2] - R[2, 0]) / (4 * q0),
                         -(R[1, 0] - R[0, 1]) / (4 * q0)])


def transformation_error(trans, info):
    """mrComputeTransformationError: er = [t; -q(2:4)], p = er' info er / info(1, 1)."""
    trans, info = np.asarray(trans, dtype=np.float64), np.asarray(info, dtype=np.float64)
    er = np.concatenate([trans[:3, 3], -dcm2quat(trans[:3, :3])[1:4]])
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return float(er @ info @ er / info[0, 0])


def _nanmean(x):
    return float(np.mean(x)) if len(x) else float("nan")


def _ratio(a, b):
    return a / b if b else float("nan") if a == 0 else float("inf")


def evaluate_registration(result, gt_head, gt_T, gt_info, err2=ERR2):
    """mrEvaluateRegistrationMy.m.  result: dict of head (n, >= 2), T (n, 4, 4), inlier_num, inlier_ratio (as
    read_registration_log gives); gt_head (m, >= 2), gt_T (m, 4, 4), gt_info (m, 6, 6) in gt.log's order.  Only pairs
    with j - i > 1 count; a result pair absent from gt is a false positive; the last gt entry of a repeated pair wins
    (the mask's overwrite).  -> dict of recall, precision, inlier_num, inlier_ratio (means over the good pairs), good,
    bad, false_pos, gt_num, rs_num and the errors p of the matched pairs."""
    mask, gt_num = {}, 0
    for e, (i, j) in enumerate(np.asarray(gt_head)[:, :2]):
        if j - i > 1:
            mask[(int(i), int(j))] = e
            gt_num += 1
    rs_num = good = bad = false_pos = 0
    errors, inl_num, inl_ratio = [], [], []
    for e, (i, j) in enumerate(np.asarray(result["head"]).reshape(-1, 3)[:, :2]):
        if not j - i > 1:
            continue
        rs_num += 1
        g = mask.get((int(i), int(j)))
        if g is None:
            false_pos += 1
            continue
        p = transformation_error(np.linalg.inv(gt_T[g]) @ result["T"][e], gt_info[g])
        errors.append(p)
        if p <= err2:
            good += 1
            inl_num.append(float(result["inlier_num"][e]))
            inl_ratio.append(float(result["inlier_ratio"][e]))
        else:
            bad += 1
    return {"recall": _ratio(good, gt_num), "precision": _ratio(good, rs_num), "inlier_num": _nanmean(inl_num),
            "inlier_ratio": _nanmean(inl_ratio), "good": good, "bad": bad, "false_pos": false_pos, "gt_num": gt_num,
            "rs_num": rs_num, "errors": errors}


def _f(x):
    return "NaN" if np.isnan(x) else "%f" % x


def summary_line(scores):
    """evaluate.m's last line: the mean over scenes of recall, precision, round(inlierNum) and inlierRatio."""
    m = {k: float(np.mean([s[k] for s in scores])) for k in ("recall", "precision", "inlier_num", "inlier_ratio")}
    n = "NaN" if np.isnan(m["inlier_num"]) else "%d" % math.floor(m["inlier_num"] + 0.5)
    return ("Mean registration recall: %s precision: %s inlierNum: %s inlierRatio: %s"
            % (_f(m["recall"]), _f(m["precision"]), n, _f(m["inlier_ratio"])), m)


def scene_lines(scene, s):
    return ["--- " + scene,
            "recall : %.4g ( %d / %d )" % (s["recall"], s["good"], s["gt_num"]),
            "precision : %.4g ( %d / %d )" % (s["precision"], s["good"], s["rs_num"]),
            "inlier number : %.5g inlier ratio : %.5g" % (s["inlier_num"], s["inlier_ratio"])]


def score_logs(log_dir, scenes, eval_dir):
    """evaluate.m over existing logs: <log_dir>/<scene>.log for every scene (a missing log has no entries), scored
    against eval_dir(scene)/gt.log and gt.info -> ({scene: evaluate_registration dict}, summary line, means)."""
    out = {}
    for scene in scenes:
        head, T = read_gt_log4(os.path.join(eval_dir(scene), "gt.log"))
        ihead, info = read_gt_info(os.path.join(eval_dir(scene), "gt.info"))
        if len(ihead) != len(head) or np.any(ihead[:, :2] != head[:, :2]):
            raise ValueError("%s: gt.info does not list gt.log's pairs in gt.log's order" % eval_dir(scene))
        path = os.path.join(log_dir, "%s.log" % scene)
        res = read_registration_log(path) if os.path.isfile(path) else read_registration_log(os.devnull)
        out[scene] = evaluate_registration(res, head, T, info)
    line, means = summary_line(list(out.values()))
    return out, line, means


# ----------------------------------------------------------------------------------------------- one pair
def _rows(a, cols, what):
    t = torch.as_tensor(a) if not isinstance(a, torch.Tensor) else a
    t = t.detach().to(torch.float32)
    if t.dim() != 2 or (cols is not None and t.shape[1] != cols):
        raise ValueError("%s must be (n, %s)" % (what, cols if cols is not None else "D"))
    return t


def fast_global_registration(points1, features1, points2, features2, seed=0):
    """fast_global_registration.cpp's interface for one pair: points (n_f, 3) and features (n_f, D), numpy or CUDA
    tensors, at most 1024 rows and 512 dims -> T (4, 4) float64 with T[:3, :3] points2 + T[:3, 3] aligned to points1.
    Runs usip_desc_match_mutual_f64 and usip_fgr_f64 on the pair; with fewer than 10 tuple correspondences (or a
    degenerate scale) T is [I | mean1 - mean2], as the mex returns."""
    p1, p2 = _rows(points1, 3, "points1"), _rows(points2, 3, "points2")
    f1, f2 = _rows(features1, None, "features1"), _rows(features2, None, "features2")
    if len(f1) != len(p1) or len(f2) != len(p2) or f1.shape[1] != f2.shape[1]:
        raise ValueError("features must have one row per point and the same length on both sides")
    n1, n2, D = len(p1), len(p2), f1.shape[1]
    if not 1 <= D <= FGR_MAX_DIM or max(n1, n2) > FGR_MAX_ROWS:
        raise ValueError("at most %d rows and 1 to %d feature dims" % (FGR_MAX_ROWS, FGR_MAX_DIM))
    dev = next((t.device for t in (p1, p2, f1, f2) if t.is_cuda), torch.device("cuda"))
    L = max(n1, n2, 1)
    xyz = torch.zeros((2, L, 3), dtype=torch.float32, device=dev)
    desc = torch.zeros((2, L, D), dtype=torch.float32, device=dev)
    xyz[0, :n1], xyz[1, :n2] = p1.to(dev), p2.to(dev)
    desc[0, :n1], desc[1, :n2] = f1.to(dev), f2.to(dev)
    count = torch.tensor([n1, n2], dtype=torch.int32, device=dev)
    pairs = torch.tensor([[0, 1]], dtype=torch.int32, device=dev)
    m, n = ops.desc_match_mutual(desc, count, pairs, [L])
    out = ops.fgr(xyz, count, pairs, [L], m, n, INLIER_THRESHOLD, seed)
    T = np.eye(4)
    T[:3] = out["Rt"][0, 0].cpu().numpy()
    return T


# ----------------------------------------------------------------------------------------------- the evaluator
class IndoorRegistrationResult:
    """Per scene: pairs (P, 2) frame numbers, n_fragments, n_matches (P, nK), and per (pair, K, maxTrials) arrays Rt
    (.., 4, 4) (the identity without a model), n_inliers, inlier_ratio, aligned (ratioAligned(1), NaN where not
    computed), info (.., 6, 6) and accepted (the log's filter).  scores[(K, maxTrials)] = ({scene: evaluate dict},
    summary line, means).  solver "fgr": one trial entry, maxTrials None."""

    def __init__(self, dataset, keypoint_nums, max_trials, overlap_threshold, scenes, per_scene, gt, solver="ransac"):
        self.solver = solver
        self.dataset, self.keypoint_nums, self.max_trials = dataset, list(keypoint_nums), list(max_trials)
        self.overlap_threshold, self.scenes, self.per_scene = overlap_threshold, list(scenes), per_scene
        self.scores = {}
        for k, K in enumerate(self.keypoint_nums):
            for t, T in enumerate(self.max_trials):
                sc = {s: evaluate_registration(self.log_entries(s, k, t), *gt[s]) for s in self.scenes}
                line, means = summary_line(list(sc.values()))
                self.scores[(K, T)] = (sc, line, means)

    def log_entries(self, scene, k, t):
        """The entries of scene's log for the k-th K and t-th maxTrials, as read_registration_log returns them."""
        r = self.per_scene[scene]
        sel = np.nonzero(r["accepted"][:, k, t])[0]
        head = np.concatenate([r["pairs"][sel], np.full((len(sel), 1), r["n_fragments"])], axis=1)
        return {"head": head.reshape(-1, 3), "T": r["Rt"][sel, k, t], "inlier_num": r["n_inliers"][sel, k, t],
                "inlier_ratio": r["inlier_ratio"][sel, k, t], "info": r["info"][sel, k, t]}

    def lines(self):
        out = []
        for (K, T), (sc, line, _) in self.scores.items():
            head = "K=%d FGR %s" % (K, self.dataset) if self.solver == "fgr" else \
                "K=%d maxTrials=%d %s" % (K, T, self.dataset)
            for s in self.scenes:
                out += ["%s: %s" % (head, v) for v in scene_lines(s, sc[s])]
            out.append("%s: %s" % (head, line))
        return out

    def to_dict(self):
        nan = lambda v: None if isinstance(v, float) and not math.isfinite(v) else v
        runs = []
        for (K, T), (sc, _, means) in self.scores.items():
            runs.append({"K": K, "max_trials": T, "mean": {k: nan(v) for k, v in means.items()},
                         "scenes": {s: {k: nan(v) for k, v in d.items() if k != "errors"} for s, d in sc.items()},
                         "log_entries": {s: int(self.per_scene[s]["accepted"][:, self.keypoint_nums.index(K),
                                                                                 self.max_trials.index(T)].sum())
                                         for s in self.scenes}})
        return {"dataset": self.dataset, "solver": self.solver, "keypoint_nums": self.keypoint_nums,
                "max_trials": None if self.solver == "fgr" else self.max_trials,
                "overlap_threshold": self.overlap_threshold,
                "pairs": {s: int(len(self.per_scene[s]["pairs"])) for s in self.scenes}, "runs": runs}


def _scene_order(source):
    scenes = []
    for scene, _ in source.items:
        if scene not in scenes:
            scenes.append(scene)
    return scenes


class IndoorRegistration(Registration):
    """Registration of a Redwood or 3DMatch test set: wraps a RedwoodRepeatability / Match3DRepeatability (its source
    and detection) and eval_dir(scene), the folder of the scene's gt.log and gt.info.  describe, read_descriptor_tree
    and write_descriptor_tree are Registration's."""

    def __init__(self, evaluator, eval_dir):
        super().__init__(evaluator)
        self.eval_dir = eval_dir
        src = evaluator.source
        self.scenes = _scene_order(src)
        self.index = {src.key(i): i for i in range(len(src))}
        self.frames_of = {s: sorted(f for sc, f in src.items if sc == s) for s in self.scenes}
        self.gt = {}
        for s in self.scenes:
            head, T = read_gt_log4(os.path.join(eval_dir(s), "gt.log"))
            ihead, info = read_gt_info(os.path.join(eval_dir(s), "gt.info"))
            if len(ihead) != len(head) or np.any(ihead[:, :2] != head[:, :2]):
                raise ValueError("%s: gt.info does not list gt.log's pairs in gt.log's order" % eval_dir(s))
            self.gt[s] = (head, T, info)
        self.result = None

    @classmethod
    def redwood(cls, npy_root, gt_root, opt, **kw):
        """Redwood: fragments <npy_root>/<scene>/%d.npy, gt.log and gt.info in <gt_root>/original/<scene>-evaluation/."""
        ev = RedwoodRepeatability(npy_root, gt_root, opt, **kw)
        return cls(ev, lambda s: os.path.join(gt_root, "original", "%s-evaluation" % s))

    @classmethod
    def match3d(cls, root, opt, gt_root=None, **kw):
        """3DMatch: fragments <root>/<scene>/cloud_bin_<k>.npy, gt.log and gt.info in <gt_root>/<scene>-evaluation/
        (gt_root = root by default)."""
        ev = Match3DRepeatability(root, opt, gt_root=gt_root, **kw)
        return cls(ev, lambda s: os.path.join(gt_root or root, "%s-evaluation" % s))

    def scene_pairs(self, scene, pairs="all"):
        """(P, 2) frame numbers: every i < j by frame number ("all") or gt.log's pairs in its order ("gt")."""
        if pairs == "all":
            f = self.frames_of[scene]
            return np.array([(a, b) for x, a in enumerate(f) for b in f[x + 1:]], dtype=np.int64).reshape(-1, 2)
        if pairs == "gt":
            return self.gt[scene][0][:, :2].copy()
        raise ValueError("pairs must be 'all' or 'gt', got %r" % (pairs,))

    def _fragments(self, scene):
        """Columns 0:3 of every fragment of the scene, packed on the device -> (xyz (R, 3) f32, offsets, {frame: f})."""
        src = self.ev.source
        rows, where = [], {}
        for frame in self.frames_of[scene]:
            a = np.load(src.paths[self.index[(scene, frame)]], mmap_mode="r")
            where[frame] = len(rows)
            rows.append(np.ascontiguousarray(a[:, :3], dtype=np.float32))
        offsets = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
        return torch.from_numpy(np.concatenate(rows)).to(src.device), offsets, where

    def _register(self, scene, fp, ks, ts, seed, uniforms, solver="ransac"):
        """Matching, then RANSAC and the information matrix (solver "ransac") or mutual matching and FGR (solver "fgr",
        one trial entry), of one scene's pairs fp (P, 2 frames), a chunk of pairs per launch -> dict of numpy arrays."""
        dev = self.xyz.device
        L = min(self.xyz.shape[1], ks[-1])
        xyz, desc = self.xyz[:, :L].contiguous(), self.desc[:, :L].contiguous()
        count = torch.clamp(self.count, max=L).to(torch.int32).contiguous()
        per_pair = len(ks) * L * 8 if solver == "fgr" else len(ks) * 2 * MATCH_K * L * 8
        chunk = max(1, MATCH_BUFFER_BYTES // per_pair)
        keys = ("n_matches", "Rt", "n_inliers", "status", "info", "n_info")
        parts = {k: [] for k in keys}
        for c0 in range(0, len(fp), chunk):
            sel = fp[c0:c0 + chunk]
            pairs = torch.tensor([[self.index[(scene, int(a))], self.index[(scene, int(b))]] for a, b in sel],
                                 dtype=torch.int32, device=dev).reshape(-1, 2)
            if solver == "fgr":
                m, n = ops.desc_match_mutual(desc, count, pairs, ks)
                out = ops.fgr(xyz, count, pairs, ks, m, n, INLIER_THRESHOLD, seed)
                got = {"n_matches": n, "Rt": out["Rt"][:, :, None], "n_inliers": out["n_inliers"][:, :, None],
                       "status": out["status"][:, :, None], "info": out["info"][:, :, None],
                       "n_info": out["n_inliers"][:, :, None]}
                for k in keys:
                    parts[k].append(got[k].cpu().numpy())
                continue
            frames = torch.from_numpy(np.broadcast_to(np.eye(3, 4), (len(sel), 3, 3, 4)).copy()).to(dev)
            m, n = ops.desc_match(desc, count, pairs, ks, MATCH_K)
            out = ops.ransac_rt(xyz, count, pairs, frames, m, n, ts, INLIER_THRESHOLD, seed, uniforms)
            info, n_info = ops.ransac_info(xyz, count, pairs, frames, m, n, ts, out["best_trial"], out["status"],
                                           INLIER_THRESHOLD, seed, uniforms)
            got = {"n_matches": n, "Rt": out["Rt"], "n_inliers": out["n_inliers"], "status": out["status"],
                   "info": info, "n_info": n_info}
            for k in keys:
                parts[k].append(got[k].cpu().numpy())
        return {k: np.concatenate(v) for k, v in parts.items()}

    def score(self, keypoint_nums=DEFAULT_KEYPOINT_NUMS, max_trials=None,
              overlap_threshold=DEFAULT_OVERLAP_THRESHOLD, pairs="all", seed=0, uniforms=None, solver="ransac"):
        """Registers every pair of every scene for every K and maxTrials (DEFAULT_MAX_TRIALS when None), runs the overlap
        test where it can decide the log, filters and scores -> IndoorRegistrationResult (also kept as self.result).
        overlap_threshold None skips the overlap test (the lite variant's ratioAligned = 0.8).  solver "fgr" registers
        with Fast Global Registration: no maxTrials and no uniforms, one trial entry."""
        if solver not in SOLVERS:
            raise ValueError("solver must be 'ransac' or 'fgr', got %r" % (solver,))
        ks = check_sweep(keypoint_nums, 1.0)
        if solver == "fgr":
            if max_trials is not None or uniforms is not None:
                raise ValueError("solver 'fgr' takes no max_trials and no uniforms")
            ts = [None]
        else:
            ts = check_trials(DEFAULT_MAX_TRIALS if max_trials is None else max_trials, INLIER_THRESHOLD)
        _check_keypoint_limit(ks)
        if self.xyz is None:
            raise RuntimeError("describe() or read_descriptor_tree() first")
        if pairs not in ("all", "gt"):
            raise ValueError("pairs must be 'all' or 'gt', got %r" % (pairs,))
        if uniforms is not None:
            uniforms = torch.as_tensor(np.ascontiguousarray(uniforms, dtype=np.float64)).to(self.xyz.device)
        per_scene = {}
        for scene in self.scenes:
            fp = self.scene_pairs(scene, pairs)
            r = self._register(scene, fp, ks, ts, seed, uniforms, solver) if len(fp) else None
            per_scene[scene] = self._finish(scene, fp, r, len(ks), len(ts), overlap_threshold)
        self.result = IndoorRegistrationResult(self.dataset, ks, ts, overlap_threshold, self.scenes, per_scene,
                                               self.gt, solver)
        return self.result

    def _finish(self, scene, fp, r, nK, nT, overlap_threshold):
        P = len(fp)
        if r is None:
            r = {"n_matches": np.zeros((0, nK), np.int32), "Rt": np.zeros((0, nK, nT, 3, 4)),
                 "n_inliers": np.zeros((0, nK, nT), np.int32), "status": np.zeros((0, nK, nT), np.int32),
                 "info": np.zeros((0, nK, nT, 6, 6)), "n_info": np.zeros((0, nK, nT), np.int32)}
        model = r["status"] == 0
        Rt = np.broadcast_to(np.eye(4), (P, nK, nT, 4, 4)).copy()
        Rt[model, :3] = r["Rt"][model]
        n_inl = np.where(model, r["n_inliers"], 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio = n_inl / r["n_matches"][:, :, None].astype(np.float64)      # 0 / 0 = NaN never passes
        candidate = ratio > INLIER_RATIO_THRESHOLD
        aligned = np.full((P, nK, nT), np.nan)
        if overlap_threshold is None:
            aligned[candidate] = 0.8
        elif candidate.any():
            aligned[candidate] = self._overlap(scene, fp, Rt, candidate)
        accepted = candidate & (aligned > (0.23 if overlap_threshold is None else overlap_threshold))
        return {"pairs": fp, "n_fragments": len(self.frames_of[scene]), "n_matches": r["n_matches"], "Rt": Rt,
                "n_inliers": n_inl, "inlier_ratio": ratio, "aligned": aligned, "info": r["info"],
                "n_info": r["n_info"], "status": r["status"], "accepted": accepted}

    def _overlap(self, scene, fp, Rt, candidate):
        """ratioAligned(1) of the candidate (pair, K, maxTrials) entries, each distinct (pair, Rt) run once."""
        xyz, offsets, where = self._fragments(scene)
        idx = np.argwhere(candidate)
        jobs, maps, slot, of = [], [], {}, []
        for p, k, t in idx:
            key = (int(p), Rt[p, k, t, :3].tobytes())
            if key not in slot:
                slot[key] = len(jobs)
                jobs.append((where[int(fp[p, 0])], where[int(fp[p, 1])]))
                maps.append(Rt[p, k, t, :3])
            of.append(slot[key])
        hits = ops.fragment_overlap(xyz, offsets, np.array(jobs, dtype=np.int32),
                                    torch.from_numpy(np.ascontiguousarray(maps)).to(xyz.device), OVERLAP_RADIUS)
        hits = hits.cpu().numpy()
        rows = np.diff(offsets)
        return np.array([hits[s] / rows[jobs[s][0]] for s in of], dtype=np.float64)

    def write_registration_logs(self, out_dir, K, max_trials=None):
        """writeLog.m for the last score's K and maxTrials (None for an FGR score): <out_dir>/<scene>.log, one entry per
        accepted pair."""
        if self.result is None:
            raise RuntimeError("score() first")
        res = self.result
        if (res.solver == "fgr") != (max_trials is None):
            raise ValueError("max_trials is None exactly for an FGR score")
        k = res.keypoint_nums.index(int(K))
        t = 0 if max_trials is None else res.max_trials.index(int(max_trials))
        os.makedirs(out_dir, exist_ok=True)
        for scene in self.scenes:
            e = res.log_entries(scene, k, t)
            with open(os.path.join(out_dir, "%s.log" % scene), "w") as f:
                for x in range(len(e["head"])):
                    f.write(format_log_entry(*e["head"][x], e["T"][x], e["inlier_num"][x], e["inlier_ratio"][x],
                                             e["info"][x]))

    def score_logs(self, log_dir):
        """evaluate.m on existing logs for this test set's scenes."""
        return score_logs(log_dir, self.scenes, self.eval_dir)


# ----------------------------------------------------------------------------------------------- command line
def _scene_eval_dir(dataset, root, gt_root):
    if dataset == "redwood":
        return lambda s: os.path.join(gt_root, "original", "%s-evaluation" % s)
    return lambda s: os.path.join(gt_root or root, "%s-evaluation" % s)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m usip_b200.evaluation.indoor_registration",
                                 description="The indoor geometric-registration benchmark (runFragmentRegistration.m, "
                                             "writeLog.m, evaluate.m) on the Redwood or 3DMatch test set.")
    ap.add_argument("dataset", choices=("redwood", "3dmatch"))
    ap.add_argument("--root", help="redwood: numpy_gt_normal/; 3dmatch: 3DMatch_eval_npy/")
    ap.add_argument("--gt-root", help="redwood: the folder of original/<scene>-evaluation/{gt.log,gt.info}; 3dmatch: "
                                      "the folder of <scene>-evaluation/ (default --root)")
    ap.add_argument("--detector", help="detector state dict (the reference's *_net_detector.pth); --method tsf only")
    ap.add_argument("--descriptor", help="descriptor state dict (the reference's *_net_descriptor.pth)")
    ap.add_argument("--descriptor-tree", metavar="DIR", help="score an existing result tree <DIR>/<scene>/<frame>.bin")
    ap.add_argument("--feature-dim", type=int, default=128, help="descriptor length of --descriptor-tree")
    ap.add_argument("--pairs", choices=("all", "gt"), default="all")
    ap.add_argument("--keypoint-nums", type=int, nargs="+", default=list(DEFAULT_KEYPOINT_NUMS))
    ap.add_argument("--solver", choices=SOLVERS, default="ransac",
                    help="ransac (register2Fragments.m) or fgr (register2FragmentsFGR.m, Fast Global Registration)")
    ap.add_argument("--max-trials", type=int, nargs="+", help="RANSAC trial budgets (default %s)"
                    % " ".join(str(t) for t in DEFAULT_MAX_TRIALS))
    ap.add_argument("--overlap-threshold", default=str(DEFAULT_OVERLAP_THRESHOLD),
                    help="writeLog.m's ratioAligned(1) threshold, or 'none' to skip the overlap test")
    ap.add_argument("--write-logs", metavar="DIR", help="write <DIR>/<scene>.log for the largest K and maxTrials")
    ap.add_argument("--score-logs", metavar="DIR", help="only score existing logs <DIR>/<scene>.log")
    ap.add_argument("--nms-radius", type=float, default=0.0)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--input-pc-num", type=int, default=10240)
    ap.add_argument("--node-num", type=int, default=512)
    ap.add_argument("--json", metavar="OUT", help="write the summary as JSON")
    add_method_args(ap)
    a = ap.parse_args(argv)
    if a.dataset == "redwood" and not a.gt_root:
        ap.error("redwood needs --gt-root")
    if a.solver == "fgr" and a.max_trials is not None:
        ap.error("--max-trials applies to --solver ransac only")
    if a.solver == "ransac" and a.max_trials is None:
        a.max_trials = list(DEFAULT_MAX_TRIALS)
    if a.score_logs:
        scenes = [s for s, _ in REDWOOD_SCENES] if a.dataset == "redwood" else list(MATCH3D_SCENES)
        sc, line, means = score_logs(a.score_logs, scenes, _scene_eval_dir(a.dataset, a.root, a.gt_root))
        for s in scenes:
            print("\n".join(scene_lines(s, sc[s])))
        print("===\n" + line)
        if a.json:
            with open(a.json, "w") as f:
                json.dump({"scenes": {s: {k: v for k, v in d.items() if k != "errors"} for s, d in sc.items()},
                           "mean": means}, f, indent=1)
        return sc
    thr = None if a.overlap_threshold.lower() == "none" else float(a.overlap_threshold)
    ks = check_sweep(a.keypoint_nums, 1.0)
    _check_keypoint_limit(ks)
    if a.solver == "ransac":
        check_trials(a.max_trials, INLIER_THRESHOLD)
    if not a.root:
        ap.error("give --root")
    hc = detector_from_args(a, ap)
    if not a.descriptor_tree and not ((a.detector or hc is not None) and a.descriptor):
        ap.error("give --detector (--method tsf) and --descriptor, or --descriptor-tree")
    if hc is not None and a.nms_radius >= 0.01:
        ap.error("--nms-radius applies to --method tsf only")
    opt = descriptor_opt(a.dataset, batch_size=a.batch_size, input_pc_num=a.input_pc_num, node_num=a.node_num)
    kw = {"seed": a.seed, "batch_size": a.batch_size}
    if a.dataset == "redwood":
        ev = IndoorRegistration.redwood(a.root, a.gt_root, opt, **kw)
    else:
        ev = IndoorRegistration.match3d(a.root, opt, gt_root=a.gt_root, **kw)
    if a.descriptor_tree:
        ev.read_descriptor_tree(a.descriptor_tree, a.feature_dim)
    else:
        from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
        from usip_b200.models.keypoint_detector import ModelDetector
        from .registration import load_descriptor_checkpoint
        from .repeatability import load_detector_checkpoint
        det = ModelDetector(opt) if hc is None else hc
        des = ModelDescriptorIndoor(opt)
        if hc is None:
            load_detector_checkpoint(det, a.detector)
        load_descriptor_checkpoint(des, a.descriptor)
        ev.describe(det, des, a.nms_radius, L=ks[-1])
    extra = () if a.solver == "ransac" else (None, a.solver)            # (uniforms, solver)
    res = ev.score(ks, a.max_trials, thr, a.pairs, a.seed, *extra)
    print("\n".join(res.lines()))
    if hc is not None and not a.descriptor_tree:
        print(hc.count_summary())
    if a.write_logs:
        ev.write_registration_logs(a.write_logs, ks[-1], a.max_trials[-1] if a.solver == "ransac" else None)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res.to_dict(), f, indent=1)
    return res


if __name__ == "__main__":
    main()
