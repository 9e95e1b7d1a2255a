"""Numpy restatement of the indoor registration benchmark's new pieces, cited against the reference's MATLAB
(evaluation/matlab/eval_indoor/3dmatch/):
  overlap          register2Fragments.m:126-137 (ratioAligned(1)) in usip_fragment_overlap_f32's rule: b' = fp64 map
                   rounded once to fp32, hit iff the fp32 d2 <= the largest t with sqrtf(t) < radius; scipy's cKDTree
                   (fp64) only proposes candidates, within a radius wide enough for every fp32 hit
  information      register2Fragments.m:77-88 on top of tests/reg_ref.py's RANSAC
  files and score  mrLoadInfo.m, mrLoadLogMy.m, mrEvaluateRegistrationMy.m (external/ElasticReconstruction/)
"""
import numpy as np
from scipy.spatial import cKDTree

from tests import reg_ref as rr


# ----------------------------------------------------------------------------------------------- overlap
def tlim(radius):
    r = np.float32(radius)
    t = np.float32(r * r)
    while t > 0 and not np.sqrt(t) < r:
        t = np.nextafter(t, np.float32(0))
    while True:
        up = np.nextafter(t, np.float32(np.inf))
        if not np.isfinite(up) or not np.sqrt(up) < r:
            return t
        t = up


def map_b(Rt, b):
    """((r0 x + r1 y) + r2 z) + t in fp64, rounded once to fp32."""
    b = np.asarray(b, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        out = [((Rt[r, 0] * b[:, 0] + Rt[r, 1] * b[:, 1]) + Rt[r, 2] * b[:, 2]) + Rt[r, 3] for r in range(3)]
        return np.stack(out, 1).astype(np.float32)


def overlap_ref(a, b, Rt, radius=0.2):
    """Number of rows of a (n, 3) f32 with some mapped row of b within radius, by the kernel's rule."""
    a = np.asarray(a, np.float32)
    bp = map_b(np.asarray(Rt, np.float64), b)
    fa = np.all(np.isfinite(a), 1)
    fb = np.all(np.isfinite(bp), 1)
    bp = bp[fb]
    if len(bp) == 0 or not fa.any():
        return 0
    t = tlim(radius)
    tree = cKDTree(bp.astype(np.float64))
    cand = tree.query_ball_point(a[fa].astype(np.float64), float(radius) * (1 + 1e-5) + 1e-30)
    lens = np.array([len(c) for c in cand])
    if lens.sum() == 0:
        return 0
    q = np.repeat(a[fa], lens, axis=0)
    with np.errstate(over="ignore", invalid="ignore"):
        d = q - bp[np.concatenate([np.asarray(c, np.int64) for c in cand])]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    owner = np.repeat(np.arange(len(lens)), lens)
    return int(len(np.unique(owner[d2 <= t])))


# ----------------------------------------------------------------------------------------------- information matrix
def info_of(points):
    """Sum over the points, in order, of A^T A, A = [I3 | [[0, 2z, -2y], [-2z, 0, 2x], [2y, -2x, 0]]]."""
    M = np.zeros((6, 6))
    for x, y, z in np.asarray(points, np.float64).reshape(-1, 3):
        A = np.array([[1, 0, 0, 0, 2 * z, -2 * y], [0, 1, 0, -2 * z, 0, 2 * x], [0, 0, 1, 2 * y, -2 * x, 0]])
        for r in range(6):
            for c in range(6):
                M[r, c] += (A[0, r] * A[0, c] + A[1, r] * A[1, c]) + A[2, r] * A[2, c]
    return M


def info_ref(x1, x2, trials, thr, uniforms):
    """Per trial budget (info, n_info) of ransac_ref's best model: its inliers' anchors x1, in match order."""
    res = rr.ransac_ref(x1, x2, trials, thr, uniforms)
    n = len(x1)
    out = []
    for r in res:
        if r["status"] != 0:
            out.append((np.zeros((6, 6)), 0))
            continue
        if n == 3:
            mask = np.ones(3, bool)
        else:
            counts = rr._LazyCounts(x1, x2, uniforms, thr)
            mask = rr.inliers(counts.hypotheses(r["best_trial"], r["best_trial"] + 1), x1, x2, thr)[0]
        out.append((info_of(x1[mask]), int(mask.sum())))
    return res, out


# ----------------------------------------------------------------------------------------------- files and score
def load_info(path):
    """mrLoadInfo.m -> list of (info (3,), mat (6, 6))."""
    tok = open(path).read().split()
    out, at = [], 0
    while at + 3 <= len(tok):
        x = [int(v) for v in tok[at:at + 3]]
        m = np.array(tok[at + 3:at + 39], np.float64).reshape(6, 6, order="F")     # fscanf [6 6]
        out.append((x, m.T))
        at += 39
    return out


def load_log_my(path):
    """mrLoadLogMy.m -> list of dicts info, trans, inlierNum, inlierRatio, information."""
    tok = open(path).read().split()
    out, at = [], 0
    while at + 3 <= len(tok):
        x = [int(v) for v in tok[at:at + 3]]
        m = np.array(tok[at + 3:at + 19], np.float64).reshape(4, 4, order="F")
        num, ratio = int(tok[at + 19]), float(tok[at + 20])
        inf = np.array(tok[at + 21:at + 57], np.float64).reshape(6, 6, order="F")
        out.append(dict(info=x, trans=m.T, inlierNum=num, inlierRatio=ratio, information=inf))
        at += 57
    return out


def evaluate_my(result, gt, gt_info, err2=0.04):
    """mrEvaluateRegistrationMy.m with its mask: result and gt lists of dicts with info and trans; gt_info of mat."""
    num = gt[0]["info"][2]
    mask = {}
    gt_num = 0
    for i, g in enumerate(gt):
        if g["info"][1] - g["info"][0] > 1:
            mask[g["info"][0] + g["info"][1] * num] = i + 1
            gt_num += 1
    rs_num = good = 0
    inl, rat = [], []
    for r in result:
        if r["info"][1] - r["info"][0] > 1:
            rs_num += 1
            idx = mask.get(r["info"][0] + r["info"][1] * num, 0)
            if idx:
                trans = np.linalg.inv(gt[idx - 1]["trans"]) @ r["trans"]
                D = trans[:3, :3]
                with np.errstate(invalid="ignore", divide="ignore"):
                    q1 = 0.5 * np.sqrt(1 + D[0, 0] + D[1, 1] + D[2, 2])
                    q = [-(D[2, 1] - D[1, 2]) / (4 * q1), -(D[0, 2] - D[2, 0]) / (4 * q1), -(D[1, 0] - D[0, 1]) / (4 * q1)]
                    er = np.concatenate([trans[:3, 3], -np.array(q)])
                    info = gt_info[idx - 1]
                    p = er @ info @ er / info[0, 0]
                if p <= err2:
                    good += 1
                    inl.append(r["inlierNum"]); rat.append(r["inlierRatio"])
    nan = float("nan")
    return dict(recall=good / gt_num if gt_num else nan, precision=good / rs_num if rs_num else nan,
                inlier_num=np.mean(inl) if inl else nan, inlier_ratio=np.mean(rat) if rat else nan, good=good,
                gt_num=gt_num, rs_num=rs_num)
