"""Float64 restatement of evaluate_kitti.m / evaluate_oxford.m's matching and of ransacfitRt.m -> ransac.m ->
estimateRigidTransform.m in usip_desc_match_f64 / usip_ransac_rt_f64's operation order, elementwise (no `@` and no
np.sum, whose summation orders differ), vectorised across hypotheses.  The reference is MATLAB and cannot run here, so
this file cites it instead:
  matching       evaluate_kitti.m:50-53 (pdist2 'smallest' 1), evaluate_oxford.m:58-66 (k = 5 both ways, union 'rows')
  sampling       ransac.m:170 randsample(npts, 3): replaced by the header's index rule on uploaded uniforms
  fit            estimateRigidTransform.m:60-93, quat2rot.m, crossTimesMatrix.m
  loop           ransac.m:162-236 (bestscore, N, trialcount, the maxTrials break)
  refit          ransacfitRt.m:78-84
"""
import numpy as np

from tests.rep_ref import apply_map

EPS = np.finfo(np.float64).eps
PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
SWEEPS = 8


# ----------------------------------------------------------------------------------------------- matching
def desc_d2(a, b):
    """(na, D), (nb, D) f32 -> (na, nb) f64: sum_c (a_c - b_c)^2, c ascending."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    acc = np.zeros((len(a), len(b)))
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(a.shape[1]):
            d = a[:, None, c] - b[None, :, c]
            acc = acc + d * d
    return acc


def match_ref(da, dp, k):
    """Matches of anchor rows da against positive rows dp -> (n, 2) int (anchor row, positive row)."""
    na, npos = len(da), len(dp)
    if na == 0 or npos == 0:
        return np.zeros((0, 2), np.int64)
    d2 = desc_d2(da, dp)
    d2 = np.where(np.isnan(d2), np.inf, d2)                      # a non-finite descriptor orders as +inf, by index
    if k == 1:
        return np.stack([np.arange(na), np.argmin(d2, axis=1)], 1)
    pos = np.argsort(d2, axis=1, kind="stable")[:, :k]           # (d^2, index) order
    anc = np.argsort(d2.T, axis=1, kind="stable")[:, :k]
    rows = {(i, int(j)) for i in range(na) for j in pos[i]} | {(int(i), j) for j in range(npos) for i in anc[j]}
    return np.array(sorted(rows), dtype=np.int64).reshape(-1, 2)


# ----------------------------------------------------------------------------------------------- sampling
def pick3(u, n):
    """The header's index rule: u (H, 3) in [0, 1), n >= 3 -> (H, 3) distinct indices below n."""
    u = np.asarray(u, np.float64).reshape(-1, 3)
    i0 = np.maximum(np.minimum(np.floor(u[:, 0] * n).astype(np.int64), n - 1), 0)
    i1 = np.maximum(np.minimum(np.floor(u[:, 1] * (n - 1)).astype(np.int64), n - 2), 0)
    i2 = np.maximum(np.minimum(np.floor(u[:, 2] * (n - 2)).astype(np.int64), n - 3), 0)
    i1 = i1 + (i1 >= i0)
    lo, hi = np.minimum(i0, i1), np.maximum(i0, i1)
    i2 = i2 + (i2 >= lo)
    i2 = i2 + (i2 >= hi)
    return np.stack([i0, i1, i2], 1)


# ----------------------------------------------------------------------------------------------- Horn's fit
def ata(x, y):
    """A^T A of Horn's A for centred correspondences x, y (..., 3) -> (..., 4, 4)."""
    u = [y[..., c] - x[..., c] for c in range(3)]
    v = [x[..., c] - y[..., c] for c in range(3)]
    w = [y[..., c] + x[..., c] for c in range(3)]
    z = np.zeros_like(u[0])
    A = [[z, u[0], u[1], u[2]], [v[0], z, -w[2], w[1]], [v[1], w[2], z, -w[0]], [v[2], -w[1], w[0], z]]
    M = np.empty(x.shape[:-1] + (4, 4))
    for r in range(4):
        for c in range(4):
            M[..., r, c] = ((A[0][r] * A[0][c] + A[1][r] * A[1][c]) + A[2][r] * A[2][c]) + A[3][r] * A[3][c]
    return M


def horn_finish(B, xbar, ybar):
    """B (H, 4, 4), centroids (H, 3) -> Rt (H, 3, 4): cyclic Jacobi, smallest eigenvector, quat2rot, t."""
    a = np.array(B, dtype=np.float64, copy=True)
    H = len(a)
    V = np.broadcast_to(np.eye(4), (H, 4, 4)).copy()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for _ in range(SWEEPS):
            for p, q in PAIRS:
                apq = a[:, p, q].copy()
                on = apq != 0.0
                theta = (a[:, q, q] - a[:, p, p]) / (2.0 * apq)
                t = np.where(theta >= 0.0, 1.0, -1.0) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                for r in range(4):
                    if r in (p, q):
                        continue
                    arp, arq = a[:, r, p].copy(), a[:, r, q].copy()
                    nP = np.where(on, c * arp - s * arq, arp)
                    nQ = np.where(on, s * arp + c * arq, arq)
                    a[:, r, p] = nP; a[:, p, r] = nP; a[:, r, q] = nQ; a[:, q, r] = nQ
                app, aqq = a[:, p, p].copy(), a[:, q, q].copy()
                a[:, p, p] = np.where(on, app - t * apq, app)
                a[:, q, q] = np.where(on, aqq + t * apq, aqq)
                a[:, p, q] = np.where(on, 0.0, apq); a[:, q, p] = a[:, p, q]
                for r in range(4):
                    vp, vq = V[:, r, p].copy(), V[:, r, q].copy()
                    V[:, r, p] = np.where(on, c * vp - s * vq, vp)
                    V[:, r, q] = np.where(on, s * vp + c * vq, vq)
    m = np.zeros(H, np.int64)
    amin = a[:, 0, 0].copy()
    for r in range(1, 4):
        lt = a[:, r, r] < amin
        amin = np.where(lt, a[:, r, r], amin)
        m = np.where(lt, r, m)
    q0, q1, q2, q3 = (V[np.arange(H), r, m] for r in range(4))
    s00, s11, s22, s33 = q0 * q0, q1 * q1, q2 * q2, q3 * q3
    R = np.empty((H, 3, 3))
    R[:, 0, 0] = ((s00 + s11) - s22) - s33
    R[:, 0, 1] = 2.0 * (q1 * q2 - q0 * q3)
    R[:, 0, 2] = 2.0 * (q1 * q3 + q0 * q2)
    R[:, 1, 0] = 2.0 * (q1 * q2 + q0 * q3)
    R[:, 1, 1] = ((s00 - s11) + s22) - s33
    R[:, 1, 2] = 2.0 * (q2 * q3 - q0 * q1)
    R[:, 2, 0] = 2.0 * (q1 * q3 - q0 * q2)
    R[:, 2, 1] = 2.0 * (q2 * q3 + q0 * q1)
    R[:, 2, 2] = ((s00 - s11) - s22) + s33
    Rt = np.empty((H, 3, 4))
    Rt[:, :, :3] = R
    for r in range(3):
        Rt[:, r, 3] = xbar[:, r] - ((R[:, r, 0] * ybar[:, 0] + R[:, r, 1] * ybar[:, 1]) + R[:, r, 2] * ybar[:, 2])
    return Rt


def _seqsum(a):
    """((0 + a_0) + a_1) + ... along axis 1 (np.add.accumulate is sequential)."""
    z = np.zeros((a.shape[0], 1) + a.shape[2:])
    return np.add.accumulate(np.concatenate([z, a], axis=1), axis=1)[:, -1]


def fit(x, y):
    """estimateRigidTransform.m for H point sets at once: x, y (H, n, 3) (anchor, positive) -> Rt (H, 3, 4)."""
    n = x.shape[1]
    xb, yb = _seqsum(x) / n, _seqsum(y) / n
    B = _seqsum(ata(x - xb[:, None], y - yb[:, None]))
    return horn_finish(B, xb, yb)


def inliers(Rt, x1, x2, thr):
    """(H, n) bool: sqrt(|x1 - (R x2 + t)|^2) < thr, in the kernel's order."""
    e = [((Rt[:, r, None, 0] * x2[None, :, 0] + Rt[:, r, None, 1] * x2[None, :, 1]) + Rt[:, r, None, 2] * x2[None, :, 2])
         + Rt[:, r, None, 3] for r in range(3)]
    d = [x1[None, :, r] - e[r] for r in range(3)]
    return np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) < thr


# ----------------------------------------------------------------------------------------------- the loop
def ransac_loop(counts, npts, trials):
    """ransac.m's sequential update over per-trial inlier counts (an indexable, evaluated in trial order) -> one
    (trialcount, best_trial, n_inliers) per trial budget."""
    best, bestscore, N, tc, out = -1, 0, 1.0, 0, []
    log_1mp = np.log(1.0 - 0.99)
    while len(out) < len(trials):
        n = int(counts[tc])
        if n >= bestscore:
            best, bestscore = tc, n
            frac = n / npts
            pno = min(max(EPS, 1.0 - (frac * frac) * frac), 1.0 - EPS)
            N = max(log_1mp / np.log(pno), 10.0)
        tc += 1
        stop = not (N > tc)
        while len(out) < len(trials) and (stop or tc > trials[len(out)]):
            out.append((tc, best, bestscore))
    return out


class _LazyCounts:
    """Inlier counts of the hypotheses of trials 0, 1, ..., computed a chunk at a time on first use."""

    def __init__(self, x1, x2, uniforms, thr, chunk=1024):
        self.x1, self.x2, self.u, self.thr, self.chunk = x1, x2, uniforms, thr, chunk
        self.counts = np.zeros(0, np.int64)

    def hypotheses(self, j0, j1):
        idx = pick3(self.u[j0:j1], len(self.x1))
        return fit(self.x1[idx], self.x2[idx])

    def __getitem__(self, j):
        while j >= len(self.counts):
            j0 = len(self.counts)
            Rt = self.hypotheses(j0, j0 + self.chunk)
            self.counts = np.concatenate([self.counts, inliers(Rt, self.x1, self.x2, self.thr).sum(1)])
        return self.counts[j]


def ransac_ref(x1, x2, trials, thr, uniforms):
    """ransacfitRt.m on correspondences x1 (anchor), x2 (positive) (n, 3) f64 -> per trial budget a dict of Rt, n_inliers,
    trialcount, best_trial, status (as usip_ransac_rt_f64)."""
    n = len(x1)
    if n < 3:
        return [dict(Rt=np.zeros((3, 4)), n_inliers=0, trialcount=0, best_trial=-1, status=1) for _ in trials]
    if n == 3:
        Rt = fit(x1[None], x2[None])[0]
        return [dict(Rt=Rt, n_inliers=3, trialcount=0, best_trial=-1, status=0) for _ in trials]
    counts = _LazyCounts(x1, x2, uniforms, thr)
    out = []
    for tc, best, nin in ransac_loop(counts, n, trials):
        if nin < 3:
            out.append(dict(Rt=np.zeros((3, 4)), n_inliers=nin, trialcount=tc, best_trial=best, status=2))
            continue
        mask = inliers(counts.hypotheses(best, best + 1), x1, x2, thr)[0]
        Rt = fit(x1[mask][None], x2[mask][None])[0]
        out.append(dict(Rt=Rt, n_inliers=nin, trialcount=tc, best_trial=best, status=0))
    return out


def register_pair_ref(anc, pos, F_a, F_p, K, k, trials, thr, uniforms):
    """One pair and K from the scans' rows [xyz (camera frame) | descriptor] (n, 3 + D) f32 in selection order ->
    (matches (n, 2), per-budget results of ransac_ref)."""
    a, p = anc[:K], pos[:K]
    m = match_ref(a[:, 3:], p[:, 3:], k)
    x1 = apply_map(F_a, a[:, :3])[m[:, 0]]
    x2 = apply_map(F_p, p[:, :3])[m[:, 1]]
    return m, ransac_ref(x1, x2, trials, thr, uniforms)
