"""Float64 restatement of usip_desc_match_mutual_f64 and usip_fgr_f64 (csrc/fgr.cu) in the header's operation order:
elementwise numpy (no `@`, no np.sum) for the vector steps and Python floats for the 6x6 solve, so that every tuple,
every one of the 27 sums and every Cholesky pivot is the kernel's.  The one step that is not bit-exact is sin / cos
(libm here, CUDA's on the device).  It cites the reference, whose FGR library sources are absent:
  mutual matches   AdvancedMatching's initial matching and cross-check, with tests/reg_ref.py's d^2, tie and NaN rule
  normalise        NormalizePoints (GlobalScale = max centred norm, relative scale)
  tuples           AdvancedMatching's tuple test: 100 * ncorr trials, 0.95f, at most 10000 tuples, Philox for rand()
  GNC              OptimizePairwise(true, 640): par /= 1.4 every 4 iterations down to 0.05, Gauss-Newton by LLT
  output           GetOutputTrans; the inlier count and information matrix under the result (usip_ransac_info_f64's)
"""
import math

import numpy as np

from tests import indoor_reg_ref as ir
from tests import philox_ref as ph
from tests import reg_ref as rr

THREADS, WARPS = 256, 8
TAG = 0x46475254                          # "FGRT"
ITERATIONS = 640
TRIALS_PER_MATCH = 100
TUPLE_CAP = 10000
MIN_CORR = 10
DIV, STOP = 1.4, 0.05
SIM = float(np.float32(0.95))
DBL_MAX = np.finfo(np.float64).max
UPPER = [(a, b) for a in range(6) for b in range(a, 6)]


# ----------------------------------------------------------------------------------------------- matching
def mutual_ref(da, dp):
    """(i, j) with j the nearest of dp to da[i] and i the nearest of da to dp[j], ascending i -> (n, 2) int64."""
    if len(da) == 0 or len(dp) == 0:
        return np.zeros((0, 2), np.int64)
    d2 = rr.desc_d2(da, dp)
    d2 = np.where(np.isnan(d2), np.inf, d2)
    fwd, back = np.argmin(d2, axis=1), np.argmin(d2, axis=0)         # first minimum: the lower index wins a tie
    i = np.flatnonzero(back[fwd] == np.arange(len(da)))
    return np.stack([i, fwd[i]], 1).astype(np.int64)


# ----------------------------------------------------------------------------------------------- steps 1 and 2
def seq_mean(x):
    """(((0 + x_0) + x_1) + ...) / max(n, 1) per column of x (n, 3)."""
    x = np.asarray(x, np.float64).reshape(-1, 3)
    s = np.add.accumulate(np.concatenate([np.zeros((1, 3)), x]), axis=0)[-1]
    return s / max(len(x), 1)


def norm3(d):
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def normalise(f1, f2):
    """-> (mean1, mean2, scale, degenerate)."""
    f1, f2 = np.asarray(f1, np.float64).reshape(-1, 3), np.asarray(f2, np.float64).reshape(-1, 3)
    m1, m2 = seq_mean(f1), seq_mean(f2)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.concatenate([norm3(f1 - m1), norm3(f2 - m2)])
    finite = bool(np.all(r <= DBL_MAX))
    scale = float(r.max()) if finite and len(r) else (0.0 if finite else float("nan"))
    return m1, m2, scale, not (finite and scale > 0.0)


def tuple_indices(seed, n, T):
    """The three indices of trials 0..T-1 -> (T, 3) int64."""
    seed = int(seed) & (2 ** 64 - 1)
    w = ph.philox4x32_10(np.arange(T, dtype=np.uint64), 0, TAG, 0, seed & 0xFFFFFFFF, seed >> 32)
    return np.stack([np.minimum(np.floor((x.astype(np.float64) * 2.0 ** -32) * n).astype(np.int64), n - 1)
                     for x in w[:3]], 1)


def accept(li, lj):
    """The strict 0.95f rule on edge lengths (..., 3) -> (...,) bool."""
    return np.all((li * SIM < lj) & (lj < li / SIM), axis=-1)


def tuples(p, q, seed):
    """p, q (n, 3) normalised points of the matches -> (n_tuples, multiplicity (n,) int64, kept trial indices)."""
    n = len(p)
    if n < 3:
        return 0, np.zeros(n, np.int64), np.zeros(0, np.int64)
    idx = tuple_indices(seed, n, TRIALS_PER_MATCH * n)
    nxt = idx[:, [1, 2, 0]]
    li, lj = norm3(p[idx] - p[nxt]), norm3(q[idx] - q[nxt])
    kept = np.flatnonzero(accept(li, lj))[:TUPLE_CAP]
    return len(kept), np.bincount(idx[kept].reshape(-1), minlength=n).astype(np.int64), kept


# ----------------------------------------------------------------------------------------------- step 3
def terms(p, q, par, w):
    """The 27 weighted terms of each used correspondence -> (k, 27)."""
    r = [p[:, c] - q[:, c] for c in range(3)]
    rr_ = (r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]
    t = par / (rr_ + par)
    ws = w * (t * t)
    z, one = np.zeros(len(p)), np.ones(len(p))
    qx, qy, qz = q[:, 0], q[:, 1], q[:, 2]
    Jx = [z, -qz, qy, -one, z, z]
    Jy = [qz, z, -qx, z, -one, z]
    Jz = [-qy, qx, z, z, z, -one]
    out = np.empty((len(p), 27))
    for e, (a, b) in enumerate(UPPER):
        out[:, e] = ((Jx[a] * Jx[b] + Jy[a] * Jy[b]) + Jz[a] * Jz[b]) * ws
    for a in range(6):
        out[:, 21 + a] = ((Jx[a] * r[0] + Jy[a] * r[1]) + Jz[a] * r[2]) * ws
    return out


def reduce27(tm):
    """The header's reduction: per-thread stride sums, a butterfly per warp, then the warps in order -> (27,)."""
    k = len(tm)
    rows = -(-k // THREADS)
    pad = np.zeros((rows * THREADS, 27))
    pad[:k] = tm
    acc = np.zeros((THREADS, 27))
    for r in range(rows):
        acc = acc + pad[r * THREADS:(r + 1) * THREADS]
    V = acc.reshape(WARPS, 32, 27)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        V = V + V[:, lane ^ o]
    S = V[0, 0].copy()
    for w in range(1, WARPS):
        S = S + V[w, 0]
    return S


def cholesky_solve(S):
    """Solve J^T J xi = -J^T r from the 27 sums by the header's Cholesky -> xi (6,) list, or None on a bad pivot."""
    A = [[0.0] * 6 for _ in range(6)]
    for e, (a, b) in enumerate(UPPER):
        A[a][b] = A[b][a] = float(S[e])
    L = [[0.0] * 6 for _ in range(6)]
    for j in range(6):
        v = A[j][j]
        for k in range(j):
            v = v - L[j][k] * L[j][k]
        if not (v > 0.0 and v <= DBL_MAX):
            return None
        d = math.sqrt(v)
        L[j][j] = d
        for i in range(j + 1, 6):
            u = A[i][j]
            for k in range(j):
                u = u - L[i][k] * L[j][k]
            L[i][j] = u / d
    x = [0.0] * 6
    for i in range(6):
        v = -float(S[21 + i])
        for k in range(i):
            v = v - L[i][k] * x[k]
        x[i] = v / L[i][i]
    for i in range(5, -1, -1):
        v = x[i]
        for k in range(i + 1, 6):
            v = v - L[k][i] * x[k]
        x[i] = v / L[i][i]
    return x


def delta_matrix(xi):
    """[Rz(xi2) Ry(xi1) Rx(xi0) | xi3, xi4, xi5] -> (3, 4)."""
    sx, cx, sy, cy, sz, cz = (math.sin(xi[0]), math.cos(xi[0]), math.sin(xi[1]), math.cos(xi[1]), math.sin(xi[2]),
                              math.cos(xi[2]))
    czsy, szsy = cz * sy, sz * sy
    return np.array([[cz * cy, czsy * sx - sz * cx, czsy * cx + sz * sx, xi[3]],
                     [sz * cy, szsy * sx + cz * cx, szsy * cx - cz * sx, xi[4]],
                     [-sy, cy * sx, cy * cx, xi[5]]])


def compose(D, T):
    """delta T for 3x4 maps, entry (r, c) ((D_r0 T_0c + D_r1 T_1c) + D_r2 T_2c), + D_r3 in column 3."""
    N = np.empty((3, 4))
    for r in range(3):
        for c in range(4):
            v = (D[r, 0] * T[0, c] + D[r, 1] * T[1, c]) + D[r, 2] * T[2, c]
            N[r, c] = v + D[r, 3] if c == 3 else v
    return N


def apply(D, q):
    return np.stack([((D[r, 0] * q[:, 0] + D[r, 1] * q[:, 1]) + D[r, 2] * q[:, 2]) + D[r, 3] for r in range(3)], 1)


def gnc(p, q, mult):
    """OptimizePairwise on the used matches -> (T (3, 4), status 0 or 2)."""
    use = np.flatnonzero(mult > 0)
    P, Q, W = p[use], q[use].copy(), mult[use].astype(np.float64)
    T, par = np.eye(3, 4), 1.0
    for itr in range(ITERATIONS):
        if itr % 4 == 0 and par > STOP:
            par = par / DIV
        xi = cholesky_solve(reduce27(terms(P, Q, par, W)))
        if xi is None:
            return T, 2
        D = delta_matrix(xi)
        T = compose(D, T)
        Q = apply(D, Q)
    return T, 0


# ----------------------------------------------------------------------------------------------- the whole call
def fgr_ref(f1, f2, matches, seed=0, thr=0.2):
    """usip_fgr_f64 for one (pair, K): fragments f1 (n1, 3), f2 (n2, 3) f32 and the match list (n, 2) -> dict of Rt
    (3, 4), n_tuples, n_inliers, info (6, 6), status, and the intermediate mult, scale, mean1, mean2."""
    f1, f2 = np.asarray(f1, np.float32).reshape(-1, 3), np.asarray(f2, np.float32).reshape(-1, 3)
    m = np.asarray(matches, np.int64).reshape(-1, 2)
    if len(m) and (m[:, 0].min() < 0 or m[:, 0].max() >= len(f1) or m[:, 1].min() < 0 or m[:, 1].max() >= len(f2)):
        return dict(Rt=np.zeros((3, 4)), n_tuples=0, n_inliers=0, info=np.zeros((6, 6)), status=3)
    m1, m2, scale, degenerate = normalise(f1, f2)
    x1, x2 = f1[m[:, 0]].astype(np.float64), f2[m[:, 1]].astype(np.float64)
    n_tuples, mult, T, status = 0, np.zeros(len(m), np.int64), np.eye(3, 4), 4 if degenerate else 0
    if not degenerate:
        p, q = (x1 - m1) / scale, (x2 - m2) / scale
        n_tuples, mult, _ = tuples(p, q, seed)
        if 3 * n_tuples < MIN_CORR:
            status = 1
        else:
            T, status = gnc(p, q, mult)
    moved = status in (0, 2)
    sc, R = (scale, T) if moved else (0.0, np.eye(3, 4))
    Rt = np.empty((3, 4))
    Rt[:, :3] = R[:, :3]
    for r in range(3):
        a = (R[r, 0] * m2[0] + R[r, 1] * m2[1]) + R[r, 2] * m2[2]
        Rt[r, 3] = ((-a) + R[r, 3] * sc) + m1[r]
    with np.errstate(invalid="ignore", over="ignore"):
        inl = rr.inliers(Rt[None], x1, x2, thr)[0] if len(m) else np.zeros(0, bool)
    return dict(Rt=Rt, n_tuples=n_tuples, n_inliers=int(inl.sum()), info=ir.info_of(x1[inl]), status=status,
                mult=mult, scale=scale, mean1=m1, mean2=m2, inliers=inl)


def register_ref(xyz1, desc1, xyz2, desc2, K, seed=0, thr=0.2):
    """Mutual matching of the first min(K, n) rows of each scan, then fgr_ref -> (matches, fgr_ref dict)."""
    a, b = np.asarray(xyz1)[:K], np.asarray(xyz2)[:K]
    m = mutual_ref(np.asarray(desc1)[:K], np.asarray(desc2)[:K])
    return m, fgr_ref(a, b, m, seed, thr)
