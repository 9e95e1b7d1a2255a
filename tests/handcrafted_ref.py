"""Numpy restatement of csrc/handcrafted.cu (include/usip_b200.h, "Handcrafted keypoint baselines"): the fp32 neighbour
rule exactly, the ISS scatter and the Harris normals and response in float64 (np.linalg.eigh), the non-maximum rule and
the Philox selection through tests/philox_ref.py.  One cloud P (N, 3) float32 at a time."""
import numpy as np
from scipy.spatial import cKDTree

from tests.philox_ref import pg_random

PURPOSE_HC_KEYPOINT, PURPOSE_HC_PAD = 7, 8


def neighbours(P, r):
    """CSR (ptr (N+1,), idx) of N_r(i): (dx*dx + dy*dy) + dz*dz in float32 <= fl32(r*r), i included, ascending j;
    non-finite rows have no neighbours and are nobody's."""
    P = np.ascontiguousarray(P, np.float32)
    N = len(P)
    fin = np.isfinite(P).all(axis=1)
    rows = np.flatnonzero(fin)
    r32 = np.float32(r)
    r2 = r32 * r32
    lists = [np.zeros(0, np.int64)] * N
    if len(rows):
        tree = cKDTree(P[rows].astype(np.float64))
        cand = tree.query_ball_point(P[rows].astype(np.float64), float(r) * 1.001 + 1e-30, return_sorted=True)
        for a, c in zip(rows, cand):
            j = rows[np.asarray(c, np.int64)]
            d = P[j] - P[a]
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            lists[a] = j[d2 <= r2]
    cnt = np.array([len(x) for x in lists], np.int64)
    ptr = np.concatenate([[0], np.cumsum(cnt)])
    idx = np.concatenate(lists) if N else np.zeros(0, np.int64)
    return ptr, idx.astype(np.int64)


def _segsum(vals, ptr):
    """Per-segment sums of vals (nnz, k) over CSR ptr; empty segments give 0."""
    N = len(ptr) - 1
    out = np.zeros((N,) + vals.shape[1:], np.float64)
    nz = np.flatnonzero(ptr[1:] > ptr[:-1])
    if len(nz):
        out[nz] = np.add.reduceat(vals, ptr[nz], axis=0)
    return out


def _rows_of(ptr):
    return np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))


def _outer6(d):
    return np.stack([d[:, 0] * d[:, 0], d[:, 0] * d[:, 1], d[:, 0] * d[:, 2], d[:, 1] * d[:, 1], d[:, 1] * d[:, 2],
                     d[:, 2] * d[:, 2]], axis=1)


def _sym(c6):
    return np.stack([np.stack([c6[:, 0], c6[:, 1], c6[:, 2]], 1), np.stack([c6[:, 1], c6[:, 3], c6[:, 4]], 1),
                     np.stack([c6[:, 2], c6[:, 4], c6[:, 5]], 1)], 1)


def iss_saliency(P, salient_radius, gamma_21, gamma_32, min_neighbors, nb=None):
    """-> (saliency (N,) f64, count (N,) i64, eig (N, 3) f64 descending)."""
    ptr, idx = nb if nb is not None else neighbours(P, salient_radius)
    P64 = np.asarray(P, np.float64)
    d = P64[idx] - P64[_rows_of(ptr)]
    C = _segsum(_outer6(d), ptr)
    cnt = np.diff(ptr)
    fin = np.isfinite(P64).all(axis=1)
    eig = np.zeros((len(P), 3))
    if fin.any():
        eig[fin] = np.linalg.eigh(_sym(C[fin]))[0][:, ::-1]
    e1, e2, e3 = eig[:, 0], eig[:, 1], eig[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        ok = fin & (cnt >= min_neighbors) & (e2 / e1 < gamma_21) & (e3 / e2 < gamma_32) & (e3 >= 0)
    return np.where(ok, e3, 0.0), cnt, eig


def harris_response(P, radius, nb=None):
    """-> (response (N,) f64, count (N,) i64, normals (N, 3) f64, normal eigenvalues (N, 3) ascending)."""
    ptr, idx = nb if nb is not None else neighbours(P, radius)
    P64 = np.asarray(P, np.float64)
    N = len(P)
    cnt = np.diff(ptr)
    d = P64[idx] - P64[_rows_of(ptr)]
    s1 = _segsum(d, ptr)
    s2 = _segsum(_outer6(d), ptr)
    nrm = np.full((N, 3), np.nan)
    lam = np.full((N, 3), np.nan)
    ok = cnt >= 3
    if ok.any():
        m = s1[ok] / cnt[ok, None]
        cov = _sym(s2[ok] / cnt[ok, None]) - m[:, :, None] * m[:, None, :]
        w, v = np.linalg.eigh(cov)
        nrm[ok] = v[:, :, 0]
        lam[ok] = w
    nj = nrm[idx]
    good = np.isfinite(nj).all(axis=1)
    A6 = _segsum(np.where(good[:, None], _outer6(np.nan_to_num(nj)), 0.0), ptr)
    cf = _segsum(good.astype(np.float64)[:, None], ptr)[:, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        a = A6 / cf[:, None]
    a0, a1, a2, a3, a4, a5 = a.T
    tr = a0 + a3 + a5
    det = a0 * a3 * a5 + 2.0 * a1 * a2 * a4 - a2 * a2 * a3 - a1 * a1 * a5 - a4 * a4 * a0
    R = np.where(tr != 0, 0.04 + det - 0.04 * tr * tr, 0.0)
    R = np.where(cf > 0, R, np.nan)
    return R, cnt, nrm, lam


def nonmax(P, score, radius, threshold, strict, min_neighbors, nb=None):
    """-> (flag (N,) bool, count (N,) i64, gap (N,) f64): gap = score_i - the largest score of a neighbour at other
    coordinates (-inf without one; NaN scores ignored)."""
    ptr, idx = nb if nb is not None else neighbours(P, radius)
    P = np.asarray(P, np.float32)
    cnt = np.diff(ptr)
    fin = np.isfinite(P).all(axis=1)
    rows = _rows_of(ptr)
    sj = np.where(np.isnan(score[idx]), -np.inf, score[idx])
    same = (P[idx] == P[rows]).all(axis=1)
    mx_all = np.full(len(P), -np.inf)
    mx_other = np.full(len(P), -np.inf)
    np.maximum.at(mx_all, rows, sj)
    np.maximum.at(mx_other, rows, np.where(same, -np.inf, sj))
    with np.errstate(invalid="ignore"):
        elig = fin & ((score > threshold) if strict else (score >= threshold))
        flag = elig & (cnt >= min_neighbors) & ~(mx_all > score)
        gap = score - mx_other
    return flag, cnt, gap


def select(flag, N, L, seed, step, cloud):
    """usip_hc_select for one cloud -> (order (L,) i64, count)."""
    rows = np.arange(N)
    cnt = 0 if flag is None else int(np.count_nonzero(flag))
    parts = []
    if cnt:
        fr = np.flatnonzero(flag)
        k = pg_random(seed, step, cloud, fr, PURPOSE_HC_KEYPOINT)[0]
        parts.append(fr[np.lexsort((fr, k))][:min(cnt, L)])
    rest = L - min(cnt, L)
    if rest:
        k2 = pg_random(seed, step, cloud, rows, PURPOSE_HC_PAD)[0]
        parts.append(rows[np.lexsort((rows, k2))][:rest])
    return np.concatenate(parts).astype(np.int64), cnt


def iss_flags(P, salient_radius=2.0, non_max_radius=2.0, gamma_21=0.975, gamma_32=0.975, min_neighbors=5):
    sal = iss_saliency(P, salient_radius, gamma_21, gamma_32, min_neighbors)[0]
    return nonmax(P, sal, non_max_radius, 0.0, True, min_neighbors)[0]


def harris_flags(P, radius=1.0, threshold=0.001):
    R = harris_response(P, radius)[0]
    return nonmax(P, R, radius, threshold, False, 1)[0]


def detect(method, pc, M, seed, step, **kw):
    """A detector's run_model on one batch pc (B, 3, N) float32 numpy -> (keypoints (B, 3, M), counts (B,))."""
    B, _, N = pc.shape
    kp = np.empty((B, 3, M), np.float32)
    counts = np.empty(B, np.int64)
    for b in range(B):
        P = np.ascontiguousarray(pc[b].T)
        f = None if method == "random" else (iss_flags(P, **kw) if method == "iss" else harris_flags(P, **kw))
        order, counts[b] = select(f, N, M, seed, step, b)
        kp[b] = pc[b][:, order]
    return kp, counts
