"""Float64 restatement of eval_rep.m:142-146 in usip_repeatability_f64's operation order, elementwise (no `@`, whose
BLAS summation order is unspecified), so that the kernel's counts can be compared exactly."""
import numpy as np


def apply_map(T, pts):
    """T (3, 4) f64, pts (n, 3) -> (n, 3): ((m0 x + m1 y) + m2 z) + m3 per row, no fused multiply-add."""
    p = np.asarray(pts, dtype=np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], axis=1)


def pair_counts(anc, pos, F_a, F_p, T_gt, ks, radius):
    """anc (na, 3), pos (np, 3) keypoints in selection order -> (inliers, n_anc) lists over ks."""
    a = apply_map(F_a, anc)
    q = apply_map(T_gt, apply_map(F_p, pos))
    inl, nanc = [], []
    for K in ks:
        na, npk = min(K, len(a)), min(K, len(q))
        if na == 0 or npk == 0:
            inl.append(0); nanc.append(na)
            continue
        d = q[None, :npk, :] - a[:na, None, :]
        s = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        inl.append(int((np.sqrt(s.min(axis=1)) < radius).sum()))
        nanc.append(na)
    return inl, nanc


def repeatability_ref(kp, order, count, pairs, frames, ks, radius):
    """The kernel's contract on host arrays: kp (S, 3, M) f32, order (S, M), count (S,), pairs (P, 2), frames
    (P, 3, 3, 4) -> (inliers (P, nK), n_anc (P, nK)) int."""
    kmax = max(ks)
    sel = lambda s: kp[s][:, order[s, :min(int(count[s]), kmax)]].T
    out = [pair_counts(sel(a), sel(p), f[0], f[1], f[2], ks, radius) for (a, p), f in zip(pairs, frames)]
    return (np.array([o[0] for o in out], dtype=np.int64).reshape(-1, len(ks)),
            np.array([o[1] for o in out], dtype=np.int64).reshape(-1, len(ks)))
