"""Float64 restatement of the SceneNN descriptor pair kernels of csrc/pairgen.cu (pg_icp, pair_gather_icp_f64_kernel,
pg_scenenn_f64, scenenn_desc_pair_augment_kernel) and of FarthestSampler on float64 points (csrc/fps.cu, usip_fps_f64).

The fp32 and float64 rounding points are the kernels'; the fused multiply-adds are not (pg_icp's and pg_rowvec's chains
are plain float64 here, pg_colvec's fp32 chain a float64 add rounded to fp32 per step, as in tests/pairgen_ref.py).  So
the outputs agree with the kernel to within one fp32 ulp, and FPS indices exactly where no two distances tie within
float64 rounding."""
import numpy as np

from tests.pairgen_ref import ANY_ROT, ROT_HORIZONTAL, TRANSLATION, _colvec, _dst_transform, _rows_of, \
    _rowvec, _transform_outputs, f32, f64
# ------------------------------------------------------------------------------ SceneNN descriptor pairs (float64)
def icp_map(T, xyz):
    """pg_icp: hom2cart(T @ [x y z 1]) in float64 (numpy's order, not the kernel's fused chain), w divided literally."""
    h = xyz.astype(f64) @ T[:, 0:3].T + T[:, 3]
    return h[:, 0:3] / h[:, 3:4]


def gather_candidates_icp(scans, offsets, scan_of_cloud, rows, cand, icp):
    """pair_gather_icp_f64_kernel -> (2B, n_cand, 3) f64: the anchor's (c even) ICP'd, the positive's exact."""
    pts = np.stack([_rows_of(scans, offsets, scan_of_cloud, rows, c)[cand[c], 0:3].astype(f64)
                    for c in range(len(scan_of_cloud))])
    for b in range(len(scan_of_cloud) // 2):
        pts[2 * b] = icp_map(icp[b], pts[2 * b])
    return pts


def farthest_sampler(pts, start, k):
    """data/*_loader.py FarthestSampler.sample on float64 points, the start given -> (k,) selected indices."""
    pts = np.asarray(pts, f64)
    idx = [int(start)]
    d = ((pts[idx[0]] - pts) ** 2).sum(axis=1)
    for _ in range(1, k):
        idx.append(int(np.argmax(d)))
        d = np.minimum(d, ((pts[idx[-1]] - pts) ** 2).sum(axis=1))
    return np.array(idx, np.int64)


def _scenenn_f64(flags, kind, P, X):
    """pg_scenenn_f64: rotations (kind >= 1), scale and shift (kind 2), float64, no jitter."""
    if kind >= 1:
        for r in range(3):
            if flags & (ROT_HORIZONTAL << r):
                X = _rowvec(X, P[9 * r:9 * r + 9].reshape(3, 3))
    if kind == 2:
        X = X * P[27]
        if flags & TRANSLATION:
            X = X + P[28:31]
    return X


def scenenn_desc_pair_augment(scans, offsets, scan_of_cloud, rows, icp, cand_pts, node_idx, params, S, flags):
    """scenenn_desc_pair_augment_kernel: numpy arrays in usip_scenenn_desc_pair_augment's layout -> its nine outputs."""
    B, N, M = len(scan_of_cloud) // 2, rows.shape[1], node_idx.shape[1]
    out = [np.empty((B, k, n), f32) for k, n in ((3, N), (S, N), (3, M), (3, N), (S, N), (3, M))]
    for c in range(2 * B):
        b, side = c >> 1, c & 1
        P = params[b]
        kind = int(P[45]) if P[45] in (1.0, 2.0) else 0
        p = _rows_of(scans, offsets, scan_of_cloud, rows, c)
        xyz, sn = p[:, 0:3].copy(), p[:, 3:3 + S].copy()
        if side == 0:
            xyz = _scenenn_f64(flags, kind, P, icp_map(icp[b], xyz)).astype(f32)
            sn[:, 0:3] = icp_map(icp[b], sn[:, 0:3]).astype(f32)
        elif kind >= 1 and flags & ANY_ROT:
            xyz = _scenenn_f64(flags, kind, P, xyz.astype(f64)).astype(f32)
        elif kind == 2:
            xyz = (xyz.astype(f64) * f64(f32(P[27]))).astype(f32)
            if flags & TRANSLATION:
                xyz = (xyz.astype(f64) + P[28:31]).astype(f32)
        if kind >= 1:
            for r in range(3):
                if flags & (ROT_HORIZONTAL << r):
                    sn[:, 0:3] = _rowvec(sn[:, 0:3].astype(f64), P[9 * r:9 * r + 9].reshape(3, 3)).astype(f32)
        nd = _scenenn_f64(flags, kind, P, cand_pts[c][node_idx[c]].astype(f64)).astype(f32)
        if side == 1:
            xyz, nd = _dst_transform(P, xyz), _dst_transform(P, nd)
            sn[:, 0:3] = _colvec(sn[:, 0:3], P[31:40].astype(f32).reshape(3, 3))
        out[3 * side][b], out[3 * side + 1][b], out[3 * side + 2][b] = xyz.T, sn.T, nd.T
    return tuple(out) + _transform_outputs(params)
