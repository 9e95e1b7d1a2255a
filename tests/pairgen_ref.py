"""Numpy restatement of csrc/pairgen.cu's device-mode random streams and of its per-point arithmetic.

Streams (bit-exact up to the math library, see `normals`):
  pg_normal2 (pairgen.cu:41-48): u1 = (a + 1) 2^-32 in (0, 1], u2 = b 2^-32, r = sqrt(-2 log u1), (z0, z1) =
    r (cospi(2 u2), sinpi(2 u2)).  sincospi is restated by exact quadrant reduction, not sin(2 pi u2).
  pg_clip (:50): min(max(v, -lim), lim).
  pg_jitter_xyz (:381-392): one Philox draw of (cloud, item, purpose, sub 0) -> four normals, the first three scaled
    by sigma and clipped.  pg_jitter_sn (:426-445): block q of four sn columns draws (cloud, item, PURPOSE_JIT_SN,
    sub q / 4).  test_cloud_gather_kernel (:703-716): PURPOSE_NOISE, n = fl32(z), x + fl32(n sigma) in fp32.
  Which key each kernel uses: pair_augment_kernel and desc_pair_augment_kernel the cloud c (:519, :521, :543, :655,
  :657, :675), pc and nodes N(0, 0.04^2) clipped at 0.12, sn N(0, 0.01^2) clipped at 0.05; modelnet_pair_augment_kernel
  the pair b (:601, :603, :621), pc and sn 0.01 / 0.05, nodes 0.04 / 0.1.

Arithmetic (`pair_augment`, `modelnet_pair_augment`, `desc_pair_augment`, `cloud_gather`): the kernels' rounding
points, each fp32 step as a float64 operation rounded to fp32 and each float64 step plainly in float64.  The kernels
fuse the rotations' multiply-adds (pg_rowvec in float64, pg_colvec in fp32) and this restatement does not: pg_rowvec's
chain is plain float64 here, and pg_colvec's fp32 chain is a float64 add rounded to fp32 per step.  So they agree to
within one fp32 ulp, not bit for bit: use it where indexing, not the last bit, is under test."""
import numpy as np

from tests.philox_ref import pg_random

PURPOSE_ROWS, PURPOSE_CAND, PURPOSE_START, PURPOSE_JIT_PC, PURPOSE_JIT_SN, PURPOSE_JIT_NODE, PURPOSE_NOISE = range(7)
TRAIN, ROT_HORIZONTAL, ROT_3D, ROT_PERTURBATION, TRANSLATION, ENU_TO_CAM, HEIGHT_SCALE = 1, 2, 4, 8, 16, 32, 64
ANY_ROT = ROT_HORIZONTAL | ROT_3D | ROT_PERTURBATION
PC_LAW, SN_LAW, NODE_LAW = (0.04, 0.12), (0.01, 0.05), (0.04, 0.12)                  # KITTI / Oxford, per cloud
MN_PC_LAW, MN_SN_LAW, MN_NODE_LAW = (0.01, 0.05), (0.01, 0.05), (0.04, 0.1)          # ModelNet, per pair
_TWO_M32 = 2.3283064365386963e-10                                                  # 2^-32
f32, f64 = np.float32, np.float64


def counter(seed, step, cloud, item, purpose, sub=0):
    """pg_random's Philox counter and key (pairgen.cu:34-38) -> (c0, c1, c2, c3, k0, k1) as Python ints."""
    step, seed = int(step) & (2 ** 64 - 1), int(seed) & (2 ** 64 - 1)
    return (int(item) & 0xFFFFFFFF, int(cloud) & 0xFFFFFFFF, step & 0xFFFFFFFF,
            (int(purpose) | (int(sub) << 8) | ((step >> 32) << 16)) & 0xFFFFFFFF, seed & 0xFFFFFFFF, seed >> 32)


def ulp_shift(v, k):
    """v (float64 array) moved k ulps along the ordered doubles (k < 0: down); -0 and +0 are one point."""
    i = np.asarray(v, f64).view(np.int64)
    o = np.where(i < 0, -(i & 0x7FFFFFFFFFFFFFFF), i) + np.asarray(k, np.int64)
    return np.where(o < 0, (-o) | np.int64(-0x8000000000000000), o).view(f64)


def _sincospi(x):
    """(sin(pi x), cos(pi x)) for x = k 2^-31 in [0, 2): x = q/2 + t with q the nearest quadrant and |t| <= 1/4, both
    exact, then sin / cos of pi t."""
    q = np.rint(2.0 * x)
    t = x - 0.5 * q
    s, c = np.sin(np.pi * t), np.cos(np.pi * t)
    q = q.astype(np.int64) & 3
    sin = np.choose(q, [s, c, -s, -c])
    cos = np.choose(q, [c, -s, -c, s])
    return sin, cos


def normal2(a, b):
    """pg_normal2 on uint32 arrays -> (z0, z1) float64."""
    u1 = (np.asarray(a, f64) + 1.0) * _TWO_M32
    u2 = np.asarray(b, f64) * _TWO_M32
    r = np.sqrt(-2.0 * np.log(u1))
    s, c = _sincospi(2.0 * u2)
    return r * c, r * s


def normals(seed, step, cloud, items, purpose, sub=0, ulps=0):
    """The four normals of pg_random(seed, step, cloud, item, purpose, sub) -> (len(items), 4) float64.  ulps (scalar
    or (4,)): every normal moved that many double ulps, for brackets around the device's libm."""
    u = pg_random(seed, step, cloud, items, purpose, sub)
    z0, z1 = normal2(u[0], u[1])
    z2, z3 = normal2(u[2], u[3])
    z = np.stack([z0, z1, z2, z3], axis=-1)
    return ulp_shift(z, np.broadcast_to(np.asarray(ulps, np.int64), (4,))) if np.any(ulps) else z


def clip(v, lim):
    """pg_clip."""
    return np.minimum(np.maximum(v, -lim), lim)


def jitter_xyz(seed, step, key, n, purpose, law, ulps=0):
    """pg_jitter_xyz for items 0..n-1 of one key (cloud or pair) -> (n, 3)."""
    sigma, lim = law
    return clip(sigma * normals(seed, step, key, np.arange(n), purpose, 0, ulps)[:, :3], lim)


def jitter_sn(seed, step, cloud, n, S, ulps=0):
    """pg_jitter_sn for items 0..n-1 of one cloud -> (n, S): columns q..q+3 from sub q / 4."""
    sigma, lim = SN_LAW
    u = np.broadcast_to(np.asarray(ulps, np.int64), (4,))
    blocks = [clip(sigma * normals(seed, step, cloud, np.arange(n), PURPOSE_JIT_SN, q // 4, u), lim)
              for q in range(0, S, 4)]
    return np.concatenate(blocks, axis=1)[:, :S]


def kitti_jitter(seed, step, n_clouds, N, M, S, ulps=0):
    """Device-mode jitter of usip_pair_augment / usip_desc_pair_augment in upload layout: (2B, N, 3), (2B, N, S),
    (2B, M, 3), keyed by cloud."""
    pc = np.stack([jitter_xyz(seed, step, c, N, PURPOSE_JIT_PC, PC_LAW, ulps) for c in range(n_clouds)])
    sn = np.stack([jitter_sn(seed, step, c, N, S, ulps) for c in range(n_clouds)])
    nd = np.stack([jitter_xyz(seed, step, c, M, PURPOSE_JIT_NODE, NODE_LAW, ulps) for c in range(n_clouds)])
    return pc, sn, nd


def modelnet_jitter(seed, step, n_pairs, N, M, ulps=0):
    """Device-mode jitter of usip_modelnet_pair_augment in upload layout: (B, N, 3) x 2, (B, M, 3), keyed by pair."""
    pc = np.stack([jitter_xyz(seed, step, b, N, PURPOSE_JIT_PC, MN_PC_LAW, ulps) for b in range(n_pairs)])
    sn = np.stack([jitter_xyz(seed, step, b, N, PURPOSE_JIT_SN, MN_SN_LAW, ulps) for b in range(n_pairs)])
    nd = np.stack([jitter_xyz(seed, step, b, M, PURPOSE_JIT_NODE, MN_NODE_LAW, ulps) for b in range(n_pairs)])
    return pc, sn, nd


def noise_draws(seed, step, n_clouds, N, ulps=0):
    """Device-mode noise of usip_test_cloud_gather in upload layout: (B, 3, N) f32 = fl32(z)."""
    return np.stack([normals(seed, step, c, np.arange(N), PURPOSE_NOISE, 0, ulps)[:, :3].T.astype(f32)
                     for c in range(n_clouds)])


# ------------------------------------------------------------------------------------------------ the arithmetic
def _rowvec(v, R):
    """pg_rowvec (:353-358) without the fused multiply-adds: v (n, 3) float64 @ R (3, 3)."""
    return v[:, 0:1] * R[0] + v[:, 1:2] * R[1] + v[:, 2:3] * R[2]


def _colvec(v, RT):
    """pg_colvec (:362-367): R @ v per point in fp32, v (n, 3) f32, as the kernel's chain fl32(R0 a), then
    fl32(R1 b + t), fl32(R2 c + t).  An fp32 product is exact in float64, so each step is one float64 add rounded to
    fp32 (a double rounding, which can differ from the fused one in the last bit)."""
    v = v.astype(f64)
    RT = RT.astype(f32).astype(f64)
    t = (v[:, 0:1] * RT[:, 0]).astype(f32)
    t = (v[:, 1:2] * RT[:, 1] + t).astype(f32)
    return (v[:, 2:3] * RT[:, 2] + t).astype(f32)


def _enu_to_cam(flags, hs, xyz, sn):
    """pg_enu_to_cam (:466-475) on f32 arrays (copies)."""
    xyz, sn = xyz.copy(), None if sn is None else sn.copy()
    if not flags & ENU_TO_CAM:
        return xyz, sn
    if flags & (TRAIN | HEIGHT_SCALE) == TRAIN | HEIGHT_SCALE:
        xyz[:, 2] = (xyz[:, 2].astype(f64) * f64(f32(hs))).astype(f32)
    xyz[:, 1], xyz[:, 2] = -xyz[:, 2], xyz[:, 1].copy()
    if sn is not None and sn.shape[1] >= 3:
        sn[:, 1], sn[:, 2] = -sn[:, 2], sn[:, 1].copy()
    return xyz, sn


def _augment_point(flags, P, sc, j, xyz, sn):
    """pg_augment_point (:395-423): rotations, jitter, scale, shift of f32 rows; sn (n, S) f32 or None."""
    X = xyz.astype(f64)
    for r in range(3):
        if flags & (ROT_HORIZONTAL << r):
            R = P[9 * r:9 * r + 9].reshape(3, 3)
            X = _rowvec(X, R)
            if sn is not None and sn.shape[1] >= 3:
                sn = sn.copy()
                sn[:, 0:3] = _rowvec(sn[:, 0:3].astype(f64), R).astype(f32)
    if flags & ANY_ROT:
        X = (X + j) * sc
        if flags & TRANSLATION:
            X = X + P[28:31]
        return X.astype(f32), sn
    x = (xyz.astype(f64) + j).astype(f32)
    x = (x.astype(f64) * f64(f32(sc))).astype(f32)
    if flags & TRANSLATION:
        x = (x.astype(f64) + P[28:31]).astype(f32)
    return x, sn


def _augment_node(flags, P, sc, j, xyz):
    """pg_augment_node (:448-457): float64 from the f32 node to the final cast."""
    X = xyz.astype(f64)
    for r in range(3):
        if flags & (ROT_HORIZONTAL << r):
            X = _rowvec(X, P[9 * r:9 * r + 9].reshape(3, 3))
    X = (X + j) * sc
    if flags & TRANSLATION:
        X = X + P[28:31]
    return X.astype(f32)


def _dst_transform(P, xyz):
    """pg_dst_transform (:479-484): fp32 R, then fp32 scale and shift."""
    RT = P[31:40].astype(f32).reshape(3, 3)
    x = _colvec(xyz, RT)
    x = (x.astype(f64) * f64(f32(P[43]))).astype(f32)
    return (x.astype(f64) + P[40:43].astype(f32).astype(f64)).astype(f32)


def _rows_of(scans, offsets, scan_of_cloud, rows, c):
    return scans[offsets[scan_of_cloud[c]] + rows[c].astype(np.int64)]


def _transform_outputs(params):
    B = params.shape[0]
    return (params[:, 31:40].astype(f32).reshape(B, 3, 3), params[:, 43].astype(f32),
            params[:, 40:43].astype(f32).reshape(B, 3, 1))


def pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, jit_pc=None, jit_sn=None,
                 jit_node=None):
    """pair_augment_kernel (:487-552): numpy arrays in usip_pair_augment's layout -> its nine outputs.  Jitter arrays
    (2B, N, 3), (2B, N, S), (2B, M, 3) are needed in train mode."""
    B, N, M, C = len(scan_of_cloud) // 2, rows.shape[1], nodes.shape[2], scans.shape[1]
    sn_col = C - 1 if S == 1 else 3
    out = [np.empty((B, k, n), f32) for k, n in ((3, N), (S, N), (3, M), (3, N), (S, N), (3, M))]
    for c in range(2 * B):
        b, side = c >> 1, c & 1
        P = params[b]
        p = _rows_of(scans, offsets, scan_of_cloud, rows, c)
        xyz, sn = _enu_to_cam(flags, P[44], p[:, 0:3], p[:, sn_col:sn_col + S])
        nd, _ = _enu_to_cam(flags & ~HEIGHT_SCALE, 1.0, nodes[c].T, None)
        if flags & TRAIN:
            xyz, sn = _augment_point(flags, P, P[27], jit_pc[c], xyz, sn)
            sn = (sn.astype(f64) + jit_sn[c]).astype(f32)
            nd = _augment_node(flags, P, P[27], jit_node[c], nd)
        if side == 1:
            xyz, nd = _dst_transform(P, xyz), _dst_transform(P, nd)
            if S >= 3:
                sn = sn.copy()
                sn[:, 0:3] = _colvec(sn[:, 0:3], P[31:40].astype(f32).reshape(3, 3))
        out[3 * side][b], out[3 * side + 1][b], out[3 * side + 2][b] = xyz.T, sn.T, nd.T
    return tuple(out) + _transform_outputs(params)


def _modelnet_sn(flags, P, sc, j, sn):
    """pg_modelnet_sn (:557-567)."""
    if flags & ANY_ROT:
        return _augment_node(flags & ~TRANSLATION, P, sc, j, sn)
    x = (sn.astype(f64) + j).astype(f32)
    return (x.astype(f64) * f64(f32(sc))).astype(f32)


def modelnet_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, flags, jit_pc=None, jit_sn=None,
                          jit_node=None):
    """modelnet_pair_augment_kernel (:573-628): jitter per pair, (B, N, 3), (B, N, 3), (B, M, 3)."""
    B, N, M = len(scan_of_cloud) // 2, rows.shape[1], nodes.shape[2]
    out = [np.empty((B, 3, n), f32) for n in (N, N, M, N, N, M)]
    for c in range(2 * B):
        b, side = c >> 1, c & 1
        P = params[b]
        p = _rows_of(scans, offsets, scan_of_cloud, rows, c)
        xyz, sn, nd = p[:, 0:3], p[:, 3:6], nodes[c].T
        if flags & TRAIN:
            xyz, _ = _augment_point(flags, P, P[27], jit_pc[b], xyz, None)
            sn = _modelnet_sn(flags, P, P[27], jit_sn[b], sn)
            nd = _augment_node(flags, P, P[27], jit_node[b], nd)
        if side == 1:
            xyz, nd = _dst_transform(P, xyz), _dst_transform(P, nd)
            sn = _colvec(sn, P[31:40].astype(f32).reshape(3, 3))
        out[3 * side][b], out[3 * side + 1][b], out[3 * side + 2][b] = xyz.T, sn.T, nd.T
    return tuple(out) + _transform_outputs(params)


def desc_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, jit_pc=None, jit_sn=None,
                      jit_node=None):
    """desc_pair_augment_kernel (:633-683): params (2B, 32) per cloud, no dst transform, sn = columns 3:3+S."""
    B, N, M = len(scan_of_cloud) // 2, rows.shape[1], nodes.shape[2]
    out = [np.empty((B, k, n), f32) for k, n in ((3, N), (S, N), (3, M), (3, N), (S, N), (3, M))]
    for c in range(2 * B):
        b, side = c >> 1, c & 1
        P = params[c]
        p = _rows_of(scans, offsets, scan_of_cloud, rows, c)
        xyz, sn = _enu_to_cam(flags, 1.0, p[:, 0:3], p[:, 3:3 + S])
        nd, _ = _enu_to_cam(flags, 1.0, nodes[c].T, None)
        if flags & TRAIN:
            xyz, sn = _augment_point(flags, P, P[27], jit_pc[c], xyz, sn)
            sn = (sn.astype(f64) + jit_sn[c]).astype(f32)
            nd = _augment_node(flags, P, P[27], jit_node[c], nd)
        out[3 * side][b], out[3 * side + 1][b], out[3 * side + 2][b] = xyz.T, sn.T, nd.T
    return tuple(out)


def cloud_gather(scans, offsets, scan_of_cloud, rows, nodes, S, flags=0, noise_sigma=0.0, noise=None):
    """test_cloud_gather_kernel (:688-730): (pc (B,3,N), sn (B,S,N), node (B,3,M)); noise (B, 3, N) f32."""
    B, N = len(scan_of_cloud), rows.shape[1]
    pc, sn_out, nd_out = np.empty((B, 3, N), f32), np.empty((B, S, N), f32), np.empty_like(nodes)
    for c in range(B):
        p = _rows_of(scans, offsets, scan_of_cloud, rows, c)
        xyz, sn = _enu_to_cam(flags, 1.0, p[:, 0:3], p[:, 3:3 + S])
        nd, _ = _enu_to_cam(flags, 1.0, nodes[c].T, None)
        if f32(noise_sigma) != 0:
            n = (noise[c].astype(f64) * f64(f32(noise_sigma))).astype(f32)
            xyz = (xyz.astype(f64) + n.T).astype(f32)
        pc[c], sn_out[c], nd_out[c] = xyz.T, sn.T, nd.T
    return pc, sn_out, nd_out


def gather_candidates(scans, offsets, scan_of_cloud, rows, cand, z_scale=None):
    """pair_gather_kernel (:339-349) -> (2B, n_cand, 3) f32."""
    pts = np.stack([_rows_of(scans, offsets, scan_of_cloud, rows, c)[cand[c], 0:3] for c in range(len(scan_of_cloud))])
    if z_scale is not None:
        pts[:, :, 2] = (pts[:, :, 2].astype(f64) * z_scale.astype(f64)[:, None]).astype(f32)
    return pts

