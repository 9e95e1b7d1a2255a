"""Plain numpy restatements of the index-producing kernels: ball query and ball group, kNN group, farthest point
sampling, radius NMS, the stable cluster sort and the nearest-node assignment.  tests/test_gpu_neighbour_ops.py compares
the CUDA kernels with these bit for bit; tests/test_neighbour_refs.py pins them to the reference's frozen outputs.

Distances are float32 (dx*dx + dy*dy) + dz*dz with every operation rounded (numpy float32 has no FMA, so this is
sqdist_rn bit for bit), and a radius test is float32 np.sqrt(d2) <= r, as torch.norm followed by the reference's
`<= radius` computes it."""
import numpy as np

f32 = np.float32


def sqdist(c, p):
    """c (3,) or (3, M, 1), p (3, N) or (3, 1, N) -> float32 (dx*dx + dy*dy) + dz*dz."""
    c = np.asarray(c, f32); p = np.asarray(p, f32)
    with np.errstate(invalid="ignore", over="ignore"):                   # inf - inf, overflowing squares
        dx, dy, dz = c[0] - p[0], c[1] - p[1], c[2] - p[2]
        return ((dx * dx + dy * dy) + dz * dz).astype(f32)


def _pad(hits, K):
    """ball_query_cuda.cu:22-46: the first K hits; u < K hits repeat cyclically (out[u+i] = out[i % u]); none -> 0."""
    u = min(len(hits), K)
    if u == 0:
        return np.zeros(K, np.int32)
    return np.asarray(hits[:u], np.int32)[np.arange(K) % u]


def ball_query_dist(dist, radius, K):
    """ball_query.forward_cuda_shared_mem (ball_query_cuda.cu:10-49) on a (B, M, N) distance matrix: first K n with
    dist <= radius in index order, cyclic pad, 0 when nothing hits.  NaN distances and a NaN radius never hit."""
    B, M, N = dist.shape
    hit = dist <= f32(radius)
    out = np.empty((B, M, K), np.int32)
    for b in range(B):
        for m in range(M):
            out[b, m] = _pad(np.flatnonzero(hit[b, m]), K)
    return out


def ball_query(xyz, centers, radius, K):
    """models/networks.py:355-359: torch.norm(node - pc) then ball_query.  xyz (B,3,N), centers (B,3,M) -> (B,M,K)."""
    B, M = xyz.shape[0], centers.shape[2]
    out = np.empty((B, M, K), np.int32)
    r = f32(radius)
    for b in range(B):
        d = np.sqrt(sqdist(centers[b][:, :, None], xyz[b][:, None, :]))      # (M, N)
        hit = d <= r
        for m in range(M):
            out[b, m] = _pad(np.flatnonzero(hit[m]), K)
    return out


def group(xyz, feat, centers, idx):
    """networks.py:361-373 (ball) and :562-565 (kNN): x_aug = cat(xyz, feat) gathered at idx, centre subtracted from the
    xyz channels.  -> (B, 3+S, M, K) float32."""
    x_aug = xyz if feat is None or feat.shape[1] == 0 else np.concatenate([xyz, feat], 1)
    B, C, _ = x_aug.shape
    _, M, K = idx.shape
    g = np.take_along_axis(x_aug, np.broadcast_to(idx.reshape(B, 1, M * K).astype(np.int64), (B, C, M * K)), 2)
    g = g.reshape(B, C, M, K).copy()
    g[:, :3] = g[:, :3] - centers[:, :, :, None]
    return g.astype(f32)


def rows(grp, ld):
    """The group as point-major rows [B*M*K, ld]: channels 0..C-1, zeros after."""
    B, C, M, K = grp.shape
    out = np.zeros((B * M * K, ld), f32)
    out[:, :C] = grp.transpose(0, 2, 3, 1).reshape(B * M * K, C)
    return out


def knn_group_idx(xyz, centers, K):
    """networks.py:556-560: torch.norm + topk(K, largest=False).  The K smallest float32 d^2 (sqrt is monotone), ties at
    the K-th key taken lowest index first, NaN and inf d^2 given the same (largest) key; returned in ascending index."""
    B, M = xyz.shape[0], centers.shape[2]
    out = np.empty((B, M, K), np.int32)
    for b in range(B):
        d2 = sqdist(centers[b][:, :, None], xyz[b][:, None, :])
        key = np.where(d2 <= np.finfo(f32).max, d2, np.inf).astype(f32)
        for m in range(M):
            sel = np.lexsort((np.arange(key.shape[1]), key[m]))[:K]
            out[b, m] = np.sort(sel)
    return out


def fps(pts, start, k):
    """data/kitti_detector_loader.py:68-83 (FarthestSampler.sample) returning indices: float64 running minima of
    ((p0 - pts)**2).sum(axis=1) with p0 a float64 copy of a float32 point, np.minimum, first arg-max (np.argmax).
    Points must be finite: np.minimum propagates NaN, the kernel keeps the smaller value."""
    pts = np.asarray(pts, f32)
    out = np.empty(k, np.int32)
    sel = int(start)
    out[0] = sel
    dist = ((pts[sel].astype(np.float64) - pts) ** 2).sum(axis=1)
    for i in range(1, k):
        sel = int(np.argmax(dist))
        out[i] = sel
        dist = np.minimum(dist, ((pts[sel].astype(np.float64) - pts) ** 2).sum(axis=1))
    return out


def nms(kp, sigma, radius):
    """evaluation/save_keypoints.py:180-216 nms(), tracking indices: kp (M,3) f32, sigma (M,) f32 -> original indices of
    the kept keypoints in emission order.  Repeated np.argmin (the first NaN when there is one) and float32
    np.linalg.norm(...) > radius, literally as the reference loop does it."""
    if radius < 0.01:
        return np.arange(kp.shape[0], dtype=np.int32)
    keep = []
    rem = np.arange(kp.shape[0])
    k, s = kp, sigma
    while k.shape[0] > 0:
        i = np.argmin(s, axis=0)
        keep.append(rem[i])
        mask = np.linalg.norm(k[i:i + 1, :] - k, axis=1, keepdims=False) > radius
        k, s, rem = k[mask, ...], s[mask], rem[mask]
    return np.asarray(keep, np.int32)


def cluster_sort(min_idx, M):
    """usip_cluster_sort: stable argsort of every cloud's node ids plus bincount.  min_idx (B,N) ->
    seg_off (B,M+1), perm (B,N), row_seg (B,N)."""
    B, N = min_idx.shape
    seg_off = np.zeros((B, M + 1), np.int32)
    perm = np.empty((B, N), np.int32)
    row_seg = np.empty((B, N), np.int32)
    for b in range(B):
        p = np.argsort(min_idx[b], kind="stable")
        perm[b] = p
        seg_off[b, 1:] = np.cumsum(np.bincount(min_idx[b], minlength=M))
        row_seg[b] = b * M + min_idx[b][p]
    return seg_off, perm, row_seg


def som_assign(xyz, node):
    """util/som.py:35-39 with k = 1: nearest node by float32 d^2, the first arg-min on ties.  -> min_idx (B,N), count (B,M)."""
    B, N = xyz.shape[0], xyz.shape[2]
    M = node.shape[2]
    idx = np.empty((B, N), np.int32)
    for b in range(B):
        idx[b] = np.argmin(sqdist(node[b][:, :, None], xyz[b][:, None, :]), axis=0)
    count = np.stack([np.bincount(idx[b], minlength=M) for b in range(B)]).astype(np.int32)
    return idx, count
