"""-m gpu: the neighbour-search, sampling and NMS kernels against the numpy restatements of tests/neighbour_ref.py, bit
for bit, at their dispatch edges: ball group (bucket grid and in-order scan), kNN group, FPS, NMS, cluster sort, the
brute-force nearest-node assignment and the distance-matrix ball query.  Output buffers are pre-filled with sentinels, so
a slot a kernel forgets to write (a pad index, a zero row padding) shows up."""
import numpy as np
import pytest
import torch

from tests import neighbour_ref as R
from tests.util_gpu import cu, dev

pytestmark = pytest.mark.gpu

i32, f32 = torch.int32, torch.float32


def _lib():
    from usip_b200 import _lib as L
    return L.load()


def _call(name, *args):
    from usip_b200 import _lib as L
    from usip_b200.ops import _stream
    L.check(getattr(_lib(), name)(*args, _stream()), name)


def P(t, off=0):
    import ctypes
    return None if t is None else ctypes.c_void_p(t.data_ptr() + 4 * off)


def same_bits(got, ref, what=""):
    """Equal bit patterns (so -0 != +0), except that any NaN matches any NaN."""
    got = np.ascontiguousarray(got); ref = np.ascontiguousarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), what
    bad = got.view(np.int32)[~nan] != ref.view(np.int32)[~nan]
    assert not bad.any(), (what, int(bad.sum()))


# ------------------------------------------------------------------------------------------ ball group
BX_MAX_CELLS = 128 * 128


def _bx_zero_bytes(B):
    """Size of the scratch's counter region (fill counts, overflow counts, arrival counters): BxScratch in ballgroup.cu."""
    a = lambda x: (x + 255) & ~255
    return a(4 * B * BX_MAX_CELLS) + a(4 * B) + a(4 * B)


def fresh_scratch(B, S, N, M, K):
    nbytes = int(_lib().usip_ball_group_scratch_bytes(B, S, N, M, K))
    buf = torch.empty((nbytes,), dtype=torch.uint8, device=dev())
    _call("usip_ball_group_scratch_init", P(buf), nbytes, B)
    return buf, nbytes


def ball_group_abi(pc, sn, kp, r, K, ld=8, path="grid", group=True, rows=True, rows_off=0, scratch=None):
    """usip_ball_group_f32 through the C ABI.  path "grid": the cached per-stream scratch of ops.ball_group (or the given
    one); "brute": scratch = NULL, the in-order scan kernel.  rows_off shifts out_rows by that many floats."""
    from usip_b200 import ops
    B, _, N = pc.shape
    M, S = kp.shape[2], 0 if sn is None else sn.shape[1]
    idx = torch.full((B, M, K), -7, dtype=i32, device=dev())
    grp = torch.full((B, 3 + S, M, K), float("nan"), dtype=f32, device=dev()) if group else None
    nrow = B * M * K * ld
    rbuf = torch.full((nrow + rows_off + 4,), float("nan"), dtype=f32, device=dev()) if rows else None
    buf, nbytes = None, 0
    if path == "grid":
        buf, nbytes = scratch if scratch is not None else ops._ball_group_scratch(_lib(), dev(), B, S, N, M, K)
    _call("usip_ball_group_f32", P(pc), P(sn) if S else None, P(kp), float(r), P(idx), P(grp), P(rbuf, rows_off),
          ld if rows else 0, P(buf), int(nbytes), B, S, N, M, K)
    out_rows = None
    if rows:
        h = rbuf.cpu().numpy()
        assert np.isnan(h[:rows_off]).all() and np.isnan(h[rows_off + nrow:]).all(), "wrote outside out_rows"
        out_rows = h[rows_off:rows_off + nrow].reshape(B * M * K, ld)
    return idx.cpu().numpy(), None if grp is None else grp.cpu().numpy(), out_rows


def check_ball_group(pc, sn, kp, r, K, ld=8, **kw):
    """Both paths against the restatement, and against each other."""
    ri = R.ball_query(pc, kp, r, K)
    rg = R.group(pc, sn, kp, ri)
    rr = R.rows(rg, ld)
    outs = []
    for path in ("grid", "brute"):
        idx, grp, rows = ball_group_abi(cu(pc), None if sn is None else cu(sn), cu(kp), r, K, ld, path=path, **kw)
        assert np.array_equal(idx, ri), (path, int((idx != ri).sum()))
        if grp is not None:
            same_bits(grp, rg, path + " group")
        if rows is not None:
            same_bits(rows, rr, path + " rows")
        outs.append((idx, grp, rows))
    (ig, gg, rg_), (ib, gb, rb) = outs
    assert np.array_equal(ig, ib)
    if gg is not None:
        same_bits(gg, gb, "grid vs brute group")
    if rg_ is not None:
        same_bits(rg_, rb, "grid vs brute rows")
    return ri


def lidar_cloud(rng, B, N, M, S, ext=10.0):
    pc = np.stack([rng.uniform(-ext, ext, (B, N)), rng.uniform(-0.5, 0.5, (B, N)), rng.uniform(-ext, ext, (B, N))], 1)
    pc = pc.astype(np.float32)
    sn = rng.normal(size=(B, S, N)).astype(np.float32)
    kp = (pc[:, :, rng.integers(0, N, M)] + rng.normal(0, 0.2, (B, 3, M))).astype(np.float32)
    return pc, sn, kp


def stacked_cloud(rng, B=2, N=4096, M=45):
    """Five stacks of 20 points each inside one bucket, a centre on every stack: the bucket fills its 8 slots and the
    other records go to the cloud's overflow list.  Every ball holds well under 64 points."""
    pc, sn, kp = lidar_cloud(rng, B, N, M, 4)
    for s in range(5):
        at = np.array([-8 + 4 * s, 0.0, 3.0 - s], np.float32)
        sl = slice(100 + 200 * s, 120 + 200 * s)                     # spread through the index range
        pc[:, :, sl] = at[None, :, None] + rng.uniform(-1e-3, 1e-3, (B, 3, 20)).astype(np.float32)
        kp[:, :, 7 * s] = at + np.float32(0.01)
    return pc, sn, kp


def flooded_cloud(rng, B=2, N=8192, M=40):
    """5000 points in one cell, farther than the radius from every centre but inside the bucket grid: the overflow list
    takes more than 4096 records and the whole cloud goes to the in-order scan."""
    pc, sn, kp = lidar_cloud(rng, B, N, M, 4)
    flood = np.array([0.0, 0.0, 0.0], np.float32)
    pc[:, :, 1000:6000] = flood[None, :, None] + rng.uniform(-1e-3, 1e-3, (B, 3, 5000)).astype(np.float32)
    far = np.sqrt(((kp - flood[None, :, None]) ** 2).sum(1)) < 2.0
    kp[:, 0][far] += 5.0                                              # keep every ball off the flood
    kp[:, 0, 0] = -9.0; kp[:, 0, 1] = 9.0                             # the grid spans the flood
    return pc, sn, kp


@pytest.mark.parametrize("S", [0, 1, 2, 3, 4, 5])
def test_ball_group_channels(S):
    """S = 1, 2, 3 and 4 on the bucket grid, S > 4 on ball_group_brute_kernel; M % 8 != 0."""
    rng = np.random.default_rng(40 + S)
    pc, sn, kp = lidar_cloud(rng, 2, 3000, 37, S)
    check_ball_group(pc, sn if S else None, kp, 1.0, 32, ld=8)


BALL_CASES = ["K_over_64", "bucket_overflow", "overflow_flood", "ld7", "ld12", "rows_misaligned", "no_group", "idx_only",
              "nonfinite", "all_centres_nonfinite", "radius_zero", "radius_negative", "radius_nan", "radius_inf",
              "small_radius_large_extent"]


@pytest.mark.parametrize("case", BALL_CASES)
def test_ball_group_edges(case):
    rng = np.random.default_rng(BALL_CASES.index(case) + 100)
    r, K, ld, kw = 1.0, 32, 8, {}
    pc, sn, kp = lidar_cloud(rng, 2, 3000, 29, 4)
    if case == "K_over_64":
        # in-order scan with K > 64: balls of 0, 1, a few and more than K hits
        K, r = 100, 0.8
        kp[:, :, 0] = 50.0                                            # nothing within r
        pc[:, :, 2000] = np.array([30, 0, 30], np.float32)            # an isolated point: one hit
        kp[:, :, 1] = pc[:, :, 2000]
        pc[:, :, :150] = rng.uniform(-0.3, 0.3, (2, 3, 150)).astype(np.float32)
        kp[:, :, 2] = 0.0                                             # more than K hits
    elif case == "bucket_overflow":
        pc, sn, kp = stacked_cloud(rng)
        r = 0.5
    elif case == "overflow_flood":
        pc, sn, kp = flooded_cloud(rng)
        r = 0.5
    elif case == "ld7":
        ld = 7
    elif case == "ld12":
        sn = sn[:, :2].copy(); ld = 12
    elif case == "rows_misaligned":
        kw = dict(rows_off=1)                                         # out_rows 4 bytes off 16: the in-order scan
    elif case == "no_group":
        kw = dict(group=False)
    elif case == "idx_only":
        kw = dict(group=False, rows=False)
    elif case == "nonfinite":
        pc[0, 0, ::11] = np.nan; pc[1, 2, ::13] = np.inf; pc[1, 1, 5] = -np.inf
        kp[0, 1, 3] = np.nan; kp[1, 0, 4] = np.inf; kp[1, :, 6] = -np.inf
    elif case == "all_centres_nonfinite":
        kp[0] = np.nan; kp[1, 0] = np.inf
    elif case == "radius_zero":
        kp[:, :, :10] = pc[:, :, 100:110]                             # exact coincidences hit at r = 0
        kp[:, :, 3] = pc[:, :, 50]; pc[:, :, 2000] = pc[:, :, 50]     # two coincident points
        r = 0.0
    elif case == "radius_negative":
        r = -1.0
    elif case == "radius_nan":
        r = float("nan")
    elif case == "radius_inf":
        pc[0, 0, ::17] = np.nan                                        # NaN distances never hit, even at r = inf
        r, K = float("inf"), 40
    elif case == "small_radius_large_extent":
        pc, sn, kp = lidar_cloud(rng, 2, 6000, 33, 4, ext=500.0)      # 2000 radii across: the cell grows 1.26x per step
        kp[:, :, :20] = pc[:, :, 10:30] + np.float32(0.1)
        r = 0.5
    ri = check_ball_group(pc, sn, kp, r, K, ld, **kw)
    if case in ("K_over_64", "bucket_overflow"):
        u = np.array([len(set(row.tolist())) for row in ri.reshape(-1, K)])
        assert (u > 8).any() and ((u > 1) & (u < K)).any()


def test_ball_group_scratch_counters_cleared():
    """Two clouds in a row through the cached scratch (one with a bucket overflow, one with a flooded overflow list):
    afterwards the counter region is all zero again, and a third call equals the same call on fresh scratch."""
    from usip_b200 import ops
    rng = np.random.default_rng(7)
    B, K, r = 2, 32, 0.5
    a = stacked_cloud(rng, B, 8192, 40)
    b = flooded_cloud(rng, B, 8192, 40)
    c = stacked_cloud(rng, B, 8192, 40)
    for pc, sn, kp in (a, b):
        idx, _, _ = ball_group_abi(cu(pc), cu(sn), cu(kp), r, K)
        assert np.array_equal(idx, R.ball_query(pc, kp, r, K))
    torch.cuda.synchronize()
    key = (dev().index, torch.cuda.current_stream().cuda_stream, B)
    buf, nbytes = ops._BG_SCRATCH[key]
    zb = _bx_zero_bytes(B)
    assert nbytes >= zb
    assert int(torch.count_nonzero(buf[:zb])) == 0
    pc, sn, kp = c
    got = ball_group_abi(cu(pc), cu(sn), cu(kp), r, K)
    ref = ball_group_abi(cu(pc), cu(sn), cu(kp), r, K, scratch=fresh_scratch(B, 4, 8192, 40, K))
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[0], R.ball_query(pc, kp, r, K))
    same_bits(got[1], ref[1]); same_bits(got[2], ref[2])


# ------------------------------------------------------------------------------------------ kNN group
def knn_group_abi(pc, sn, kp, K, ld):
    B, _, N = pc.shape
    M, S = kp.shape[2], 0 if sn is None else sn.shape[1]
    idx = torch.full((B, M, K), -7, dtype=i32, device=dev())
    grp = torch.full((B, 3 + S, M, K), float("nan"), dtype=f32, device=dev())
    rows = torch.full((B * M * K, ld), float("nan"), dtype=f32, device=dev())
    pc_, sn_, kp_ = cu(pc), cu(sn) if S else None, cu(kp)                 # held until the call has been enqueued
    _call("usip_knn_group_f32", P(pc_), P(sn_), P(kp_), P(idx), P(grp), P(rows), ld, B, S, N, M, K)
    return idx.cpu().numpy(), grp.cpu().numpy(), rows.cpu().numpy()


KNN_CASES = ["tail_tile", "K_eq_N", "K1", "low_bytes", "kth_tie", "S5_ld10", "nonfinite"]


@pytest.mark.parametrize("case", KNN_CASES)
def test_knn_group(case):
    rng = np.random.default_rng(KNN_CASES.index(case) + 200)
    B, N, M, K, S, ld = 2, 1000, 13, 64, 4, 8
    if case == "tail_tile":
        N, M = 5000, 29                                               # 2048-point tiles, the last one partial
    elif case == "K_eq_N":
        N, K, S, ld = 200, 200, 0, 3
    elif case == "K1":
        K = 1
    elif case == "S5_ld10":
        S, ld = 5, 10
    pc = rng.normal(size=(B, 3, N)).astype(np.float32)
    sn = rng.normal(size=(B, S, N)).astype(np.float32)
    kp = rng.normal(size=(B, 3, M)).astype(np.float32)
    if case == "low_bytes":
        # d^2 of consecutive floats just above 1: the same top bytes, so every radix pass decides
        pc = (rng.uniform(5, 9, (B, 3, N)) * rng.choice([-1, 1], (B, 3, N))).astype(np.float32)
        x = (np.float32(1) + np.arange(300, dtype=np.float32) * np.float32(2.0 ** -23)).astype(np.float32)
        perm = rng.permutation(N)[:300]
        pc[:, :, perm] = 0.0
        pc[:, 0, perm] = x
        kp[:] = 0.0
        K = 150
    elif case == "kth_tie":
        # 50 copies of one point at indices 0..49, 30 nearer points after them: K = 64 takes 34 of the ties, lowest first
        pc = (rng.uniform(5, 9, (B, 3, N)) * rng.choice([-1, 1], (B, 3, N))).astype(np.float32)
        pc[:, :, :50] = np.array([2, 0, 0], np.float32)[:, None]
        pc[:, :, 50:80] = rng.uniform(-0.5, 0.5, (B, 3, 30)).astype(np.float32)
        kp[:] = 0.0
    elif case == "nonfinite":
        N, K = 300, 290
        pc, sn = pc[:, :, :N].copy(), sn[:, :, :N].copy()
        pc[0, 0, 10:20] = np.nan; pc[0, 1, 40:45] = np.inf; pc[1, 2, 100:110] = -np.inf; pc[1, 0, 200] = np.nan
    ri = R.knn_group_idx(pc, kp, K)
    rg = R.group(pc, sn if S else None, kp, ri)
    idx, grp, rows = knn_group_abi(pc, sn if S else None, kp, K, ld)
    assert np.array_equal(idx, ri), int((idx != ri).sum())
    same_bits(grp, rg, "group")
    same_bits(rows, R.rows(rg, ld), "rows")
    if case == "kth_tie":
        assert idx[0, 0].tolist() == list(range(34)) + list(range(50, 80))


# ------------------------------------------------------------------------------------------ FPS
FPS_CASES = [("Ns1_k1", 1, 1), ("Ns1_k3", 1, 3), ("Ns8192", 8192, 300), ("Ns1000_k_eq_Ns", 1000, 1000),
             ("k_gt_Ns", 700, 750), ("k1", 3000, 1), ("dup", 2048, 700), ("dup8192", 8192, 200)]


@pytest.mark.parametrize("case,Ns,k", FPS_CASES, ids=[c[0] for c in FPS_CASES])
def test_fps(case, Ns, k):
    from usip_b200 import ops
    rng = np.random.default_rng(Ns + k)
    B = 3
    pts = (rng.uniform(-20, 20, (B, Ns, 3)) * np.array([1, 0.1, 1])).astype(np.float32)
    if case == "dup":
        pts[:, 512:1024] = pts[:, 0:512]                              # ties across warps (thread t and t + 512)
        pts[:, 1024:2048] = pts[:, 0:1024]                            # and across a thread's points
    elif case == "dup8192":
        pts[:, 4096:] = pts[:, :4096]
    start = np.array([0, Ns - 1, rng.integers(0, Ns)], np.int32)
    idx, nodes = ops.fps(cu(pts), cu(start), k)
    idx, nodes = idx.cpu().numpy(), nodes.cpu().numpy()
    for b in range(B):
        ref = R.fps(pts[b], start[b], k)
        assert np.array_equal(idx[b], ref), (b, int((idx[b] != ref).sum()))
        assert np.array_equal(nodes[b], pts[b][ref].T)


def test_fps_refuses_more_than_8192_points():
    from usip_b200 import ops
    with pytest.raises(RuntimeError):
        ops.fps(torch.zeros((1, 8193, 3), device=dev()), torch.zeros(1, dtype=i32, device=dev()), 4)


# ------------------------------------------------------------------------------------------ NMS
NMS_CASES = ["M3000", "M8533", "distance_equals_radius", "radius_0.01", "radius_below_0.01", "signed_zero_inf_sigmas",
             "nan_keypoints", "nan_sigma_first", "nan_sigma_middle", "nan_sigma_all"]


@pytest.mark.parametrize("case", NMS_CASES)
def test_nms(case):
    from usip_b200 import ops
    rng = np.random.default_rng(NMS_CASES.index(case) + 300)
    B, M, r = 3, 700, 1.5
    if case == "M3000":
        M = 3000
    elif case == "M8533":
        M = 8533                                                      # 6 * 4 * M bytes: the largest M that fits
    kp = (rng.uniform(-20, 20, (B, 3, M)) * np.array([1, 0.1, 1]).reshape(1, 3, 1)).astype(np.float32)
    sg = rng.uniform(0.01, 2.0, (B, M)).astype(np.float32)
    if case == "distance_equals_radius":
        # pairs exactly r apart (suppressed: the reference keeps only `> r`) and pairs one ulp beyond (kept)
        r = 3.0
        kp = np.zeros((B, 3, M), np.float32)
        kp[:, 0] = (np.arange(M) // 2 * 20).astype(np.float32)
        kp[:, 2, 1::2] = 3.0
        kp[:, 2, 3::4] = np.nextafter(np.float32(3.0), np.float32(4.0))
        sg = np.tile(np.arange(M, dtype=np.float32), (B, 1))
    elif case == "radius_0.01":
        r = 0.01
        kp = kp * np.float32(0.0005)
    elif case == "radius_below_0.01":
        r = float(np.nextafter(np.float32(0.01), np.float32(0)))      # pass-through, input order
    elif case == "signed_zero_inf_sigmas":
        sg[:, ::5] = 0.0; sg[:, 1::5] = -0.0; sg[:, 2::9] = np.inf; sg[:, 3::11] = -np.inf
    elif case == "nan_keypoints":
        kp[0, 0, ::7] = np.nan; kp[1, :, 3] = np.nan; kp[2, 2, 0] = np.nan
        sg[2, 0] = 0.0                                                # a NaN keypoint first: it suppresses everything
    elif case == "nan_sigma_first":
        sg[:, :4] = np.nan
    elif case == "nan_sigma_middle":
        sg[:, [100, 350, 351, 600]] = np.nan
    elif case == "nan_sigma_all":
        sg[:] = np.nan
    idx, cnt = ops.nms(cu(kp), cu(sg), r)
    idx, cnt = idx.cpu().numpy(), cnt.cpu().numpy()
    for b in range(B):
        ref = R.nms(kp[b].T.copy(), sg[b], r)
        assert cnt[b] == len(ref), (b, int(cnt[b]), len(ref))
        assert np.array_equal(idx[b, :cnt[b]], ref), b
        assert np.all(idx[b, cnt[b]:] == -1), b
    if case == "distance_equals_radius":
        assert cnt[0] == 3 * M // 4
    if case == "radius_below_0.01":
        assert np.all(cnt == M)
    if case == "radius_0.01":
        assert np.all(cnt < M)


def test_nms_refuses_m_above_shared_memory():
    from usip_b200 import ops
    with pytest.raises(RuntimeError):
        ops.nms(torch.zeros((1, 3, 8534), device=dev()), torch.zeros((1, 8534), device=dev()), 1.0)


# ------------------------------------------------------------------------------------------ cluster sort
SORT_CASES = [("M5000", 2, 20000, 5000), ("M4000", 2, 9000, 4000), ("N_tail", 3, 300, 64), ("single_node", 2, 1000, 300)]


@pytest.mark.parametrize("case,B,N,M", SORT_CASES, ids=[c[0] for c in SORT_CASES])
def test_cluster_sort(case, B, N, M):
    """M > 4096: the chunk-rank kernels; 3072 < M <= 4096: the warp-match kernels above 48 KB of shared memory.  perm and
    row_seg get two clouds' worth of slack that must stay untouched."""
    rng = np.random.default_rng(N + M)
    min_idx = rng.integers(0, M, (B, N)).astype(np.int32)
    if case == "single_node":
        min_idx[:] = 7
    elif case == "M5000":
        min_idx[:, ::3] = rng.integers(0, 40, (B, len(range(0, N, 3))))   # long runs of one key inside a chunk
    seg_off = torch.full((B, M + 1), -7, dtype=i32, device=dev())
    perm = torch.full(((B + 2) * N,), -7, dtype=i32, device=dev())
    row_seg = torch.full(((B + 2) * N,), -7, dtype=i32, device=dev())
    scratch = torch.empty((B * ((N + 255) // 256) * M,), dtype=i32, device=dev())
    mi = cu(min_idx)
    _call("usip_cluster_sort", P(mi), P(seg_off), P(perm), P(row_seg), P(scratch), B, N, M)
    rs, rp, rr = R.cluster_sort(min_idx, M)
    perm, row_seg = perm.cpu().numpy(), row_seg.cpu().numpy()
    assert np.all(perm[B * N:] == -7) and np.all(row_seg[B * N:] == -7), "wrote past perm / row_seg"
    assert np.array_equal(seg_off.cpu().numpy(), rs)
    assert np.array_equal(perm[:B * N].reshape(B, N), rp)
    assert np.array_equal(row_seg[:B * N].reshape(B, N), rr)


# ------------------------------------------------------------------------------------------ nearest node (brute force)
SOM_CASES = [("M2000", 2000), ("M10", 10), ("chunk_tie", 1500)]


@pytest.mark.parametrize("case,M", SOM_CASES, ids=[c[0] for c in SOM_CASES])
def test_som_assign_brute(case, M):
    """usip_som_assign_f32 steps through the nodes 1024 at a time; an exact tie between node 50 (first chunk) and node
    1100 (second chunk) goes to node 50."""
    from usip_b200 import ops
    rng = np.random.default_rng(M)
    B, N = 2, 3000
    x = rng.normal(size=(B, 3, N)).astype(np.float32)
    node = rng.normal(size=(B, 3, M)).astype(np.float32)
    if case == "chunk_tie":
        node[:, :, 1100] = node[:, :, 50]
        x[:, :, :200] = node[:, :, 50:51] + rng.normal(0, 1e-3, (B, 3, 200)).astype(np.float32)
    idx, count = ops.som_assign(cu(x), cu(node), method="brute")
    ri, rc = R.som_assign(x, node)
    assert np.array_equal(idx.cpu().numpy(), ri)
    assert np.array_equal(count.cpu().numpy(), rc)
    if case == "chunk_tie":
        assert (ri[:, :200] == 50).mean() > 0.9


# ------------------------------------------------------------------------------------------ ball query on distances
BQ_CASES = [("N300", 300, 16, 0.9), ("K_gt_N", 300, 400, 0.9), ("nonfinite", 300, 64, 0.9),
            ("nonfinite_radius_inf", 300, 64, float("inf")), ("radius_nan", 300, 16, float("nan")),
            ("radius_negative", 300, 16, -0.5)]


@pytest.mark.parametrize("case,N,K,r", BQ_CASES, ids=[c[0] for c in BQ_CASES])
def test_ball_query_dist(case, N, K, r):
    rng = np.random.default_rng(N + K)
    B, M = 2, 21
    dist = np.abs(rng.normal(size=(B, M, N))).astype(np.float32)
    dist[0, 0] = 100.0; dist[0, 1, :3] = 0.0; dist[0, 2] = 0.0
    if case.startswith("nonfinite"):
        dist[:, :, ::7] = np.nan; dist[:, :, 3::11] = np.inf; dist[1, 4] = np.nan
    out = torch.full((B, M, K), -7, dtype=i32, device=dev())
    d = cu(dist)
    _call("usip_ball_query_dist_f32", P(d), float(r), P(out), B, M, N, K)
    assert np.array_equal(out.cpu().numpy(), R.ball_query_dist(dist, r, K))
