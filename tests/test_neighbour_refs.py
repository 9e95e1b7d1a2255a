"""The numpy restatements of tests/neighbour_ref.py (used by tests/test_gpu_neighbour_ops.py to check the neighbour-search,
sampling and NMS kernels) against outputs of the reference frozen in tests/golden/, against torch.norm + topk, and
against oracle/.  CPU only."""
import numpy as np
import torch

from oracle import usip_oracle as orc
from tests import neighbour_ref as R
from tests.util_gpu import golden


def ball_query_inputs():
    """The inputs of reference_ops.npz's ball_query entry (tests/test_gpu_ops.py::ball_query_inputs)."""
    rng = np.random.default_rng(1)
    pc = rng.random((8, 3, 4096), dtype=np.float32) * np.float32(8)
    kp = (pc[:, :, :256] + np.float32(0.05) * rng.standard_normal((8, 3, 256), dtype=np.float32)).astype(np.float32)
    return pc, kp


def ball_group_inputs(dense):
    """The inputs of reference_ops.npz's ball_group / ball_group_dense (tests/test_gpu_ops.py::ball_group_inputs)."""
    B, N, M = (16, 16384, 1024) if not dense else (2, 8192, 256)
    rng = np.random.default_rng(3 + dense)
    ext = np.array([40.0, 2.0, 40.0], np.float32).reshape(1, 3, 1) * np.float32(0.08 if dense else 1.0)
    pc = ((rng.random((B, 3, N), dtype=np.float32) * 2 - 1) * ext).astype(np.float32)
    sn = rng.standard_normal((B, 4, N), dtype=np.float32)
    sel = rng.integers(0, N, (B, M))
    kp = (np.take_along_axis(pc, sel[:, None, :], axis=2) + np.float32(0.1) * rng.standard_normal((B, 3, M), dtype=np.float32))
    return pc, sn, kp.astype(np.float32)


def test_ball_query_ref_vs_reference_cuda_golden():
    """The reference's own ball-query kernel on the torch.norm distance matrix (reference_ops.npz)."""
    pc, kp = ball_query_inputs()
    theirs = golden("reference_ops.npz")["ball_query"].astype(np.int32)
    assert np.array_equal(R.ball_query(pc, kp, 1.0, 64), theirs)
    d = np.sqrt(R.sqdist(kp[:, :, :, None].transpose(1, 0, 2, 3), pc[:, :, None, :].transpose(1, 0, 2, 3)))
    assert np.array_equal(R.ball_query_dist(d, 1.0, 64), theirs)
    assert np.array_equal(R.ball_query_dist(d, 1.0, 64), orc.ball_query_dist(d, 1.0, 64))


def test_ball_group_ref_vs_reference_cuda_golden():
    """reference_ops.npz ball_group (every 8th keypoint of the Oxford descriptor shape) and ball_group_dense (dense balls
    with more than K hits); the group is checked against the oracle's indices gathered the same way."""
    g = golden("reference_ops.npz")
    for dense in (False, True):
        pc, sn, kp = ball_group_inputs(dense)
        kp = kp if dense else kp[:, :, ::8].copy()
        idx = R.ball_query(pc, kp, 1.0, 64)
        assert np.array_equal(idx, g["ball_group_dense" if dense else "ball_group"].astype(np.int32)), dense
        assert np.array_equal(idx[:2], orc.ball_query_xyz(pc[:2], kp[:2], 1.0, 64)), dense
        grp = R.group(pc[:2], sn[:2], kp[:2], idx[:2])
        ref = np.concatenate([pc[:2], sn[:2]], 1)[np.arange(2)[:, None, None, None], np.arange(7)[None, :, None, None],
                                                  idx[:2][:, None, :, :]]
        ref[:, :3] -= kp[:2, :, :, None]
        assert np.array_equal(grp, ref)
        assert np.array_equal(R.rows(grp, 8)[:, :7], grp.transpose(0, 2, 3, 1).reshape(-1, 7))


def test_ball_query_ref_edges_vs_oracle():
    """Few hits (cyclic pad), no hit, radius 0 with a coincident point, non-finite points: the oracle's C loop."""
    rng = np.random.default_rng(4)
    B, N, M, K = 2, 700, 30, 16
    pc = rng.uniform(-3, 3, (B, 3, N)).astype(np.float32)
    kp = pc[:, :, :M] + rng.normal(0, 0.2, (B, 3, M)).astype(np.float32)
    kp[:, :, 0] = 50.0
    pc[0, 0, ::13] = np.nan; pc[1, 2, ::17] = np.inf
    for r in (0.0, 0.3, 1.0):
        assert np.array_equal(R.ball_query(pc, kp, r, K), orc.ball_query_xyz(pc, kp, r, K)), r
    kp[:, :, 1] = pc[:, :, 5]
    assert R.ball_query(pc, kp, 0.0, K)[0, 1].tolist() == [5] * K


def test_knn_group_ref_vs_torch_topk():
    """networks.py:556-560: torch.norm over the xyz difference + topk(k, largest=False, sorted=False), compared as sets
    (torch leaves the order unspecified); continuous data, so no ties at the K-th distance."""
    rng = np.random.default_rng(6)
    B, N, M, K = 2, 3000, 40, 64
    pc = rng.normal(size=(B, 3, N)).astype(np.float32)
    kp = rng.normal(size=(B, 3, M)).astype(np.float32)
    ours = R.knn_group_idx(pc, kp, K)
    d = torch.norm(torch.from_numpy(kp).unsqueeze(3) - torch.from_numpy(pc).unsqueeze(2), dim=1)
    _, nn = torch.topk(d, k=K, dim=2, largest=False, sorted=False)
    assert np.array_equal(ours, np.sort(nn.numpy(), axis=2).astype(np.int32))
    oi, _ = orc.knn(kp, pc, K)
    assert np.array_equal(ours, np.sort(oi, axis=2))
    assert np.all(np.diff(ours, axis=2) > 0)


def test_knn_group_ref_ties_and_nonfinite():
    """Ties at the K-th key go lowest index first; NaN and inf distances share the largest key."""
    pc = np.zeros((1, 3, 10), np.float32)
    pc[0, 0] = [3, 1, 2, 2, 2, np.nan, np.inf, 2, 0.5, 9]
    kp = np.zeros((1, 3, 1), np.float32)
    assert R.knn_group_idx(pc, kp, 4)[0, 0].tolist() == [1, 2, 3, 8]
    assert R.knn_group_idx(pc, kp, 9)[0, 0].tolist() == [0, 1, 2, 3, 4, 5, 7, 8, 9]
    assert R.knn_group_idx(pc, kp, 10)[0, 0].tolist() == list(range(10))


def test_fps_ref_vs_reference_golden_and_oracle():
    """fps.npz: the reference's FarthestSampler outputs (float64 nodes) incl. duplicated points and k beyond the
    distinct points."""
    g = golden("fps.npz")
    for name in ("lidar", "dup", "few"):
        pts, k, st = g["pts_" + name], int(g["k_" + name]), int(g["start_" + name])
        idx = R.fps(pts, st, k)
        assert np.array_equal(pts[idx].astype(np.float64), g["nodes_" + name]), name
        assert np.array_equal(idx, orc.fps(pts, st, k)), name
    rng = np.random.default_rng(2)
    pts = rng.uniform(-5, 5, (1500, 3)).astype(np.float32)
    pts[700:800] = pts[0:100]
    for st, k in ((0, 1), (1499, 300), (3, 1500), (10, 1600)):
        assert np.array_equal(R.fps(pts, st, k), orc.fps(pts, st, k)), (st, k)


def test_nms_ref_vs_reference_golden_and_oracle():
    """nms.npz: the reference's own nms() outputs, plus the oracle on finite sigmas."""
    g = golden("nms.npz")
    for name in ("lidar", "dense", "ties", "off"):
        kp, sg, r = g["kp_" + name], g["sigma_" + name], float(g["radius_" + name])
        idx = R.nms(kp, sg, r)
        assert np.array_equal(kp[idx], g["valid_kp_" + name]) and np.array_equal(sg[idx], g["valid_sigma_" + name]), name
        assert np.array_equal(idx, orc.nms(kp, sg, r)), name


def test_nms_ref_nan_sigmas_and_oracle():
    """np.argmin returns the first NaN: every NaN-sigma keypoint is emitted first, in index order, and suppresses its
    neighbours as usual; the finite sigmas follow in (sigma, index) order.  The oracle agrees."""
    rng = np.random.default_rng(8)
    M = 60
    kp = rng.uniform(-4, 4, (M, 3)).astype(np.float32)
    base = rng.uniform(0.1, 2.0, M).astype(np.float32)
    for where in ("first", "middle", "all"):
        sg = base.copy()
        if where == "first":
            sg[:3] = np.nan
        elif where == "middle":
            sg[[20, 31, 45]] = np.nan
        else:
            sg[:] = np.nan
        idx = R.nms(kp, sg, 1.5)
        nan_kept = [i for i in idx if np.isnan(sg[i])]
        assert list(idx[:len(nan_kept)]) == nan_kept == sorted(nan_kept), where
        assert np.isnan(sg[idx[0]]), where
        assert np.array_equal(idx, orc.nms(kp, sg, 1.5)), where
    assert R.nms(kp, sg, 0.005).tolist() == list(range(M))


def nms_rank_before_fix(s):
    """The rank nms_kernel computed before NaN sigmas were ordered: #{j : s[j] < s[i] or (s[j] == s[i] and j < i)}."""
    return [sum(1 for j in range(len(s)) if s[j] < s[i] or (s[j] == s[i] and j < i)) for i in range(len(s))]


def nms_rank(s):
    """nms_kernel's rank: NaN sigmas before every finite one, in index order among themselves, then (sigma, index)."""
    n = [x != x for x in s]
    return [sum(1 for j in range(len(s)) if ((n[j] and j < i) if n[i] else (n[j] or s[j] < s[i] or (s[j] == s[i] and j < i))))
            for i in range(len(s))]


def test_nms_rank_formula_nan_collision():
    """The old rank formula gave every NaN sigma rank 0, the same rank as the smallest finite sigma: slots of order[]
    stayed unwritten and the sweep read indices from uninitialised shared memory.  The kernel's formula is a
    permutation that visits the keypoints in the numpy loop's emission order."""
    s = np.array([0.5, np.nan, 0.2, np.nan], np.float32)
    assert nms_rank_before_fix(s) == [1, 0, 0, 0]
    assert nms_rank(s) == [3, 0, 2, 1]
    rng = np.random.default_rng(0)
    for _ in range(20):
        s = np.round(rng.uniform(0, 3, 40), 1).astype(np.float32)
        s[rng.random(40) < 0.3] = np.nan
        s[rng.random(40) < 0.1] = -0.0
        s[rng.random(40) < 0.05] = np.inf
        rk = nms_rank(s)
        assert sorted(rk) == list(range(40))
        order = np.empty(40, np.int64); order[rk] = np.arange(40)
        kp = np.zeros((40, 3), np.float32); kp[:, 0] = np.arange(40) * 10     # nothing suppresses anything
        assert np.array_equal(order, R.nms(kp, s, 1.0))


def test_cluster_sort_and_som_assign_refs_vs_oracle():
    rng = np.random.default_rng(3)
    B, N, M = 2, 1000, 37
    x = rng.normal(size=(B, 3, N)).astype(np.float32)
    node = rng.normal(size=(B, 3, M)).astype(np.float32)
    node[:, :, 20] = node[:, :, 3]                                   # duplicated node: the first wins
    idx, count = R.som_assign(x, node)
    assert np.array_equal(idx, orc.som_assign(x, node))
    assert not np.any(idx == 20) and count.sum() == B * N
    seg_off, perm, row_seg = R.cluster_sort(idx, M)
    for b in range(B):
        for m in range(M):
            seg = perm[b, seg_off[b, m]:seg_off[b, m + 1]]
            assert np.array_equal(seg, np.flatnonzero(idx[b] == m))
            assert np.all(row_seg[b, seg_off[b, m]:seg_off[b, m + 1]] == b * M + m)
