"""The handcrafted baselines on the GPU (csrc/handcrafted.cu, usip_b200.evaluation.handcrafted) against the numpy
restatement (tests/handcrafted_ref.py): neighbour counts exactly, eigenvalues and responses to 1e-9 of their scale,
keypoint flags exactly wherever the decision margin exceeds 1e-7, the selection exactly, bitwise determinism, the
refusals, and the evaluators end to end."""
import os

import numpy as np
import pytest
import torch

from tests import handcrafted_ref as H
from tests.rep_ref import repeatability_ref
from tests.util_gpu import dev, make_opt
from usip_b200 import ops
from usip_b200._lib import UsipB200Error
from usip_b200.evaluation import indoor_test_loader as itl
from usip_b200.evaluation import kitti_test_loader as ktl
from usip_b200.evaluation import registration as reg
from usip_b200.evaluation import repeatability as rep
from usip_b200.evaluation.handcrafted import Harris3DDetector, IssDetector, RandomDetector

pytestmark = pytest.mark.gpu

MARGIN = 1e-7


# ----------------------------------------------------------------------------------------------- fixtures
def _box_surface(rng, n, lo, hi):
    """n points on the surface of the box [lo, hi] (faces, edges and corners), face chosen by area."""
    e = hi - lo
    areas = np.array([e[1] * e[2], e[0] * e[2], e[0] * e[1]] * 2)
    face = rng.choice(6, n, p=areas / areas.sum())
    p = lo + rng.uniform(0, 1, (n, 3)) * e
    ax = face % 3
    p[np.arange(n), ax] = np.where(face < 3, lo[ax], hi[ax])
    return p


def structured_cloud(N, extent, seed, blob=0):
    """Planes (a ground plane and box walls), edges and corners (boxes), isotropic noise and a few exact duplicates,
    scaled to `extent` metres; `blob` points packed in a ball of extent/100 give neighbourhoods of that size."""
    rng = np.random.default_rng(seed)
    n_ground, n_noise, n_dup = N // 3, N // 10, min(8, N // 4)
    n_box = N - n_ground - n_noise - n_dup - blob
    ground = np.c_[rng.uniform(-0.5, 0.5, (n_ground, 2)), np.zeros(n_ground)]
    boxes = []
    for k in range(6):
        lo = np.r_[rng.uniform(-0.45, 0.3, 2), 0.0]
        boxes.append(_box_surface(rng, n_box // 6 + (k < n_box % 6), lo, lo + rng.uniform(0.05, 0.15, 3)))
    noise = rng.uniform([-0.5, -0.5, 0], [0.5, 0.5, 0.2], (n_noise, 3))
    ball = rng.normal(0, 1, (blob, 3))
    ball = 0.005 * ball / np.maximum(np.linalg.norm(ball, axis=1, keepdims=True), 1) + [0.1, 0.1, 0.05]
    P = np.concatenate([ground] + boxes + [noise, ball])
    P = (P + rng.normal(0, 1e-4, P.shape)) * extent        # sensor noise: no plane is exact to the last bit
    P = P.astype(np.float32)
    P = np.concatenate([P, P[rng.choice(len(P), n_dup, replace=False)]]) if len(P) else P
    return P[rng.permutation(len(P))][:N] if N > 0 else P


def tiny_cloud(N, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (N, 3)).astype(np.float32)


# case: (clouds (B, N, 3), ISS radii (rs, rn), Harris radius)
def _case(name):
    if name == "n1":
        return np.zeros((1, 1, 3), np.float32), (1.0, 1.0), 1.0
    if name == "sub_warp":
        return np.stack([tiny_cloud(20, 1), tiny_cloud(20, 2) * 3]), (1.0, 0.8), 1.2
    if name == "kitti":                              # KITTI shape and radii; cloud 0 holds a 2200-point neighbourhood
        return np.stack([structured_cloud(16384, 80.0, 3, blob=2200), structured_cloud(16384, 40.0, 4)]), (2.0, 2.0), 1.0
    if name == "indoor":                             # 10240 points, indoor radii, extents 4 m and 40 m
        return np.stack([structured_cloud(10240, 4.0, 5), structured_cloud(10240, 40.0, 6)]), (0.15, 0.1), 0.1
    if name == "capped":                             # two far outliers: 64 cells per axis, the cloud in a few cells
        P = structured_cloud(4096, 8.0, 7)
        P[:2] = [[-5e3, -5e3, 0], [5e3, 5e3, 100]]
        return P[None], (0.5, 0.5), 0.4
    if name == "nan_rows":
        P = structured_cloud(3000, 6.0, 8)
        P[[3, 70, 2999]] = [[np.nan, 0, 0], [0, np.inf, 0], [1, 1, -np.inf]]
        return P[None], (0.4, 0.4), 0.3
    raise KeyError(name)


CASES = ["n1", "sub_warp", "kitti", "indoor", "capped", "nan_rows"]


def _pc(clouds):
    return torch.from_numpy(np.ascontiguousarray(clouds.transpose(0, 2, 1))).to(dev())


def _near(excl_pt, ptr, idx):
    """Rows with an excluded point in their neighbourhood."""
    rows = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    out = np.zeros(len(ptr) - 1, bool)
    np.logical_or.at(out, rows, excl_pt[idx])
    return out


def _flags_equal(got, ref, excluded, what):
    assert excluded.mean() < 0.01, (what, excluded.mean())
    bad = np.flatnonzero((got != ref) & ~excluded)
    assert len(bad) == 0, (what, bad[:10], got[bad[:10]], ref[bad[:10]])


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("case", CASES)
def test_iss_matches_restatement(case):
    clouds, (rs, rn), _ = _case(case)
    g21, g32, mn = 0.975, 0.975, 5
    grid = ops.hc_grid(_pc(clouds))
    sal, cnt, eig = ops.iss_saliency(grid, rs, g21, g32, mn, want_eig=True)
    flag, cnt_n = ops.hc_nonmax(grid, sal, rn, 0.0, True, mn)
    sal, cnt, eig, flag, cnt_n = (t.cpu().numpy() for t in (sal, cnt, eig, flag, cnt_n))
    big = 0
    for b, P in enumerate(clouds):
        nb_s = H.neighbours(P, rs)
        nb_n = H.neighbours(P, rn)
        r_sal, r_cnt, r_eig = H.iss_saliency(P, rs, g21, g32, mn, nb=nb_s)
        np.testing.assert_array_equal(cnt[b], r_cnt)
        big = max(big, int(r_cnt.max()))
        scale = np.abs(r_eig[:, :1])
        assert (np.abs(eig[b] - r_eig) <= 1e-9 * scale + 1e-300).all()
        assert (np.abs(sal[b] - r_sal) <= 1e-9 * scale[:, 0] + 1e-300).all()
        # margins: the gamma tests (with the e3 >= 0 rule), and the gap to the largest neighbour at other coordinates
        e1, e2, e3 = r_eig.T
        with np.errstate(divide="ignore", invalid="ignore"):
            m_ratio = np.minimum(np.abs(e2 / e1 - g21) / g21, np.abs(e3 / e2 - g32) / g32)
            m_ratio = np.minimum(m_ratio, np.where(e3 == 0, 1.0, np.abs(e3) / e1))
        unsure = (np.nan_to_num(m_ratio, nan=1.0) < MARGIN) & (r_cnt >= mn)     # below min_neighbors s = 0 anyway
        r_flag, r_cnt_n, gap = H.nonmax(P, r_sal, rn, 0.0, True, mn, nb=nb_n)
        np.testing.assert_array_equal(cnt_n[b], r_cnt_n)
        with np.errstate(invalid="ignore"):
            tight = (r_sal > 0) & (np.abs(gap) <= MARGIN * r_sal)
        _flags_equal(flag[b].astype(bool), r_flag, unsure | _near(unsure, *nb_n) | tight, (case, b, "iss"))
    if case == "kitti":
        assert big > 2048


@pytest.mark.parametrize("case", CASES)
def test_harris_matches_restatement(case):
    clouds, _, r = _case(case)
    thr = 0.001
    grid = ops.hc_grid(_pc(clouds))
    resp, cnt, nrm = ops.harris3d_response(grid, r)
    flag, cnt_n = ops.hc_nonmax(grid, resp, r, thr, False, 1)
    resp, cnt, flag, cnt_n = (t.cpu().numpy() for t in (resp, cnt, flag, cnt_n))
    for b, P in enumerate(clouds):
        nb = H.neighbours(P, r)
        R, r_cnt, _, lam = H.harris_response(P, r, nb=nb)
        np.testing.assert_array_equal(cnt[b], r_cnt)
        np.testing.assert_array_equal(cnt_n[b], r_cnt)
        # a normal whose two smallest covariance eigenvalues nearly coincide is ill-determined on both sides
        with np.errstate(divide="ignore", invalid="ignore"):
            weak = (lam[:, 1] - lam[:, 0]) <= 1e-5 * lam[:, 2]
        unsure = _near(weak, *nb)
        assert unsure.mean() < 0.01, unsure.mean()
        scale = 0.04 + np.abs(R) + 0.04
        np.testing.assert_array_equal(np.isnan(resp[b]), np.isnan(R))
        ok = ~unsure & ~np.isnan(R)
        assert (np.abs(resp[b][ok] - R[ok]) <= 1e-9 * scale[ok]).all()
        r_flag, _, gap = H.nonmax(P, R, r, thr, False, 1, nb=nb)
        with np.errstate(invalid="ignore"):
            tight = (np.abs(R - thr) <= MARGIN * scale) | ((R >= thr) & (np.abs(gap) <= MARGIN * scale))
        _flags_equal(flag[b].astype(bool), r_flag, unsure | _near(unsure, *nb) | tight, (case, b, "harris"))


def test_corner_and_duplicate_ties():
    from tests.test_handcrafted_host import corner_cloud
    P = corner_cloud(0)
    P = np.concatenate([P, P[:1]])                    # the corner twice
    grid = ops.hc_grid(_pc(P[None]))
    sal = ops.iss_saliency(grid, 0.25, 0.975, 0.975, 5)[0]
    f_iss = ops.hc_nonmax(grid, sal, 0.25, 0.0, True, 5)[0][0].cpu().numpy().astype(bool)
    resp = ops.harris3d_response(grid, 0.25)[0]
    f_h = ops.hc_nonmax(grid, resp, 0.25, 0.001, False, 1)[0][0].cpu().numpy().astype(bool)
    s, R = sal[0].cpu().numpy(), resp[0].cpu().numpy()
    assert s[0] == s[-1] and R[0] == R[-1]            # bitwise-equal scores for equal coordinates
    np.testing.assert_array_equal(f_iss, H.iss_flags(P, 0.25, 0.25, 0.975, 0.975, 5))
    np.testing.assert_array_equal(f_h, H.harris_flags(P, 0.25, 0.001))
    for f in (f_iss, f_h):
        assert np.sqrt((P[f].astype(np.float64) ** 2).sum(1)).min() < 0.2
        assert f[0] == f[-1]


def test_determinism():
    clouds, (rs, rn), r = _case("kitti")
    outs = []
    for _ in range(2):
        grid = ops.hc_grid(_pc(clouds))
        sal = ops.iss_saliency(grid, rs, 0.975, 0.975, 5, want_eig=True)
        fl = ops.hc_nonmax(grid, sal[0], rn, 0.0, True, 5)
        hr = ops.harris3d_response(grid, r)
        outs.append([t.cpu() for t in (sal[0], sal[1], sal[2], fl[0], hr[0], hr[2])])
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int64) if a.dtype == torch.float64 else a,
                           b.view(torch.int64) if b.dtype == torch.float64 else b)


@pytest.mark.parametrize("with_flags", [True, False])
def test_select_matches_restatement(with_flags):
    B, N, L, seed, step = 4, 5000, 512, 12345, 7
    rng = np.random.default_rng(3)
    flags = np.zeros((B, N), np.int32)
    for b, c in enumerate((37, 3000, 0, 512)):        # count < L, count > L, none, count = L
        flags[b, rng.choice(N, c, replace=False)] = 1
    f = torch.from_numpy(flags).to(dev()) if with_flags else None
    order, count = ops.hc_select(f, B, N, L, seed, step, device=dev())
    order, count = order.cpu().numpy(), count.cpu().numpy()
    for b in range(B):
        o, c = H.select(flags[b] if with_flags else None, N, L, seed, step, b)
        np.testing.assert_array_equal(order[b], o)
        assert count[b] == c


def test_refusals():
    pc = _pc(structured_cloud(256, 4.0, 1)[None])
    grid = ops.hc_grid(pc)
    for args in ((0.0, 0.9, 0.9, 5), (float("nan"), 0.9, 0.9, 5), (1.0, 0.0, 0.9, 5), (1.0, 0.9, 1.1, 5),
                 (1.0, 0.9, 0.9, 0)):
        with pytest.raises(UsipB200Error):
            ops.iss_saliency(grid, *args)
    with pytest.raises(UsipB200Error):
        ops.harris3d_response(grid, -1.0)
    s = torch.zeros((1, 256), dtype=torch.float64, device=dev())
    with pytest.raises(UsipB200Error):
        ops.hc_nonmax(grid, s, 1.0, float("nan"), True, 1)
    for L in (0, 257):
        with pytest.raises(UsipB200Error):
            ops.hc_select(None, 1, 256, L, device=dev())
    with pytest.raises(ValueError):
        ops.hc_grid(torch.zeros((1, 3, (1 << 20) + 1), dtype=torch.float32, device=dev()))
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- end to end
DETECTORS = {
    "iss": (lambda: IssDetector(seed=5), {}),
    "harris": (lambda: Harris3DDetector(seed=5), {}),
    "random": (lambda: RandomDetector(seed=5), {}),
}
INDOOR = {
    "iss": (lambda: IssDetector(0.6, 0.6, seed=5), {"salient_radius": 0.6, "non_max_radius": 0.6}),
    "harris": (lambda: Harris3DDetector(0.6, seed=5), {"radius": 0.6}),
    "random": (lambda: RandomDetector(seed=5), {}),
}


def _restated_keypoints(ev, method, M, kw):
    kp, counts = [], []
    for step, (items, (pc, sn, node)) in enumerate(ev.source.batches()):
        k, c = H.detect(method, pc.cpu().numpy(), M, 5, step, **kw)
        kp.append(k); counts.append(c)
    return np.concatenate(kp), np.concatenate(counts)


@pytest.mark.parametrize("dataset", ["kitti", "redwood"])
@pytest.mark.parametrize("method", ["iss", "harris", "random"])
def test_repeatability_end_to_end(dataset, method, tmp_path):
    root = str(tmp_path)
    M, B = 64, 2
    if dataset == "kitti":
        opt = make_opt(batch_size=B, input_pc_num=2048, node_num=M)
        txt, num, cal = (os.path.join(root, d) for d in ("txt", "numpy", "calib"))
        ktl.write_synthetic_kitti_test(txt, num, cal, [3, 2], 3000, [[(0, 1), (2, 1), (0, 2)], [(1, 0)]], seed=75)
        ev = rep.KittiRepeatability(txt, num, cal, opt, seed=9, batch_size=B)
        make, kw = DETECTORS[method]
    else:
        opt = rep.detector_opt("redwood", batch_size=B, input_pc_num=2048, node_num=M, device=dev())
        scenes = [("livingroom1", 3), ("office2", 2)]
        npy, gt = os.path.join(root, "npy"), os.path.join(root, "gt")
        itl.write_synthetic_redwood(npy, gt, 3000, {"livingroom1": [(0, 1), (2, 0)], "office2": [(1, 0)]}, seed=4,
                                    scenes=scenes)
        ev = rep.RedwoodRepeatability(npy, gt, opt, seed=9, batch_size=B, scenes=scenes)
        make, kw = INDOOR[method]
    det = make()
    ks = [4, 16, 64]
    res = ev.run(det, ks)
    kp, counts = _restated_keypoints(ev, method, M, kw)
    np.testing.assert_array_equal(det.detected.cpu().numpy(), counts)
    S = len(kp)
    inl, n_anc = repeatability_ref(kp, np.tile(np.arange(M), (S, 1)), np.full(S, M), ev.pairs, ev.frames, ks, 0.5)
    np.testing.assert_array_equal(res.n_anc, n_anc)
    np.testing.assert_array_equal(res.inliers, inl)
    again = ev.run(det, ks)                            # a second pass with the same object repeats the first
    np.testing.assert_array_equal(again.inliers, res.inliers)
    assert "keypoint number max" in det.count_summary()


def test_registration_describe_with_iss(tmp_path):
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    root = str(tmp_path)
    M, B = 64, 2
    opt = make_opt(batch_size=B, input_pc_num=1024, node_num=M)
    torch.manual_seed(5)
    des = ModelDescriptor(opt)
    txt, num, cal = (os.path.join(root, d) for d in ("txt", "numpy", "calib"))
    ktl.write_synthetic_kitti_test(txt, num, cal, [3], 1500, [[(0, 1), (1, 2), (2, 2)]], seed=3)
    ev = reg.Registration(rep.KittiRepeatability(txt, num, cal, opt, seed=9, batch_size=B))
    det = IssDetector(seed=1)
    res = ev.run(det, des, [4, 16, 64], max_trials=[100], seed=17)
    assert res.inliers.shape[:2] == (3, 3)
    assert ev.xyz.shape == (3, 64, 3) and (ev.count.cpu().numpy() == 64).all()
    with pytest.raises(ValueError):
        ev.run(det, des, [4], nms_radius=1.0)
