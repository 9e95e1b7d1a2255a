"""Registration on the GPU (csrc/registration.cu usip_desc_match_f64, usip_ransac_rt_f64, usip_ransac_uniforms;
usip_b200.evaluation.registration).

The kernels against the float64 restatement of the MATLAB scripts (tests/reg_ref.py), exactly: matches in both modes,
and RANSAC's status, trial count, best trial and inlier count over a few hundred (pair, K) cases and a full maxTrials
sweep, Rt to 1e-12; device-mode uniforms against uploaded ones; sweep and pair independence; recovery of a known
motion; and the evaluator end to end against the restatement run on the descriptor tree it writes."""
import os

import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests import reg_ref as rr
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import ops
from usip_b200.evaluation import kitti_test_loader as ktl
from usip_b200.evaluation import oxford_test_loader as otl
from usip_b200.evaluation import registration as reg
from usip_b200.evaluation import repeatability as rep

pytestmark = pytest.mark.gpu

TRIALS = [50, 100, 250, 500, 1000, 2500, 5000, 10000]


def d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def _rigid(rng, t=5.0):
    q = rng.normal(size=4)
    return rep.gt_transform(rng.uniform(-t, t, 3), q / np.linalg.norm(q))


# ----------------------------------------------------------------------------------------------- matching
@pytest.mark.parametrize("k", [1, 5, 8])
@pytest.mark.parametrize("D", [128, 352])
def test_match_kernel_matches_restatement(k, D):
    rng = np.random.RandomState(100 + k + D)
    S, L, P = 12, 40, 30
    desc = rng.randint(-2, 3, (S, L, D)).astype(np.float32) * 0.5           # coarse values: many equal distances
    desc[:, :, : D // 2] += rng.normal(0, 0.3, (S, L, D // 2)).astype(np.float32)
    desc[3, 5] = desc[3, 9]                                                  # an exact tie
    count = rng.randint(1, L + 1, S).astype(np.int32)
    count[:4] = [1, 3, L, 2]                                                 # k > count for the positive set
    pairs = rng.randint(0, S, (P, 2)).astype(np.int32)
    pairs[:4] = [[2, 1], [1, 2], [3, 3], [2, 0]]
    ks = [1, 3, 7, 20, 40, 64]                                               # K > L included
    m, n = ops.desc_match(d(desc), d(count), d(pairs), ks, k)
    m, n = m.cpu().numpy(), n.cpu().numpy()
    assert m.shape == (P, len(ks), L if k == 1 else 2 * k * L, 2)
    for p, (a, b) in enumerate(pairs):
        for j, K in enumerate(ks):
            ref = rr.match_ref(desc[a, :min(K, count[a])], desc[b, :min(K, count[b])], k)
            assert n[p, j] == len(ref), (p, K)
            np.testing.assert_array_equal(m[p, j, :n[p, j]], ref, err_msg="pair %d K %d" % (p, K))


@pytest.mark.parametrize("k", [1, 5])
def test_match_kernel_orders_non_finite_descriptors(k):
    """NaN and inf descriptor values (PCL's SHOT writes NaN for sparse neighbourhoods): their distances order as +inf,
    by index, so every row still gets min(k, n) neighbours -- against the restatement, a positive set smaller than k
    included."""
    rng = np.random.RandomState(31 + k)
    S, L, D, P = 6, 24, 352, 12
    desc = rng.normal(0, 1, (S, L, D)).astype(np.float32)
    desc[0, :3, 7] = np.nan                                                  # the first rows: row 0 of the bitset
    desc[1, 5, :] = np.nan
    desc[2, 2, 100] = np.inf
    desc[3, :, 0] = np.nan                                                   # every distance of scan 3 is NaN
    desc[4, 1, 3] = -np.inf
    count = np.array([L, L, 4, L, 3, L], np.int32)                           # 3 and 4 rows: fewer than k = 5
    pairs = np.array([[0, 1], [1, 0], [3, 2], [2, 3], [4, 1], [1, 4], [3, 3], [0, 4], [5, 3], [2, 2], [4, 0], [5, 1]],
                     np.int32)
    ks = [4, 16, 24]
    m, n = ops.desc_match(d(desc), d(count), d(pairs), ks, k)
    m, n = m.cpu().numpy(), n.cpu().numpy()
    for p, (a, b) in enumerate(pairs):
        for j, K in enumerate(ks):
            ref = rr.match_ref(desc[a, :min(K, count[a])], desc[b, :min(K, count[b])], k)
            assert n[p, j] == len(ref), (p, K)
            np.testing.assert_array_equal(m[p, j, :n[p, j]], ref, err_msg="pair %d K %d" % (p, K))


# ----------------------------------------------------------------------------------------------- RANSAC
def _correspondences(rng, n, ratio, T):
    """n correspondences, a fraction `ratio` inliers of x1 = T x2 with residual <= 0.3, the others >= 3 away."""
    x2 = rng.uniform(-30, 30, (n, 3))
    x1 = x2 @ T[:, :3].T + T[:, 3]
    inl = rng.rand(n) < ratio
    dirs = rng.normal(size=(n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    x1 += dirs * np.where(inl, rng.uniform(0, 0.3, n), rng.uniform(3, 40, n))[:, None]
    return x1, x2


def _ransac_case(rng, sizes, ratios, nK, L=128):
    """Pair p reads scans 2p (anchor) and 2p+1 (positive), whose rows hold max(sizes of p) correspondences of a random
    motion with inlier ratio ratios[p] (in the camera frame: the frame maps are inverted); its K = kk match list is
    the first sizes[p * nK + kk] of them, anchor rows permuted.  Returns the kernel inputs and each (pair, K)'s mapped
    (x1, x2)."""
    P = len(ratios)
    xyz = np.zeros((2 * P, L, 3), np.float32)
    frames = np.zeros((P, 3, 3, 4))
    matches = np.zeros((P, nK, 2 * L, 2), np.int32)
    n_m = np.zeros((P, nK), np.int32)
    cases = {}
    inv = lambda F, x: (x - F[:, 3]) @ np.linalg.inv(F[:, :3]).T
    for p in range(P):
        Fa, Fp, T = _rigid(rng, 2.0), _rigid(rng, 2.0), _rigid(rng)
        frames[p] = [Fa, Fp, np.eye(3, 4)]
        n_all = max(sizes[p * nK:(p + 1) * nK])
        c1, c2 = _correspondences(rng, n_all, ratios[p], T)
        perm = rng.permutation(L)[:n_all]
        xa, xp = np.zeros((L, 3)), np.zeros((L, 3))
        xa[perm], xp[:n_all] = c1, c2
        xyz[2 * p], xyz[2 * p + 1] = inv(Fa, xa), inv(Fp, xp)
        x1_all = rr.apply_map(Fa, xyz[2 * p].astype(np.float64))
        x2_all = rr.apply_map(Fp, xyz[2 * p + 1].astype(np.float64))
        for kk in range(nK):
            n = sizes[p * nK + kk]
            mm = np.stack([perm[:n], np.arange(n)], 1)
            matches[p, kk, :n], n_m[p, kk] = mm, n
            cases[p, kk] = (x1_all[mm[:, 0]], x2_all[mm[:, 1]])
    pairs = np.stack([np.arange(P) * 2, np.arange(P) * 2 + 1], 1).astype(np.int32)
    return xyz, np.full(2 * P, L, np.int32), pairs, frames, matches, n_m, cases


def _check(out, cases, trials, uniforms, thr=1.0):
    got = {k: v.cpu().numpy() for k, v in out.items()}
    statuses = set()
    for (p, kk), (x1, x2) in cases.items():
        ref = rr.ransac_ref(x1, x2, trials, thr, uniforms)
        for t, r in enumerate(ref):
            key = (p, kk, t)
            for f in ("status", "trialcount", "best_trial", "n_inliers"):
                assert got[f][key] == r[f], (f, key, got[f][key], r[f], len(x1))
            np.testing.assert_allclose(got["Rt"][key], r["Rt"], rtol=0, atol=1e-12, err_msg=str(key))
            statuses.add(r["status"])
    return got, statuses


def test_ransac_kernel_matches_restatement():
    rng = np.random.RandomState(7)
    nK, P = 8, 40
    sizes = [[0, 2, 3, 4, 5, 8, 20, 40, 60, 100][(p + kk) % 10] for p in range(P) for kk in range(nK)]
    ratios = [[1.0, 0.9, 0.6, 0.4, 0.25, 0.15, 0.05][p % 7] for p in range(P)]
    xyz, count, pairs, frames, matches, n_m, cases = _ransac_case(rng, sizes, ratios, nK)
    uni = np.random.RandomState(8).rand(TRIALS[-1] + 1, 3)
    out = ops.ransac_rt(d(xyz), d(count), d(pairs), d(frames), d(matches), d(n_m), TRIALS, 1.0, 0, d(uni))
    got, statuses = _check(out, cases, TRIALS, uni)
    assert {0, 1}.issubset(statuses)
    assert (got["trialcount"] == 10001).any() and ((got["trialcount"] > 0) & (got["trialcount"] < 51)).any()


def test_ransac_too_few_inliers():
    x1 = np.array([[0.0, 0, 0], [100, 0, 0], [0, 100, 0], [0, 0, 100]])
    x2 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 50, 0], [30, 30, 30]])
    xyz = np.zeros((2, 8, 3), np.float32)
    xyz[0, :4], xyz[1, :4] = x1, x2
    frames = np.stack([np.eye(3, 4)] * 3)[None]
    matches = np.zeros((1, 1, 16, 2), np.int32)
    matches[0, 0, :4] = np.stack([np.arange(4), np.arange(4)], 1)
    uni = np.random.RandomState(1).rand(101, 3)
    out = ops.ransac_rt(d(xyz), d(np.array([8, 8], np.int32)), d(np.array([[0, 1]], np.int32)), d(frames),
                        d(matches), d(np.array([[4]], np.int32)), [100], 1.0, 0, d(uni))
    got, statuses = _check(out, {(0, 0): (x1, x2)}, [100], uni)
    assert statuses == {2} and got["n_inliers"][0, 0, 0] < 3 and got["trialcount"][0, 0, 0] == 101


def test_device_mode_sweep_and_pair_independence():
    rng = np.random.RandomState(9)
    nK = 2
    sizes = [50, 100] * 3
    ratios = [0.2, 0.5, 0.02]
    xyz, count, pairs, frames, matches, n_m, cases = _ransac_case(rng, sizes, ratios, nK)
    pairs[2] = pairs[0]; frames[2] = frames[0]; matches[2] = matches[0]; n_m[2] = n_m[0]     # identical pairs
    args = [d(xyz), d(count), d(pairs), d(frames), d(matches), d(n_m)]
    dev_mode = ops.ransac_rt(*args, TRIALS, 1.0, 1234, None)
    uni = ops.ransac_uniforms(TRIALS[-1] + 1, 1234)
    assert uni.min().item() >= 0.0 and uni.max().item() < 1.0
    up = ops.ransac_rt(*args, TRIALS, 1.0, 0, uni)
    for f in dev_mode:
        assert torch.equal(dev_mode[f], up[f]), f
        assert torch.equal(dev_mode[f][0], dev_mode[f][2]), f
    alone = ops.ransac_rt(*args, [50], 1.0, 1234, None)
    for f in dev_mode:
        assert torch.equal(alone[f][:, :, 0], dev_mode[f][:, :, 0]), f
    other = ops.ransac_rt(*args, TRIALS, 1.0, 99, None)
    assert not torch.equal(other["best_trial"], dev_mode["best_trial"])


def test_noise_free_recovery():
    rng = np.random.RandomState(3)
    T = _rigid(rng)
    n = 300
    x2 = rng.uniform(-30, 30, (n, 3))
    x1 = x2 @ T[:, :3].T + T[:, 3]
    out_rows = rng.rand(n) < 0.6
    x1[out_rows] += rng.uniform(3, 40, (out_rows.sum(), 3)) * rng.choice([-1, 1], (out_rows.sum(), 3))
    xyz = np.stack([x1, x2]).astype(np.float32)
    x1, x2 = xyz[0].astype(np.float64), xyz[1].astype(np.float64)
    T = rr.fit(x1[~out_rows][None], x2[~out_rows][None])[0]      # the motion of the float32 points
    matches = np.stack([np.arange(n), np.arange(n)], 1)[None, None].astype(np.int32)
    matches = np.concatenate([matches, np.zeros((1, 1, 2 * 1024 - n, 2), np.int32)], 2)
    out = ops.ransac_rt(d(xyz), d(np.array([n, n], np.int32)), d(np.array([[0, 1]], np.int32)),
                        d(np.stack([np.eye(3, 4)] * 3)[None]), d(matches), d(np.array([[n]], np.int32)), TRIALS,
                        1.0, 5, None)
    Rt = out["Rt"].cpu().numpy()[0, 0]
    assert (out["status"].cpu().numpy() == 0).all()
    for t in range(len(TRIALS)):
        dt, dd = reg.compare_transform(T, Rt[t])
        assert dt < 1e-9 and dd < 1e-9, (t, dt, dd)
    assert (out["n_inliers"].cpu().numpy() == (~out_rows).sum()).all()


def test_refusals():
    desc = d(np.zeros((2, 8, 16), np.float32)); cnt = d(np.full(2, 8, np.int32)); pairs = d(np.zeros((1, 2), np.int32))
    for ks, k in (([8, 4], 1), (list(range(1, 34)), 1), ([4], 0), ([4], 9)):
        with pytest.raises(RuntimeError):
            ops.desc_match(desc, cnt, pairs, ks, k)
    with pytest.raises(RuntimeError, match="USIP_REG_MAX_DIM"):
        ops.desc_match(d(np.zeros((2, 8, 513), np.float32)), cnt, pairs, [4], 1)
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.desc_match(d(np.zeros((2, 1025, 8), np.float32)), cnt, pairs, [4], 1)
    m, n = ops.desc_match(desc, cnt, pairs, [4, 8], 1)
    xyz, fr = d(np.zeros((2, 8, 3), np.float32)), d(np.zeros((1, 3, 3, 4)))
    for trials, thr in (([100, 50], 1.0), ([0], 1.0), ([200000], 1.0), (list(range(1, 18)), 1.0), ([50], 0.0),
                        ([50], -1.0)):
        with pytest.raises(RuntimeError):
            ops.ransac_rt(xyz, cnt, pairs, fr, m, n, trials, thr)
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.ransac_rt(d(np.zeros((2, 1025, 3), np.float32)), cnt, pairs, fr, d(np.zeros((1, 2, 1025, 2), np.int32)), n,
                      [50], 1.0)


# ----------------------------------------------------------------------------------------------- end to end
def _models(N, M, B):
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    from usip_b200.models.keypoint_detector import ModelDetector
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M)
    md = ModelDetector(opt)
    P = orc.init_detector_params(S=4, seed=21, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    load_params(md.detector, P)
    torch.manual_seed(5)
    desc = ModelDescriptor(opt)
    return md, desc, opt


@pytest.mark.parametrize("name", ["kitti", "oxford"])
@pytest.mark.parametrize("nms_radius", [0.0, 1.0])
def test_end_to_end_against_descriptor_tree(name, nms_radius, tmp_path):
    root = str(tmp_path)
    N, M, B = 1024, 64, 2
    det, des, opt = _models(N, M, B)
    if name == "kitti":
        txt, num, cal = os.path.join(root, "txt"), os.path.join(root, "numpy"), os.path.join(root, "calib")
        ktl.write_synthetic_kitti_test(txt, num, cal, [4, 3], 1500,
                                       [[(0, 1), (1, 2), (2, 2), (3, 0)], [(0, 1), (2, 2), (1, 2)]], seed=3)
        ev = reg.Registration(rep.KittiRepeatability(txt, num, cal, opt, seed=9, batch_size=B))
    else:
        gt = os.path.join(root, "groundtruths.txt")
        otl.write_synthetic_oxford_test(root, [0, 1, 2, 3, 4], 1500, [(0, 1), (2, 2), (3, 4), (4, 4), (1, 3)], gt, seed=4)
        ev = reg.Registration(rep.OxfordRepeatability(root, gt, opt, seed=9, batch_size=B, numbers=range(5)))
    ks, trials, seed = [4, 16, 64, 100], [50, 100, 1000], 17
    res = ev.run(det, des, ks, nms_radius=nms_radius, noise_sigma=0.01, max_trials=trials, seed=seed)
    first = ev.desc.clone()
    ev.describe(det, des, nms_radius, 0.01, L=64)
    assert torch.equal(first, ev.desc)                       # describe seeds numpy: the descriptors repeat
    uni = ops.ransac_uniforms(trials[-1] + 1, seed).cpu().numpy()
    k = 1 if name == "kitti" else 5
    out = os.path.join(root, "desc")
    frames = ev.ev.frames
    for j, K in enumerate(ks):
        ev.write_descriptor_tree(out, K)
        for p, (a, b) in enumerate(ev.ev.pairs):
            rows = [np.fromfile(ev.ev.source.keypoint_path(out, s), np.float32).reshape(-1, 3 + 128) for s in (a, b)]
            m, ref = rr.register_pair_ref(rows[0], rows[1], frames[p, 0], frames[p, 1], K, k, trials, 1.0, uni)
            for t, r in enumerate(ref):
                assert res.npts[p, j, t] == len(m)
                for f, g in (("status", res.status), ("trialcount", res.trialcount), ("n_inliers", res.inliers)):
                    assert g[p, j, t] == r[f], (f, p, K, t)
                Rt = r["Rt"] if r["status"] == 0 else None
                dt, dd = reg.compare_transform(frames[p, 2], Rt)
                assert abs(dt - res.delta_t[p, j, t]) < 1e-9 and abs(dd - res.delta_deg[p, j, t]) < 1e-7
            if a == b and name == "kitti" and len(m) >= 3:
                # KITTI's self-pair matches are all correct: every budget registers exactly, every match an inlier
                assert res.delta_t[p, j].max() < 1e-6 and res.delta_deg[p, j].max() < 1e-4, (p, K)
                assert (res.inliers[p, j] == res.npts[p, j]).all()
    # Oxford's 5-NN union adds wrong matches (3 correct ones are drawn with probability >= 1/1000 per trial at these
    # sizes), so its self-pairs are checked at 10000 trials: each registers, exactly when NMS keeps the wrong matches
    # >= 1 apart
    big = ev.score(ks, [10000], 1.0, None, seed)
    for p, (a, b) in enumerate(ev.ev.pairs):
        if a != b:
            continue
        for j, K in enumerate(ks):
            if big.npts[p, j, 0] < 3:
                continue
            assert big.success[p, j, 0], (p, K, big.delta_t[p, j, 0], big.delta_deg[p, j, 0])
            if name == "kitti" or nms_radius >= 1.0:
                assert big.delta_t[p, j, 0] < 1e-6 and big.delta_deg[p, j, 0] < 1e-4, (p, K)
    assert len(res.lines()) == 2 * len(ks) * len(trials)
    # the same scoring from the tree it wrote (largest K), as --descriptor-tree runs it
    ev.write_descriptor_tree(out, ks[-1])
    tree = reg.Registration(ev.ev)
    tree.read_descriptor_tree(out, 128)
    again = tree.score(ks, trials, 1.0, None, seed)
    np.testing.assert_array_equal(again.trialcount, res.trialcount)
    np.testing.assert_array_equal(again.delta_t, res.delta_t)
