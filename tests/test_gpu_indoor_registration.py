"""Indoor registration on the GPU (csrc/overlap.cu usip_fragment_overlap_f32, csrc/registration.cu
usip_ransac_info_f64, usip_b200.evaluation.indoor_registration).

The overlap count against the restatement (tests/indoor_reg_ref.py) exactly, over fragments of 1 to 200k rows, jobs that
share fragments, the identity and a = b, points planted within a few ulps of the 0.2 shell, duplicates, a flat
fragment, far outliers and non-finite rows; refusals before any launch.  The information matrix against the
restatement on top of tests/reg_ref.py's RANSAC, and n_info == n_inliers.  End to end: a synthetic Redwood tree of
overlapping crops of one room under known motions, position-derived descriptors, recall 1 on the overlapping gt pairs,
the filters and scores against the restatement, and the written logs re-scored."""
import os

import numpy as np
import pytest
import torch

from tests import indoor_reg_ref as ir
from tests import reg_ref as rr
from tests.test_gpu_registration import TRIALS, _ransac_case, _rigid
from tests.util_gpu import dev
from usip_b200 import ops
from usip_b200._lib import UsipB200Error
from usip_b200.evaluation import indoor_registration as idr
from usip_b200.evaluation import indoor_test_loader as itl
from usip_b200.evaluation import registration as reg

pytestmark = pytest.mark.gpu


def d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def _pack(frags):
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in frags])]).astype(np.int64)
    return np.concatenate(frags).astype(np.float32), offsets


def _run(frags, jobs, maps, radius=0.2):
    xyz, offsets = _pack(frags)
    hits = ops.fragment_overlap(d(xyz), offsets, np.array(jobs, np.int32), d(np.array(maps, np.float64)), radius)
    return hits.cpu().numpy()


def _check(frags, jobs, maps, radius=0.2):
    got = _run(frags, jobs, maps, radius)
    ref = [ir.overlap_ref(frags[a], frags[b], T, radius) for (a, b), T in zip(jobs, maps)]
    np.testing.assert_array_equal(got, ref)
    return got


# ----------------------------------------------------------------------------------------------- overlap
def test_overlap_matches_restatement_sizes_and_shared_fragments():
    rng = np.random.RandomState(1)
    sizes = [1, 2, 17, 300, 4096, 30000, 200000]
    frags = [rng.uniform(-2, 2, (n, 3)).astype(np.float32) for n in sizes]
    frags[3][:, 2] = 0.5                                         # zero extent along z
    jobs, maps = [], []
    for a in range(len(frags)):
        for b in range(len(frags)):
            if (a + b) % 2 == 0 or a == b:
                jobs.append((a, b))
                maps.append(np.eye(3, 4) if a == b or (a + b) % 4 == 0 else _rigid(rng, 0.3))
    got = _check(frags, jobs, maps)
    assert got[jobs.index((5, 5))] == 30000 and 0 < got.sum()


def test_overlap_shell_ulps():
    """Points of a placed at 0.2 +- a few fp32 ulps from mapped points of b, on every axis and on diagonals."""
    rng = np.random.RandomState(2)
    b = rng.uniform(-1, 1, (200, 3)).astype(np.float32)
    T = _rigid(rng, 0.5)
    bp = ir.map_b(T, b)
    r = np.float32(0.2)
    steps = [-3, -2, -1, 0, 1, 2, 3]
    pts = []
    for i, s in enumerate(steps * 20):
        rad = r
        for _ in range(abs(s)):
            rad = np.nextafter(rad, np.float32(np.inf) if s > 0 else np.float32(0))
        axis = i % 4
        dvec = np.zeros(3, np.float32)
        if axis < 3:
            dvec[axis] = rad
        else:
            dvec[:] = np.float32(rad / np.sqrt(np.float32(3)))
        pts.append(bp[i % len(bp)] + dvec)
    a = np.array(pts, np.float32)
    got = _check([a, b], [(0, 1)], [T])
    assert 0 < got[0] < len(a)


def test_overlap_degenerate_rows():
    rng = np.random.RandomState(3)
    a = rng.uniform(-1, 1, (5000, 3)).astype(np.float32)
    b = a.copy()
    b[:100] = b[0]                                               # duplicates
    b[100] = [1e6, 0, 0]                                         # far outliers on both sides
    a[101] = [0, -3e7, 0]
    a[200:220, 0] = np.nan                                       # non-finite rows in a and in b
    a[220:230, 1] = np.inf
    b[300:320, 2] = -np.inf
    b[320:330, 0] = np.nan
    T = _rigid(rng, 0.05)
    nan_map = np.eye(3, 4)
    nan_map[0, 3] = np.nan
    zero_map = np.zeros((3, 4))                                  # every b' at the origin
    got = _check([a, b, a[:1]], [(0, 1), (1, 0), (0, 0), (0, 1), (0, 1), (2, 0)],
                 [T, T, np.eye(3, 4), nan_map, zero_map, np.eye(3, 4)])
    assert got[2] == 5000 - 30 and got[3] == 0


def test_overlap_refusals():
    xyz = d(np.zeros((10, 3), np.float32))
    Rt = d(np.zeros((1, 3, 4)))
    ok_off = np.array([0, 4, 10])
    with pytest.raises(UsipB200Error, match="out of range"):
        ops.fragment_overlap(xyz, ok_off, np.array([[0, 2]]), Rt)
    with pytest.raises(UsipB200Error, match="no rows"):
        ops.fragment_overlap(xyz, np.array([0, 0, 10]), np.array([[0, 1]]), Rt)
    for r in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(UsipB200Error, match="radius"):
            ops.fragment_overlap(xyz, ok_off, np.array([[0, 1]]), Rt, r)
    from usip_b200 import _lib
    lib = _lib.load()
    hits = torch.full((1,), 7, dtype=torch.int32, device=dev())
    off = ok_off.astype(np.int64)
    jobs = np.array([[0, 1]], np.int32)
    need = int(lib.usip_fragment_overlap_scratch_bytes(10, 2, 1))
    scratch = torch.empty((need // 16 + 1, 4), dtype=torch.int32, device=dev())
    rc = lib.usip_fragment_overlap_f32(ops._p(xyz), off.ctypes.data, 2, jobs.ctypes.data, ops._p(Rt), 1,
                                       0.2, ops._p(scratch), need - 16, ops._p(hits), None)
    assert rc == -1 and b"scratch" in lib.usip_last_error()
    big = np.array([0, (1 << 26) + 1])
    rc = lib.usip_fragment_overlap_f32(ops._p(xyz), big.ctypes.data, 1, np.zeros((1, 2), np.int32).ctypes.data,
                                       ops._p(Rt), 1, 0.2, ops._p(scratch), need, ops._p(hits), None)
    assert rc == -1 and b"MAX_ROWS" in lib.usip_last_error()
    torch.cuda.synchronize()
    assert hits.item() == 7                                      # nothing ran


# ----------------------------------------------------------------------------------------------- information matrix
def test_info_kernel_matches_restatement():
    rng = np.random.RandomState(11)
    nK, P = 6, 40
    sizes = [[0, 2, 3, 4, 5, 8, 20, 40, 60, 100][(p + kk) % 10] for p in range(P) for kk in range(nK)]
    ratios = [[1.0, 0.9, 0.6, 0.4, 0.25, 0.15, 0.05][p % 7] for p in range(P)]
    xyz, count, pairs, frames, matches, n_m, cases = _ransac_case(rng, sizes, ratios, nK)
    trials = [50, 1000, 10000]
    uni = np.random.RandomState(12).rand(trials[-1] + 1, 3)
    args = (d(xyz), d(count), d(pairs), d(frames), d(matches), d(n_m))
    out = ops.ransac_rt(*args, trials, 1.0, 0, d(uni))
    info, n_info = ops.ransac_info(*args, trials, out["best_trial"], out["status"], 1.0, 0, d(uni))
    info, n_info = info.cpu().numpy(), n_info.cpu().numpy()
    st, ninl = out["status"].cpu().numpy(), out["n_inliers"].cpu().numpy()
    np.testing.assert_array_equal(n_info[st == 0], ninl[st == 0])
    seen = set()
    for (p, kk), (x1, x2) in cases.items():
        _, ref = ir.info_ref(x1, x2, trials, 1.0, uni)
        for t, (M, n) in enumerate(ref):
            assert n_info[p, kk, t] == n, (p, kk, t)
            np.testing.assert_allclose(info[p, kk, t], M, rtol=1e-12, atol=1e-12 * max(1.0, np.abs(M).max()))
            seen.add((len(x1) == 3, st[p, kk, t] != 0))
    assert (True, False) in seen and (False, True) in seen


def test_info_kernel_philox_stream():
    rng = np.random.RandomState(13)
    nK, P = 2, 12
    sizes = [[4, 9, 30, 80][(p + kk) % 4] for p in range(P) for kk in range(nK)]
    xyz, count, pairs, frames, matches, n_m, cases = _ransac_case(rng, sizes, [0.5] * P, nK)
    args = (d(xyz), d(count), d(pairs), d(frames), d(matches), d(n_m))
    out = ops.ransac_rt(*args, TRIALS, 1.0, 99)
    info, n_info = ops.ransac_info(*args, TRIALS, out["best_trial"], out["status"], 1.0, 99)
    uni = ops.ransac_uniforms(TRIALS[-1] + 1, 99).cpu().numpy()
    for (p, kk), (x1, x2) in cases.items():
        _, ref = ir.info_ref(x1, x2, TRIALS, 1.0, uni)
        for t, (M, n) in enumerate(ref):
            assert n_info[p, kk, t].item() == n
            np.testing.assert_allclose(info[p, kk, t].cpu().numpy(), M, rtol=1e-12, atol=1e-9)


# ----------------------------------------------------------------------------------------------- end to end
SCENE = "livingroom1"


def _room_tree(tmp, n_frag=6, rows=6000, n_clusters=60, seed=21):
    """Fragments f = crops of one 8 m room along x, 3.9 m wide every 0.8 m, each in its own frame T_f.  Keypoints:
    clusters of 5 room positions (within 0.04 m of a centre), in one global order, cluster by cluster; a fragment keeps
    the clusters whose centre it crops; descriptor = the global position.  gt.log lists the pairs at most two crops
    apart (overlap about 60 %), T_ij = inv(T_i) T_j, and gt.info their info_matrix."""
    rng = np.random.RandomState(seed)
    room = rng.uniform([-4, -2, -1.5], [4, 2, 1.5], (n_frag * rows, 3))
    centres = rng.uniform([-4, -2, -1.5], [4, 2, 1.5], (n_clusters, 3))
    kp = (centres[:, None, :] + rng.uniform(-0.02, 0.02, (n_clusters, 5, 3))).reshape(-1, 3)
    npy, gt, tree = (os.path.join(tmp, x) for x in ("npy", "gt", "tree"))
    T = [np.vstack([_rigid(rng, 1.0), [0, 0, 0, 1]]) for _ in range(n_frag)]
    lo = np.arange(n_frag) * 0.8 - 4.0
    for f in range(n_frag):
        inside = lambda x: (x >= lo[f]) & (x < lo[f] + 3.9)
        local = (room[inside(room[:, 0])] - T[f][:3, 3]) @ T[f][:3, :3]
        a = np.zeros((len(local), 7), np.float32)
        a[:, :3] = local
        a[:, 3] = 1
        os.makedirs(os.path.join(npy, SCENE), exist_ok=True)
        np.save(os.path.join(npy, SCENE, "%d.npy" % f), a)
        g = kp[np.repeat(inside(centres[:, 0]), 5)]
        kl = (g - T[f][:3, 3]) @ T[f][:3, :3]
        os.makedirs(os.path.join(tree, SCENE), exist_ok=True)
        np.concatenate([kl, g], 1).astype(np.float32).tofile(os.path.join(tree, SCENE, "%d.bin" % f))
    entries, infos = [], []
    for i in range(n_frag):
        for j in range(i + 1, min(i + 3, n_frag)):
            entries.append((i, j, n_frag, np.linalg.inv(T[i]) @ T[j]))
            infos.append((i, j, n_frag, itl.info_matrix(((room[:200] - T[i][:3, 3]) @ T[i][:3, :3]))))
    ev_dir = os.path.join(gt, "original", "%s-evaluation" % SCENE)
    itl.write_gt_log(os.path.join(ev_dir, "gt.log"), entries)
    itl.write_gt_info(os.path.join(ev_dir, "gt.info"), infos)
    return npy, gt, tree, 3, entries


def test_end_to_end_room(tmp_path):
    npy, gt, tree, D, entries = _room_tree(str(tmp_path))
    opt = reg.descriptor_opt("redwood", input_pc_num=1024, batch_size=2)
    ev = idr.IndoorRegistration.redwood(npy, gt, opt, scenes=[(SCENE, 6)])
    ev.read_descriptor_tree(tree, D)
    ks, ts = [60, 120], [1000, 30000]
    res = ev.score(ks, ts, pairs="all", seed=3)
    r = res.per_scene[SCENE]
    assert len(r["pairs"]) == 15
    gt_far = [(i, j) for i, j, _, _ in entries if j - i > 1]
    assert gt_far
    for (K, T), (sc, line, means) in res.scores.items():
        s = sc[SCENE]
        assert s["recall"] == 1.0, (K, T, s)
        assert s["gt_num"] == len(gt_far)
    # filters and counts against the restatement run on the kernels' outputs
    uni = ops.ransac_uniforms(ts[-1] + 1, 3).cpu().numpy()
    xyz_np, count_np = ev.xyz.cpu().numpy(), ev.count.cpu().numpy()
    frags = [np.load(os.path.join(npy, SCENE, "%d.npy" % f))[:, :3] for f in range(6)]
    for p, (i, j) in enumerate(r["pairs"]):
        for k, K in enumerate(ks):
            a, b = xyz_np[i, :min(K, count_np[i])], xyz_np[j, :min(K, count_np[j])]
            da = ev.desc.cpu().numpy()[i, :len(a)]
            db = ev.desc.cpu().numpy()[j, :len(b)]
            m = rr.match_ref(da, db, 5)
            assert r["n_matches"][p, k] == len(m)
            x1, x2 = a[m[:, 0]].astype(np.float64), b[m[:, 1]].astype(np.float64)
            ransac, info = ir.info_ref(x1, x2, ts, 0.2, uni)
            for t in range(len(ts)):
                n = ransac[t]["n_inliers"] if ransac[t]["status"] == 0 else 0
                assert r["n_inliers"][p, k, t] == n
                ratio = n / len(m) if len(m) else float("nan")
                assert (r["inlier_ratio"][p, k, t] > 0.025) == (ratio > 0.025)
                np.testing.assert_allclose(r["info"][p, k, t], info[t][0], rtol=1e-12, atol=1e-9)
                if ratio > 0.025:
                    Rt = r["Rt"][p, k, t, :3]
                    al = ir.overlap_ref(frags[i], frags[j], Rt) / len(frags[i])
                    assert r["aligned"][p, k, t] == al
                    assert r["accepted"][p, k, t] == (al > 0.23)
                else:
                    assert not r["accepted"][p, k, t]
    # the written logs re-score identically, through the module and through the restatement
    out = os.path.join(str(tmp_path), "logs")
    ev.write_registration_logs(out, 120, 30000)
    sc, line, _ = ev.score_logs(out)
    direct = res.scores[(120, 30000)][0][SCENE]
    for key in ("recall", "precision", "good", "gt_num", "rs_num"):
        assert sc[SCENE][key] == direct[key]
    ev_dir = os.path.join(gt, "original", "%s-evaluation" % SCENE)
    gt_log = [dict(info=[int(a), int(b), int(c)], trans=T) for a, b, c, T in entries]
    gt_info = [m for _, m in ir.load_info(os.path.join(ev_dir, "gt.info"))]
    ref = ir.evaluate_my(ir.load_log_my(os.path.join(out, "%s.log" % SCENE)), gt_log, gt_info)
    assert ref["recall"] == sc[SCENE]["recall"] and ref["good"] == sc[SCENE]["good"]
    assert ref["rs_num"] == sc[SCENE]["rs_num"]
    # the lite variant: no overlap test, gt pairs only
    lite = ev.score([120], [1000], overlap_threshold=None, pairs="gt", seed=3)
    assert lite.scores[(120, 1000)][0][SCENE]["recall"] == 1.0
