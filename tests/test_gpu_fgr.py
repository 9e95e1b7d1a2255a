"""Fast Global Registration on the GPU (csrc/registration.cu usip_desc_match_mutual_f64, csrc/fgr.cu usip_fgr_f64,
usip_b200.evaluation.indoor_registration's solver "fgr" and fast_global_registration).

Mutual matches bit for bit against tests/fgr_ref.py and against usip_desc_match_f64's k = 1 run both ways, over ties,
NaN descriptors, n1 != n2, count < K, L = 1 and 1024, D = 1 and 512.  usip_fgr_f64 against the restatement: n_tuples,
status and n_inliers exactly, Rt and info within tolerances; repeat runs bit-identical, other seeds other draws;
refusals and status 3.  End to end: the synthetic room of tests/test_gpu_indoor_registration.py with solver "fgr"."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import fgr_ref as fr
from tests import indoor_reg_ref as ir
from tests.test_gpu_indoor_registration import SCENE, _room_tree
from tests.test_gpu_registration import _rigid
from tests.util_gpu import dev
from usip_b200 import _lib, ops
from usip_b200._lib import UsipB200Error
from usip_b200.evaluation import indoor_registration as idr
from usip_b200.evaluation import registration as reg

pytestmark = pytest.mark.gpu

# Tolerance against the restatement: 4x the worst Rt error measured on an H100 80GB HBM3 (700 W) over this file's
# cases, 3.58e-12 absolute in the room scene (4.9e-14 in the synthetic pairs): the sin / cos of the pose update are
# CUDA's on the device and libm's here, and 640 iterations on a few correspondences carry their last-bit differences.
# info measured exact: it sums the raw fragment-1 points of the inliers, so it is bit-exact whenever n_inliers agrees.
RT_TOL = 1.5e-11
INFO_TOL = 0.0
WORST = {"Rt": 0.0, "info": 0.0}


def d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


# ----------------------------------------------------------------------------------------------- mutual matches
def _mutual_case(desc, count, pairs, ks):
    S, L, D = desc.shape
    m, n = ops.desc_match_mutual(d(desc), d(count), d(pairs), ks)
    m, n = m.cpu().numpy(), n.cpu().numpy()
    fw, nf = ops.desc_match(d(desc), d(count), d(pairs), ks, 1)
    bw, nb = ops.desc_match(d(desc), d(count), d(pairs[:, ::-1]), ks, 1)
    fw, bw, nf, nb = fw.cpu().numpy(), bw.cpu().numpy(), nf.cpu().numpy(), nb.cpu().numpy()
    for p, (a, b) in enumerate(pairs):
        for k, K in enumerate(ks):
            na, nb_ = min(K, count[a], L), min(K, count[b], L)
            ref = fr.mutual_ref(desc[a, :na], desc[b, :nb_])
            assert n[p, k] == len(ref), (p, K)
            np.testing.assert_array_equal(m[p, k, :n[p, k]], ref)
            both = {tuple(x) for x in fw[p, k, :nf[p, k]]} & {(i, j) for j, i in bw[p, k, :nb[p, k]]}
            assert sorted(both) == [tuple(x) for x in ref]
    return m, n


def test_mutual_matches_ties_nan_and_counts():
    rng = np.random.RandomState(0)
    S, L, D = 6, 64, 8
    desc = rng.randint(0, 3, (S, L, D)).astype(np.float32)               # three levels: many exact ties
    desc[1, 5] = np.nan
    desc[2, :, 3] = np.nan                                                # every d^2 of scan 2 is NaN
    desc[3, 7, 0] = np.inf
    count = np.array([64, 40, 64, 10, 0, 33], np.int32)
    pairs = np.array([[0, 1], [1, 0], [0, 2], [2, 3], [3, 0], [4, 0], [5, 5], [0, 0]], np.int32)
    m, n = _mutual_case(desc, count, pairs, [1, 16, 40, 64, 100])
    assert n[5].sum() == 0 and (n[6] > 0).all()


def test_mutual_matches_edge_shapes():
    rng = np.random.RandomState(1)
    _mutual_case(rng.normal(size=(3, 1, 1)).astype(np.float32), np.array([1, 1, 0], np.int32),
                 np.array([[0, 1], [1, 2]], np.int32), [1, 5])
    desc = rng.normal(size=(2, 1024, 512)).astype(np.float32)
    desc[1, :700] = desc[0, 300:1000] + rng.normal(scale=0.01, size=(700, 512))
    _, n = _mutual_case(desc, np.array([1024, 1000], np.int32), np.array([[0, 1]], np.int32), [1024])
    assert n[0, 0] >= 700
    desc = rng.randint(0, 5, (2, 300, 1)).astype(np.float32)             # D = 1: ties everywhere
    _mutual_case(desc, np.array([300, 250], np.int32), np.array([[0, 1], [1, 0]], np.int32), [50, 300])


def test_mutual_refusals():
    desc, count, pairs = d(np.zeros((2, 4, 8), np.float32)), d(np.array([4, 4], np.int32)), d(np.array([[0, 1]], np.int32))
    with pytest.raises(UsipB200Error, match="USIP_REG_MAX_DIM"):
        ops.desc_match_mutual(d(np.zeros((2, 4, 513), np.float32)), count, pairs, [4])
    with pytest.raises(UsipB200Error, match="shared memory"):
        ops.desc_match_mutual(d(np.zeros((2, 1025, 8), np.float32)), count, pairs, [4])
    with pytest.raises(UsipB200Error, match="ascend"):
        ops.desc_match_mutual(desc, count, pairs, [8, 4])


# ----------------------------------------------------------------------------------------------- usip_fgr_f64
def _scans(rng, specs, L):
    """specs: (n1, n2, kind) per pair -> xyz (2P, L, 3), desc (2P, L, 4), count, pairs.  Scan 2p+1 is a rigid copy of
    scan 2p's rows in shuffled order; kind 'clean' keeps every descriptor, 'half' re-draws half of them, 'random' draws
    them all, 'flat' puts every point of both scans at one place."""
    P = len(specs)
    xyz = np.zeros((2 * P, L, 3), np.float32)
    desc = np.zeros((2 * P, L, 4), np.float32)
    count = np.zeros(2 * P, np.int32)
    for p, (n1, n2, kind) in enumerate(specs):
        a = rng.uniform(-3, 3, (L, 3))
        T = _rigid(rng, 4.0)
        perm = rng.permutation(L)
        b = (a[perm] - T[:, 3]) @ T[:, :3]                               # a = R b + t
        da = np.concatenate([a, rng.normal(size=(L, 1))], 1)
        db = da[perm].copy()
        if kind == "half":
            db[rng.rand(L) < 0.5] = rng.uniform(-3, 3, (1, 4))
        if kind == "random":
            db = rng.normal(size=(L, 4)) * 3
        if kind == "flat":
            a[:] = 1.5
            b[:] = -0.5
        xyz[2 * p], xyz[2 * p + 1] = a, b
        desc[2 * p], desc[2 * p + 1] = da, db
        count[2 * p], count[2 * p + 1] = n1, n2
    pairs = np.arange(2 * P, dtype=np.int32).reshape(P, 2)
    return xyz, desc, count, pairs


def _check_fgr(xyz, desc, count, pairs, ks, seed, thr=0.2):
    L = xyz.shape[1]
    m, n = ops.desc_match_mutual(d(desc), d(count), d(pairs), ks)
    out = ops.fgr(d(xyz), d(count), d(pairs), ks, m, n, thr, seed)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    m, n = m.cpu().numpy(), n.cpu().numpy()
    seen = set()
    for p, (a, b) in enumerate(pairs):
        for k, K in enumerate(ks):
            na, nb = min(K, count[a], L), min(K, count[b], L)
            ref = fr.fgr_ref(xyz[a, :na], xyz[b, :nb], m[p, k, :n[p, k]], seed, thr)
            assert got["status"][p, k] == ref["status"], (p, K)
            assert got["n_tuples"][p, k] == ref["n_tuples"], (p, K)
            x1 = xyz[a, m[p, k, :n[p, k], 0]].astype(np.float64)
            x2 = xyz[b, m[p, k, :n[p, k], 1]].astype(np.float64)
            if len(x1) and np.all(np.isfinite(ref["Rt"])):
                res = np.sqrt(((x1 - (x2 @ ref["Rt"][:, :3].T + ref["Rt"][:, 3])) ** 2).sum(1))
                assert not np.any(np.abs(res - thr) < 1e-9), "a residual on the threshold: change the data"
            assert got["n_inliers"][p, k] == ref["n_inliers"], (p, K)
            e_rt = np.abs(got["Rt"][p, k] - ref["Rt"]).max()
            e_info = np.abs(got["info"][p, k] - ref["info"]).max() / max(1.0, np.abs(ref["info"]).max())
            WORST["Rt"], WORST["info"] = max(WORST["Rt"], e_rt), max(WORST["info"], e_info)
            assert e_rt <= RT_TOL and e_info <= INFO_TOL, (p, K, e_rt, e_info)
            seen.add(int(ref["status"]))
    print("fgr worst error vs restatement: Rt %.3g, info %.3g (relative)" % (WORST["Rt"], WORST["info"]))
    return got, seen


def test_fgr_matches_restatement():
    rng = np.random.RandomState(5)
    L = 256
    specs = [(256, 256, "clean"), (200, 256, "half"), (256, 180, "half"), (256, 256, "random"), (2, 256, "clean"),
             (120, 90, "clean"), (256, 256, "flat"), (0, 50, "clean")]
    xyz, desc, count, pairs = _scans(rng, specs, L)
    got, seen = _check_fgr(xyz, desc, count, pairs, [2, 30, 128, 256], seed=7)
    assert {0, 1, 4} <= seen
    assert got["n_tuples"][0, 3] == fr.TUPLE_CAP                          # 256 clean matches saturate the cap


def test_fgr_full_rows_and_seeds():
    rng = np.random.RandomState(6)
    xyz, desc, count, pairs = _scans(rng, [(1024, 1024, "half"), (1024, 1000, "clean")], 1024)
    ks = [1024]
    got, _ = _check_fgr(xyz, desc, count, pairs, ks, seed=11)
    m, n = ops.desc_match_mutual(d(desc), d(count), d(pairs), ks)
    args = (d(xyz), d(count), d(pairs), ks, m, n, 0.2)
    again = {k: v.cpu().numpy() for k, v in ops.fgr(*args, 11).items()}
    for k in got:
        assert np.array_equal(got[k].view(np.uint8), again[k].view(np.uint8)), k
    other = {k: v.cpu().numpy() for k, v in ops.fgr(*args, 12).items()}
    assert other["n_tuples"][0, 0] != got["n_tuples"][0, 0] or not np.array_equal(other["Rt"], got["Rt"])


def test_fgr_status3_and_refusals():
    rng = np.random.RandomState(7)
    xyz, desc, count, pairs = _scans(rng, [(40, 40, "clean")], 64)
    m, n = ops.desc_match_mutual(d(desc), d(count), d(pairs), [40])
    bad = m.clone()
    bad[0, 0, 3, 1] = 40                                                  # a positive row beyond K = 40
    out = ops.fgr(d(xyz), d(count), d(pairs), [40], bad, n)
    assert out["status"][0, 0].item() == 3 and out["n_inliers"][0, 0].item() == 0
    assert not out["Rt"].any() and not out["info"].any()
    X, C, Pr = d(xyz), d(count), d(pairs)
    with pytest.raises(UsipB200Error, match="threshold"):
        ops.fgr(X, C, Pr, [40], m, n, 0.0)
    with pytest.raises(UsipB200Error, match="ascend"):
        ops.fgr(X, C, Pr, [40, 40], m.repeat(1, 2, 1, 1).contiguous(), n.repeat(1, 2).contiguous())
    big = torch.zeros((1, 1, 1025, 2), dtype=torch.int32, device=dev())
    with pytest.raises(UsipB200Error, match="match list"):
        ops.fgr(X, C, Pr, [40], big, n)
    with pytest.raises(UsipB200Error, match="shared memory"):
        ops.fgr(d(np.zeros((2, 1025, 3), np.float32)), C, Pr, [40], m, n)
    with pytest.raises(ValueError):
        ops.fgr(X, C, Pr, [40, 50], m, n)
    st = torch.full((1, 1), 7, dtype=torch.int32, device=dev())
    rc = _lib.load().usip_fgr_f64(ops._p(X), ops._p(C), 2, 64, ops._p(Pr), 1, (ctypes.c_int32 * 1)(40), 1, ops._p(m),
                                  ops._p(n), 64, 0, -1.0, ops._p(out["Rt"]), ops._p(st), ops._p(st), ops._p(out["info"]),
                                  ops._p(st), None)
    assert rc == -1 and b"threshold" in _lib.load().usip_last_error()
    torch.cuda.synchronize()
    assert st.item() == 7                                                  # nothing ran


# ----------------------------------------------------------------------------------------------- end to end
def test_end_to_end_room_fgr(tmp_path):
    npy, gt, tree, D, entries = _room_tree(str(tmp_path))
    opt = reg.descriptor_opt("redwood", input_pc_num=1024, batch_size=2)
    ev = idr.IndoorRegistration.redwood(npy, gt, opt, scenes=[(SCENE, 6)])
    ev.read_descriptor_tree(tree, D)
    ks = [60, 120]
    res = ev.score(ks, pairs="all", seed=3, solver="fgr")
    r = res.per_scene[SCENE]
    assert len(r["pairs"]) == 15 and r["Rt"].shape == (15, 2, 1, 4, 4)
    gt_far = [(i, j) for i, j, _, _ in entries if j - i > 1]
    for (K, T), (sc, line, means) in res.scores.items():
        assert T is None and sc[SCENE]["recall"] == 1.0 and sc[SCENE]["gt_num"] == len(gt_far), (K, sc[SCENE])
    gt_T = {(i, j): T for i, j, _, T in entries}
    xyz_np, count_np, desc_np = ev.xyz.cpu().numpy(), ev.count.cpu().numpy(), ev.desc.cpu().numpy()
    frags = [np.load(os.path.join(npy, SCENE, "%d.npy" % f))[:, :3] for f in range(6)]
    room_err = 0.0
    for p, (i, j) in enumerate(r["pairs"]):
        for k, K in enumerate(ks):
            na, nb = min(K, count_np[i]), min(K, count_np[j])
            m = fr.mutual_ref(desc_np[i, :na], desc_np[j, :nb])
            assert r["n_matches"][p, k] == len(m)
            ref = fr.fgr_ref(xyz_np[i, :na], xyz_np[j, :nb], m, 3, 0.2)
            assert r["status"][p, k, 0] == ref["status"]
            n = ref["n_inliers"] if ref["status"] == 0 else 0
            assert r["n_inliers"][p, k, 0] == n and r["n_info"][p, k, 0] == ref["n_inliers"]
            np.testing.assert_array_equal(r["info"][p, k, 0], ref["info"])
            ratio = n / len(m) if len(m) else float("nan")
            assert (r["inlier_ratio"][p, k, 0] > 0.025) == (ratio > 0.025)
            if ref["status"] == 0:
                room_err = max(room_err, np.abs(r["Rt"][p, k, 0, :3] - ref["Rt"]).max())
            if (i, j) in gt_T and ref["status"] == 0:
                assert np.abs(r["Rt"][p, k, 0] - gt_T[(i, j)]).max() < 1e-3, (i, j, K)
            if ratio > 0.025:
                al = ir.overlap_ref(frags[i], frags[j], r["Rt"][p, k, 0, :3]) / len(frags[i])
                assert r["aligned"][p, k, 0] == al and r["accepted"][p, k, 0] == (al > 0.23)
            else:
                assert not r["accepted"][p, k, 0]
    print("fgr worst Rt error vs restatement, room: %.3g" % room_err)
    assert room_err <= RT_TOL
    out = os.path.join(str(tmp_path), "logs")
    ev.write_registration_logs(out, 120)
    sc, line, _ = ev.score_logs(out)
    direct = res.scores[(120, None)][0][SCENE]
    for key in ("recall", "precision", "good", "gt_num", "rs_num"):
        assert sc[SCENE][key] == direct[key]
    lines = res.lines()
    assert lines[-1].startswith("K=120 FGR redwood: Mean registration recall: 1.000000")
    lite = ev.score([120], overlap_threshold=None, pairs="gt", seed=3, solver="fgr")
    assert lite.scores[(120, None)][0][SCENE]["recall"] == 1.0


def test_fast_global_registration_equals_batched_path():
    rng = np.random.RandomState(9)
    xyz, desc, count, pairs = _scans(rng, [(300, 260, "half")], 300)
    T = idr.fast_global_registration(xyz[0], desc[0], xyz[1, :260], desc[1, :260], seed=2)
    m, n = ops.desc_match_mutual(d(desc), d(count), d(pairs), [300])
    out = ops.fgr(d(xyz), d(count), d(pairs), [300], m, n, 0.2, 2)
    assert out["status"][0, 0].item() == 0
    assert np.array_equal(T[:3], out["Rt"][0, 0].cpu().numpy()) and np.array_equal(T[3], [0, 0, 0, 1])
    Tc = idr.fast_global_registration(d(xyz[0]), d(desc[0]), d(xyz[1, :260]), d(desc[1, :260]), seed=2)
    assert np.array_equal(T, Tc)
    few = idr.fast_global_registration(xyz[0, :2], desc[0, :2], xyz[1, :5], desc[1, :5])
    np.testing.assert_array_equal(few[:3, 3], fr.seq_mean(xyz[0, :2]) - fr.seq_mean(xyz[1, :5]))
