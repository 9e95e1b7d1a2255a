"""Host side of the registration evaluation (usip_b200.evaluation.registration) and of its float64 restatement
(tests/reg_ref.py): rotm2eul / compareTransform on hand-computed rotations, the summary's statistics and lines, the
index rule, ransac.m's sequential stop on hand-made counts, the union order, the descriptor tree and the refusals."""
import os

import numpy as np
import pytest

from tests import reg_ref as rr
from tests.test_repeatability_host import _kitti_tree
from tests.util_gpu import make_opt
from usip_b200.evaluation import registration as reg
from usip_b200.evaluation import repeatability as rep


def _rz(a):
    return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])


def _ry(a):
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1.0, 0], [-np.sin(a), 0, np.cos(a)]])


def _rx(a):
    return np.array([[1.0, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])


def test_rotm2eul_zyx():
    np.testing.assert_array_equal(reg.rotm2eul_zyx(np.eye(3)), [0, 0, 0])
    np.testing.assert_allclose(reg.rotm2eul_zyx(_rz(0.3)), [0.3, 0, 0], atol=1e-15)
    np.testing.assert_allclose(reg.rotm2eul_zyx(_ry(-0.4)), [0, -0.4, 0], atol=1e-15)
    np.testing.assert_allclose(reg.rotm2eul_zyx(_rx(1.1)), [0, 0, 1.1], atol=1e-15)
    np.testing.assert_allclose(reg.rotm2eul_zyx(_rz(0.5) @ _ry(0.2) @ _rx(-0.7)), [0.5, 0.2, -0.7], atol=1e-15)
    # pitch = +-90 degrees: cy = 0, so yaw is set to 0 and the rest goes to roll: Rz(a) Ry(90) Rx(b) = Ry(90) Rx(b - a)
    for s in (1, -1):
        R = _rz(0.3) @ _ry(s * np.pi / 2) @ _rx(0.5)
        R[0, 0] = R[1, 0] = 0.0                        # exactly singular
        e = reg.rotm2eul_zyx(R)
        assert e[0] == 0.0 and abs(e[1] - s * np.pi / 2) < 1e-15
        np.testing.assert_allclose(e[2], np.arctan2(-R[1, 2], R[1, 1]), rtol=0, atol=0)
        np.testing.assert_allclose(e[2], 0.5 - s * 0.3, atol=1e-12)


def test_compare_transform():
    T = np.concatenate([_rz(0.1), [[1.0], [2.0], [3.0]]], 1)
    E = np.concatenate([_rz(0.1) @ _ry(np.deg2rad(2.0)), [[1.0], [2.0], [3.5]]], 1)
    dt, dd = reg.compare_transform(T, E)
    assert abs(dt - 0.5) < 1e-15 and abs(dd - 2.0) < 1e-12
    assert reg.compare_transform(T, None) == (3.0, 6.0)


def _result(dt, dd, inl, npts, tc):
    a = lambda v, t=float: np.array(v, dtype=t).reshape(-1, 1, 1)
    return reg.RegistrationResult("kitti", [8], [50], 1.0, 1, a(dt), a(dd), a(inl, int), a(npts, int), a(tc, int),
                                  a([0] * len(dt), int))


def test_summary():
    r = _result([0.1, 0.3, 2.5, 3.0, 0.2], [1.0, 2.0, 1.0, 6.0, 5.5], [5, 10, 1, 0, 9], [10, 20, 10, 10, 10],
                [20, 40, 51, 0, 33])
    # failures: dt > 2 (2.5, 3.0), ddeg > 5 (6.0, 5.5): three wrong
    assert r.wrong[0, 0] == 3 and abs(r.recall[0, 0] - 0.4) < 1e-15
    assert r.inlier_ratio[0, 0] == 0.5 and r.trial_count[0, 0] == 30
    assert abs(r.rte[0, 0] - 0.2) < 1e-15 and abs(r.rte_std[0, 0] - np.std([0.1, 0.3], ddof=1)) < 1e-15
    assert abs(r.rre_std[0, 0] - np.std([1.0, 2.0], ddof=1)) < 1e-15
    assert r.lines() == ["K=8 maxTrials=50 kitti: wrong counter: 3, inlier ratio 0.500000, trial count 30.000000",
                         "K=8 maxTrials=50 kitti: successful alignment RTE: 0.200000 +- 0.141421, RRE: 1.500000 +- "
                         "0.707107"]
    none = _result([3.0], [6.0], [0], [2], [0])                    # the failure values of a missing model
    assert none.wrong[0, 0] == 1 and np.isnan(none.rte[0, 0]) and np.isnan(none.inlier_ratio[0, 0])
    assert "RTE: NaN +- NaN" in none.lines()[1]
    one = _result([0.5], [1.0], [3], [3], [0])
    assert one.rte_std[0, 0] == 0.0                                 # MATLAB std of one value
    d = r.to_dict()
    assert d["wrong"] == [[3]] and d["rte"] == [[pytest.approx(0.2)]]


def test_index_rule():
    np.testing.assert_array_equal(rr.pick3([[0, 0, 0]], 3), [[0, 1, 2]])
    np.testing.assert_array_equal(rr.pick3([[0.99, 0.99, 0.99]], 3), [[2, 1, 0]])
    np.testing.assert_array_equal(rr.pick3([[0.5, 0.5, 0.0]], 3), [[1, 2, 0]])
    # n = 4: i0 = 2; i1 = floor(0.5 * 3) = 1 < 2; i2 = floor(0.6 * 2) = 1 -> steps over 1 and 2 -> 3
    np.testing.assert_array_equal(rr.pick3([[0.5, 0.5, 0.6]], 4), [[2, 1, 3]])
    u = np.nextafter(1.0, 0.0)
    for n in (3, 4, 1000, 16384):
        idx = rr.pick3([[u, u, u]], n)[0]
        assert sorted(idx) == [n - 3, n - 2, n - 1]
    got = rr.pick3(np.random.RandomState(0).rand(5000, 3), 7)
    assert (got.min() >= 0) and (got.max() < 7) and all(len(set(r)) == 3 for r in got)


def test_sequential_stop():
    # an all-inlier first trial: N = max(log(0.01) / log(eps), 10) = 10 -> ten trials, the last tie is the best
    assert rr.ransac_loop([20] * 50, 20, [100]) == [(10, 9, 20)]
    # a cap: maxTrials + 1 trials
    assert rr.ransac_loop([1] * 200, 1000, [5, 50]) == [(6, 5, 1), (51, 50, 1)]
    # a tie takes the later trial, a smaller count does not
    assert rr.ransac_loop([4, 6, 6, 5, 2] + [0] * 100, 100, [4]) == [(5, 2, 6)]
    # 50 % inliers: N = log(0.01) / log(1 - 0.125) = 34.5 -> stops after 35 trials, before the cap of 100
    assert rr.ransac_loop([50] * 200, 100, [20, 100]) == [(21, 20, 50), (35, 34, 50)]


def test_union_order():
    a = np.array([[0.0], [1], [2]], np.float32)
    p = np.array([[0.0], [1.1], [0]], np.float32)
    np.testing.assert_array_equal(rr.match_ref(a, p, 2), [[0, 0], [0, 2], [1, 0], [1, 1], [1, 2], [2, 0], [2, 1]])
    np.testing.assert_array_equal(rr.match_ref(a, p, 1), [[0, 0], [1, 1], [2, 1]])      # tie 0 / 2 -> 0
    np.testing.assert_array_equal(rr.match_ref(a, p[:1], 5), [[0, 0], [1, 0], [2, 0]])  # fewer rows than k


def test_non_finite_descriptors_order_last_by_index():
    # d^2 NaN (a NaN value) or inf (an inf value) orders as +inf, ties by index: every row still gets min(k, n) rows
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    a = np.array([[0.0, 0], [nan, 0], [1, 1]], np.float32)
    p = np.array([[inf, 0], [0.1, 0], [nan, nan]], np.float32)
    np.testing.assert_array_equal(rr.match_ref(a, p, 1), [[0, 1], [1, 0], [2, 1]])
    # anchor 0: 1, then 0 and 2 (both +inf, by index); anchor 1: all +inf -> 0, 1; anchor 2: 1, 0
    # positive 0: all +inf -> 0, 1; positive 1: 0, 2; positive 2: all +inf -> 0, 1
    np.testing.assert_array_equal(rr.match_ref(a, p, 2), [[0, 0], [0, 1], [0, 2], [1, 0], [1, 1], [1, 2], [2, 0],
                                                          [2, 1]])
    assert len(rr.match_ref(a, p[:1], 5)) == 3                      # a set smaller than k: all of its rows


def test_compare_transforms_vectorised():
    rng = np.random.RandomState(4)
    T = np.stack([np.concatenate([_rz(a) @ _ry(b) @ _rx(c), rng.rand(3, 1)], 1) for a, b, c in rng.rand(6, 3)])
    E = np.stack([np.concatenate([_rz(a) @ _ry(b) @ _rx(c), rng.rand(3, 1)], 1) for a, b, c in rng.rand(6, 3)])
    E[5, :, :3] = T[5, :, :3] @ _ry(np.pi / 2)
    has = np.array([True] * 5 + [True])
    has[2] = False
    dt, dd = reg.compare_transforms(T, E, has)
    for i in range(6):
        ref = reg.compare_transform(T[i], E[i] if has[i] else None)
        assert abs(dt[i] - ref[0]) < 1e-14 and abs(dd[i] - ref[1]) < 1e-12
    assert (dt[2], dd[2]) == (3.0, 6.0)


def test_describe_keeps_the_global_numpy_stream():
    class Draws:
        def run_model(self, pc, sn, kp):
            return np.random.randint(1 << 30)
    np.random.seed(11)
    expect = [np.random.randint(1 << 30) for _ in range(3)]
    np.random.seed(11)
    m = reg._SeededNumpy(Draws(), 5)
    got, desc = [], []
    for _ in range(3):
        desc.append(m.run_model(None, None, None))
        got.append(np.random.randint(1 << 30))
    assert got == expect                                            # the loader's stream is untouched
    m2 = reg._SeededNumpy(Draws(), 5)
    assert desc == [m2.run_model(None, None, None) for _ in range(3)]   # and the descriptor's repeats


def test_descriptor_tree_round_trip(tmp_path):
    txt, num, cal = _kitti_tree(str(tmp_path))
    ev = reg.Registration(rep.KittiRepeatability(txt, num, cal, make_opt(input_pc_num=1024, node_num=64),
                                                 device="cpu"))
    S, L, D = len(ev.ev.source), 6, 5
    rng = np.random.RandomState(1)
    import torch
    ev.xyz = torch.from_numpy(rng.rand(S, L, 3).astype(np.float32))
    ev.desc = torch.from_numpy(rng.rand(S, L, D).astype(np.float32))
    ev.count = torch.tensor([6, 2, 6, 4, 1], dtype=torch.int32)
    out = str(tmp_path / "tree")
    ev.write_descriptor_tree(out, 4)
    for i in range(S):
        path = ev.ev.source.keypoint_path(out, i)
        a = np.fromfile(path, np.float32)
        n = min(4, int(ev.count[i]))
        assert a.size == n * (3 + D)                   # Utils.load_descriptors: (3 + D)-column float32 rows
        np.testing.assert_array_equal(a.reshape(n, 3 + D), np.concatenate([ev.xyz[i, :n], ev.desc[i, :n]], 1))
    assert ev.ev.source.keypoint_path(out, 4) == os.path.join(out, "01", "000000.bin")
    xyz, desc, count = ev.xyz, ev.desc, ev.count
    ev.read_descriptor_tree(out, D)
    np.testing.assert_array_equal(ev.count.numpy(), np.minimum(count.numpy(), 4))
    for i in range(S):
        n = int(ev.count[i])
        np.testing.assert_array_equal(ev.xyz[i, :n].numpy(), xyz[i, :n].numpy())
        np.testing.assert_array_equal(ev.desc[i, :n].numpy(), desc[i, :n].numpy())
    with pytest.raises(ValueError, match="whole number"):
        ev.read_descriptor_tree(out, D + 1)
    with pytest.raises(ValueError, match="at most 1024 keypoints"):        # refused before any launch
        ev.score([8, 2048])
    with pytest.raises(ValueError, match="at most 1024 keypoints"):
        ev.run(None, None, [8, 2048])


def test_refusals():
    for ts, thr in (([100, 50], 1.0), ([50, 50], 1.0), ([0, 50], 1.0), ([50], 0.0), ([50], -1.0), ([200000], 1.0),
                    (list(range(1, 18)), 1.0), ([], 1.0)):
        with pytest.raises(ValueError):
            reg.check_trials(ts, thr)
    assert reg.check_trials((50, 100), 1.0) == [50, 100]
    with pytest.raises(ValueError):
        rep.check_sweep(list(range(1, 34)), 1.0)
    o = reg.descriptor_opt("oxford")
    assert (o.ball_radius, o.ball_nsamples, o.descriptor_len, o.surface_normal_len) == (2.0, 64, 128, 4)
