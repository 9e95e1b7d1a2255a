"""Fast Global Registration on the host: the restatement tests/fgr_ref.py (the rotation, the Cholesky solve, recovery of
known motions with and without outliers, the tuple rules and the status rules) and the FGR solver's host logic in
usip_b200.evaluation.indoor_registration (solver validation, lines / to_dict / write_registration_logs, CLI refusals).
No GPU."""
import json

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from tests import fgr_ref as fr
from usip_b200.evaluation import indoor_registration as idr

# Recovery tolerances, set from runs of the restatement: on noise-free correspondences (fp32 points, rotations up to 60
# degrees, translations up to the 7 m scene diameter) the worst error seen was 3.0e-8 in R and t, from the fp32 rounding
# of the inputs; with half the correspondences replaced by random ones it was 1.1e-3 (the Geman-McClure weight at the
# final scale 0.05 of the normalised extent still gives outliers some pull).
NOISE_FREE_TOL = 2e-7
OUTLIER_TOL = 5e-3


def _motion(rng, deg, diameter=7.0):
    axis = rng.normal(size=3)
    R = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(deg)).as_matrix()
    t = rng.uniform(-1, 1, 3)
    return R, t / np.linalg.norm(t) * rng.uniform(0, diameter)


def _case(rng, n, deg, outliers=0.0):
    x2 = rng.uniform(-3.5, 3.5, (n, 3)).astype(np.float32)
    R, t = _motion(rng, deg)
    x1 = (x2.astype(np.float64) @ R.T + t).astype(np.float32)
    m = np.stack([np.arange(n), np.arange(n)], 1)
    k = int(round(outliers * n))
    m[:k, 1] = rng.randint(0, n, k)
    return x1, x2, m, R, t


# ----------------------------------------------------------------------------------------------- pieces
def test_rotation_is_zyx_euler():
    rng = np.random.RandomState(0)
    for _ in range(50):
        xi = list(rng.uniform(-1.5, 1.5, 6))
        D = fr.delta_matrix(xi)
        R = Rotation.from_euler("ZYX", [xi[2], xi[1], xi[0]]).as_matrix()
        np.testing.assert_allclose(D[:, :3], R, atol=1e-15, rtol=0)
        assert list(D[:, 3]) == xi[3:]


def test_cholesky_solve_matches_linalg_on_spd():
    rng = np.random.RandomState(1)
    for _ in range(50):
        G = rng.normal(size=(9, 6))
        A = G.T @ G + 0.1 * np.eye(6)
        b = rng.normal(size=6)
        S = np.concatenate([[A[a, c] for a, c in fr.UPPER], b])
        np.testing.assert_allclose(fr.cholesky_solve(S), np.linalg.solve(A, -b), rtol=1e-9, atol=1e-12)
    assert fr.cholesky_solve(np.zeros(27)) is None                            # pivot 0
    S = np.concatenate([[np.diag([1.0, 1, -1, 1, 1, 1])[a, c] for a, c in fr.UPPER], np.ones(6)])
    assert fr.cholesky_solve(S) is None                                       # pivot < 0
    S[0] = np.inf
    assert fr.cholesky_solve(S) is None                                       # not finite


def test_reduction_order_is_the_headers():
    rng = np.random.RandomState(2)
    tm = rng.normal(size=(700, 27)) * 10.0 ** rng.randint(-8, 8, (700, 27))
    got = fr.reduce27(tm)
    acc = np.zeros((256, 27))
    for k in range(700):
        acc[k % 256] = acc[k % 256] + tm[k]
    for w in range(8):
        for o in (16, 8, 4, 2, 1):
            v = acc[32 * w:32 * w + 32].copy()
            acc[32 * w:32 * w + 32] = v + v[np.arange(32) ^ o]
    ref = acc[0].copy()
    for w in range(1, 8):
        ref = ref + acc[32 * w]
    np.testing.assert_array_equal(got, ref)


# ----------------------------------------------------------------------------------------------- recovery
@pytest.mark.parametrize("deg", [0, 5, 30, 60])
def test_recovers_noise_free_motion(deg):
    rng = np.random.RandomState(10 + deg)
    for n in (40, 300):
        x1, x2, m, R, t = _case(rng, n, deg)
        r = fr.fgr_ref(x1, x2, m, seed=deg)
        assert r["status"] == 0 and r["n_inliers"] == n
        assert np.abs(r["Rt"][:, :3] - R).max() < NOISE_FREE_TOL
        assert np.abs(r["Rt"][:, 3] - t).max() < NOISE_FREE_TOL


@pytest.mark.parametrize("deg", [10, 45, 60])
def test_recovers_motion_with_half_outliers(deg):
    rng = np.random.RandomState(20 + deg)
    x1, x2, m, R, t = _case(rng, 400, deg, outliers=0.5)
    r = fr.fgr_ref(x1, x2, m, seed=1)
    assert r["status"] == 0 and r["n_inliers"] >= 200
    assert np.abs(r["Rt"][:, :3] - R).max() < OUTLIER_TOL
    assert np.abs(r["Rt"][:, 3] - t).max() < OUTLIER_TOL


# ----------------------------------------------------------------------------------------------- tuples
def test_tuple_boundaries_are_strict():
    li = np.ones((1, 3))
    assert not fr.accept(li, li * fr.SIM)[0]                                  # li 0.95f == lj: out
    assert not fr.accept(li, li / fr.SIM)[0]                                  # lj == li / 0.95f: out
    assert fr.accept(li, np.nextafter(li * fr.SIM, 2.0))[0]
    assert fr.accept(li, np.nextafter(li / fr.SIM, 0.0))[0]
    assert not fr.accept(np.zeros((1, 3)), np.zeros((1, 3)))[0]               # a repeated index: zero edges
    assert fr.SIM == float(np.float32(0.95)) != 0.95


def test_tuples_repeats_cap_and_order():
    rng = np.random.RandomState(3)
    x1, x2, m, _, _ = _case(rng, 150, 20)
    m1, m2, scale, _ = fr.normalise(x1, x2)
    p, q = (x1.astype(np.float64) - m1) / scale, (x2.astype(np.float64) - m2) / scale
    n_t, mult, kept = fr.tuples(p, q, seed=5)
    idx = fr.tuple_indices(5, 150, 100 * 150)
    distinct = (idx[:, 0] != idx[:, 1]) & (idx[:, 1] != idx[:, 2]) & (idx[:, 2] != idx[:, 0])
    assert n_t == fr.TUPLE_CAP == len(kept)                                   # every distinct triple passes: capped
    assert np.array_equal(kept, np.flatnonzero(distinct)[:fr.TUPLE_CAP])      # the first ones in trial order
    assert (~distinct).any() and kept[-1] < len(idx) - 1
    assert mult.sum() == 3 * n_t and np.array_equal(mult, np.bincount(idx[kept].ravel(), minlength=150))
    n_small, mult_small, _ = fr.tuples(p[:20], q[:20], seed=5)               # 2000 trials: under the cap
    assert n_small < fr.TUPLE_CAP and mult_small.sum() == 3 * n_small
    assert fr.tuples(p, q, seed=6)[1].tolist() != mult.tolist()               # another seed, other draws


def test_tuple_indices_are_rand_mod_n():
    idx = fr.tuple_indices(0, 7, 5000)
    assert idx.min() == 0 and idx.max() == 6
    assert not np.array_equal(fr.tuple_indices(0, 7, 50), fr.tuple_indices(1, 7, 50))


# ----------------------------------------------------------------------------------------------- status rules
def test_too_few_matches_give_identity_and_mean_difference():
    rng = np.random.RandomState(4)
    f1 = rng.uniform(-1, 1, (30, 3)).astype(np.float32)
    f2 = rng.uniform(-1, 1, (25, 3)).astype(np.float32)
    for k in range(3):
        m = np.stack([np.arange(k), np.arange(k)], 1)
        r = fr.fgr_ref(f1, f2, m)
        assert r["status"] == 1 and r["n_tuples"] == 0
        assert np.array_equal(r["Rt"][:, :3], np.eye(3))
        np.testing.assert_array_equal(r["Rt"][:, 3], fr.seq_mean(f1) - fr.seq_mean(f2))
    r = fr.fgr_ref(f1, f2, np.array([[0, 0], [1, 30]]))
    assert r["status"] == 3 and not r["Rt"].any()


def test_coincident_points_are_degenerate():
    f = np.full((12, 3), 0.25, np.float32)
    r = fr.fgr_ref(f, f, np.stack([np.arange(12), np.arange(12)], 1))
    assert r["status"] == 4 and r["n_tuples"] == 0 and r["scale"] == 0.0
    assert np.array_equal(r["Rt"], np.eye(3, 4)) and r["n_inliers"] == 12


def test_mutual_ref_rules():
    da = np.array([[0.0], [1.0], [1.0], [5.0]], np.float32)
    dp = np.array([[1.0], [0.1], [np.nan], [5.0]], np.float32)
    m = fr.mutual_ref(da, dp)
    assert m.tolist() == [[0, 1], [1, 0], [3, 3]]                             # anchor 2 ties with 1 and loses
    assert fr.mutual_ref(da[:0], dp).shape == (0, 2)


# ----------------------------------------------------------------------------------------------- host logic
def _T(t=(0, 0, 0)):
    T = np.eye(4)
    T[:3, 3] = t
    return T


class _FakeFGR(idr.IndoorRegistration):
    """One scene's worth of IndoorRegistration state with _register and _overlap replaced by fixed answers."""

    def __init__(self):
        self.dataset = "redwood"
        self.scenes = ["s"]
        self.frames_of = {"s": [0, 1, 2, 3]}
        self.gt = {"s": (np.array([[0, 2, 4], [1, 3, 4]]), np.stack([_T(), _T((1, 0, 0))]),
                         np.stack([np.eye(6), np.eye(6)]))}
        self.xyz = torch.zeros(1)
        self.result = None
        self.calls = []

    def _register(self, scene, fp, ks, ts, seed, uniforms, solver="ransac"):
        self.calls.append((solver, list(ts), seed))
        P, nK, nT = len(fp), len(ks), len(ts)
        n_inl = np.full((P, nK, nT), 30, np.int32)
        return {"n_matches": np.full((P, nK), 100, np.int32), "n_inliers": n_inl, "n_info": n_inl.copy(),
                "Rt": np.broadcast_to(np.eye(3, 4), (P, nK, nT, 3, 4)).copy(), "status": np.zeros((P, nK, nT), np.int32),
                "info": np.broadcast_to(np.eye(6), (P, nK, nT, 6, 6)).copy()}

    def _overlap(self, scene, fp, Rt, candidate):
        return np.full(int(candidate.sum()), 0.5)


def test_fgr_solver_host_logic(tmp_path):
    ev = _FakeFGR()
    with pytest.raises(ValueError, match="solver"):
        ev.score([8], solver="icp")
    with pytest.raises(ValueError, match="max_trials"):
        ev.score([8], [1000], solver="fgr")
    res = ev.score([8, 16], solver="fgr", seed=4)
    assert ev.calls[-1] == ("fgr", [None], 4)
    assert res.solver == "fgr" and res.max_trials == [None] and list(res.scores) == [(8, None), (16, None)]
    lines = res.lines()
    assert lines[0] == "K=8 FGR redwood: --- s" and lines[-1].startswith("K=16 FGR redwood: Mean registration recall")
    assert not any("maxTrials" in v for v in lines)
    d = json.loads(json.dumps(res.to_dict()))
    assert d["solver"] == "fgr" and d["max_trials"] is None and [r["max_trials"] for r in d["runs"]] == [None, None]
    assert d["runs"][0]["log_entries"] == {"s": 6}
    sc = res.scores[(16, None)][0]["s"]
    assert sc["gt_num"] == 2 and sc["good"] == 1 and sc["recall"] == 0.5       # (0, 2) right; (1, 3) misses t_gt
    ev.write_registration_logs(str(tmp_path), 16)
    logs = idr.read_registration_log(str(tmp_path / "s.log"))
    assert len(logs["head"]) == 6 and (logs["inlier_num"] == 30).all() and np.allclose(logs["inlier_ratio"], 0.3)
    with pytest.raises(ValueError):
        ev.write_registration_logs(str(tmp_path), 16, 1000)
    ransac = ev.score([8])
    assert ev.calls[-1][:2] == ("ransac", list(idr.DEFAULT_MAX_TRIALS)) and ransac.solver == "ransac"
    assert ransac.to_dict()["max_trials"] == list(idr.DEFAULT_MAX_TRIALS) and "maxTrials=1000" in ransac.lines()[0]
    with pytest.raises(ValueError):
        ev.write_registration_logs(str(tmp_path), 8)


def test_fgr_cli_refusals(tmp_path):
    base = ["redwood", "--root", str(tmp_path), "--gt-root", str(tmp_path), "--descriptor-tree", str(tmp_path)]
    with pytest.raises(SystemExit):
        idr.main(base + ["--solver", "fgr", "--max-trials", "1000"])
    with pytest.raises(SystemExit):
        idr.main(base + ["--solver", "icp"])


def test_fast_global_registration_refusals():
    p, f = np.zeros((4, 3), np.float32), np.zeros((4, 8), np.float32)
    with pytest.raises(ValueError):
        idr.fast_global_registration(p, f[:3], p, f)
    with pytest.raises(ValueError):
        idr.fast_global_registration(p, f, p, f[:, :4])
    with pytest.raises(ValueError):
        idr.fast_global_registration(np.zeros((1025, 3)), np.zeros((1025, 8)), p, f)
    with pytest.raises(ValueError):
        idr.fast_global_registration(p, np.zeros((4, 513)), p, np.zeros((4, 513)))
