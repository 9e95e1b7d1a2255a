"""CPU checks of the handcrafted baselines: the numpy restatement (tests/handcrafted_ref.py) on hand-built clouds with
known answers, the selection's contract, and the refusals of the C ABI, the detectors, Repeatability.detect and the
command lines (none of which reaches a kernel)."""
import ctypes

import numpy as np
import pytest

from tests import handcrafted_ref as H


def corner_cloud(seed=0, n=(700, 900, 800), ext=1.0):
    """Three faces of a box meeting at the origin, uniformly sampled with unequal densities, plus the corner itself."""
    rng = np.random.default_rng(seed)
    pts = [np.zeros((1, 3))]
    for ax, m in zip(range(3), n):
        p = rng.uniform(0, ext, (m, 3))
        p[:, ax] = 0
        pts.append(p)
    return np.concatenate(pts).astype(np.float32)


def plane_cloud(seed=0, n=2000):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1, 1, (n, 3))
    p[:, 2] = 0.25
    return p.astype(np.float32)


def _nearest_flag(P, flag):
    return np.sqrt((P[flag].astype(np.float64) ** 2).sum(axis=1)).min()


@pytest.mark.parametrize("seed", [0, 1])
def test_corner_is_a_keypoint(seed):
    P = corner_cloud(seed)
    assert _nearest_flag(P, H.iss_flags(P, 0.25, 0.25, 0.975, 0.975, 5)) < 0.2
    assert _nearest_flag(P, H.harris_flags(P, 0.25, 0.001)) < 0.2


def test_flat_plane_has_none():
    P = plane_cloud()
    sal = H.iss_saliency(P, 0.2, 0.975, 0.975, 5)[0]
    assert (sal == 0).all()
    assert not H.iss_flags(P, 0.2, 0.2, 0.975, 0.975, 5).any()
    R = H.harris_response(P, 0.2)[0]
    assert np.nanmax(np.abs(R)) < 1e-12
    assert not H.harris_flags(P, 0.2, 0.001).any()


def test_duplicated_points_tie_and_both_stay():
    P = corner_cloud(0)
    for flags in (lambda Q: H.iss_flags(Q, 0.25, 0.25, 0.975, 0.975, 5), lambda Q: H.harris_flags(Q, 0.25, 0.001)):
        i = np.flatnonzero(flags(P))[0]
        Q = np.concatenate([P, P[i:i + 1]])
        f = flags(Q)
        assert f[i] and f[-1]


def test_nan_row_is_never_a_neighbour():
    P = corner_cloud(0)
    Q = P.copy()
    Q[5] = [np.nan, 0, 0]
    ptr, idx = H.neighbours(Q, 0.25)
    assert ptr[6] == ptr[5] and 5 not in set(idx.tolist())
    ptr0, idx0 = H.neighbours(P, 0.25)
    cnt0, cnt = np.diff(ptr0), np.diff(ptr)
    other = np.arange(len(P)) != 5
    had5 = np.array([5 in set(idx0[ptr0[i]:ptr0[i + 1]].tolist()) for i in range(len(P))]) & other
    assert cnt[5] == 0 and had5.any()
    np.testing.assert_array_equal(cnt[~had5 & other], cnt0[~had5 & other])
    np.testing.assert_array_equal(cnt[had5], cnt0[had5] - 1)
    assert not H.iss_flags(Q, 0.25, 0.25, 0.975, 0.975, 5)[5] and not H.harris_flags(Q, 0.25, 0.001)[5]


def test_neighbour_rule_is_fp32_inclusive():
    r = np.float32(0.1)
    P = np.array([[0, 0, 0], [0.1, 0, 0], [0.1000001, 0, 0], [0, 0.06, 0.08]], np.float32)
    ptr, idx = H.neighbours(P, r)
    d2 = lambda a, b: (lambda d: (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])(P[a] - P[b])
    expect = [j for j in range(4) if d2(j, 0) <= r * r]
    assert idx[ptr[0]:ptr[1]].tolist() == expect and 1 in expect and 2 not in expect


@pytest.mark.parametrize("count", [0, 5, 40])
def test_selection_contract(count):
    N, L = 100, 20
    rng = np.random.default_rng(count)
    flag = np.zeros(N, bool)
    flag[rng.choice(N, count, replace=False)] = True
    order, c = H.select(flag, N, L, seed=3, step=2, cloud=1)
    assert c == count and len(order) == L
    head = order[:min(count, L)]
    assert flag[head].all() and len(set(head.tolist())) == len(head)
    tail = order[min(count, L):]
    assert len(set(tail.tolist())) == len(tail)
    again, _ = H.select(flag, N, L, seed=3, step=2, cloud=1)
    np.testing.assert_array_equal(order, again)
    other, _ = H.select(flag, N, L, seed=3, step=3, cloud=1)
    assert not np.array_equal(order, other) or count >= L and L == count


# ----------------------------------------------------------------------------------------------- refusals
def _lib():
    from usip_b200 import _lib
    return _lib.load()


def test_abi_refusals():
    lib = _lib()
    P = ctypes.c_void_p(0x100000)
    G = ctypes.c_void_p(0x200000)
    big = 1 << 40
    B, N = 2, 1000
    assert lib.usip_hc_grid_scratch_bytes(B, N) > 0
    assert lib.usip_hc_grid_scratch_bytes(1, (1 << 20) + 1) == 0
    assert lib.usip_hc_grid_scratch_bytes(0, 10) == 0
    assert lib.usip_hc_grid_build(P, G, big, 1, (1 << 20) + 1, None) != 0
    assert lib.usip_hc_grid_build(P, G, 16, B, N, None) != 0                          # grid too small
    assert lib.usip_hc_grid_build(P, ctypes.c_void_p(0x200004), big, B, N, None) != 0  # misaligned
    iss = lambda r=2.0, g1=0.975, g2=0.975, mn=5: lib.usip_iss_saliency_f64(P, G, big, B, N, r, g1, g2, mn, P, None,
                                                                              None, None)
    for kw in ({"r": 0.0}, {"r": -1.0}, {"r": float("nan")}, {"r": float("inf")}, {"g1": 0.0}, {"g1": 1.5},
               {"g2": float("nan")}, {"mn": 0}):
        assert iss(**kw) != 0, kw
        assert lib.usip_last_error().decode().startswith("iss_saliency")
    for r in (0.0, float("nan")):
        assert lib.usip_harris3d_response_f64(P, G, big, B, N, r, P, P, None, None) != 0
        assert lib.usip_hc_nonmax(P, G, big, B, N, P, r, 0.0, 1, 1, P, None, None) != 0
    assert lib.usip_hc_nonmax(P, G, big, B, N, P, 1.0, float("nan"), 1, 1, P, None, None) != 0
    assert lib.usip_hc_nonmax(P, G, big, B, N, P, 1.0, 0.0, 1, 0, P, None, None) != 0
    for L in (0, N + 1, 5000):
        assert lib.usip_hc_select(None, B, 8000 if L == 5000 else N, L, 0, 0, P, P, None) != 0


def test_detector_refusals():
    from usip_b200.evaluation.handcrafted import Harris3DDetector, IssDetector
    for kw in ({"salient_radius": 0}, {"non_max_radius": float("nan")}, {"gamma_21": 0}, {"gamma_32": 1.01},
               {"min_neighbors": 0}, {"min_neighbors": 2.5}):
        with pytest.raises(ValueError):
            IssDetector(**kw)
    for kw in ({"radius": -1}, {"radius": float("inf")}, {"threshold": float("nan")}):
        with pytest.raises(ValueError):
            Harris3DDetector(**kw)


def test_detect_refuses_nms_with_a_baseline():
    from usip_b200.evaluation import repeatability as rep
    from usip_b200.evaluation.handcrafted import IssDetector, RandomDetector

    class Src:
        def __len__(self):
            return 2

        def key(self, i):
            return i

    ev = rep.Repeatability(Src(), [(0, 1)], np.zeros((1, 3, 3, 4)))
    for det in (IssDetector(), RandomDetector()):
        with pytest.raises(ValueError, match="nms_radius"):
            ev.detect(det, nms_radius=0.5)


def _exits(main, argv):
    with pytest.raises(SystemExit) as e:
        main(argv)
    return e.value.code


def test_cli_refusals(capsys):
    from usip_b200.evaluation import indoor_registration, registration, repeatability
    kitti = ["kitti", "--txt-root", "t", "--numpy-root", "n", "--calib-root", "c"]
    assert _exits(repeatability.main, kitti) == 2                                   # tsf without --checkpoint
    assert "--checkpoint" in capsys.readouterr().err
    assert _exits(repeatability.main, kitti + ["--method", "iss", "--nms-radius", "0.5"]) == 2
    assert "tsf only" in capsys.readouterr().err
    assert _exits(repeatability.main, kitti + ["--method", "iss", "--iss-gamma-21", "1.5"]) == 2
    assert "gamma_21" in capsys.readouterr().err
    assert _exits(repeatability.main, kitti + ["--method", "harris", "--harris-radius", "0"]) == 2
    assert _exits(repeatability.main, kitti + ["--method", "sift"]) == 2
    assert _exits(registration.main, kitti + ["--method", "iss"]) == 2              # no --descriptor
    assert _exits(registration.main, kitti + ["--method", "random", "--descriptor", "d", "--nms-radius", "1"]) == 2
    assert _exits(registration.main, kitti + ["--descriptor", "d"]) == 2             # tsf without --detector
    indoor = ["redwood", "--root", "r", "--gt-root", "g"]
    assert _exits(indoor_registration.main, indoor + ["--method", "harris"]) == 2
    assert _exits(indoor_registration.main, indoor + ["--method", "iss", "--iss-min-neighbors", "0",
                                                      "--descriptor", "d"]) == 2
