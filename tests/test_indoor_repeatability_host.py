"""Host side of the rotated ModelNet40, Redwood and 3DMatch repeatability evaluation (usip_b200.evaluation
.modelnet_test_loader / indoor_test_loader / repeatability): the gt.log and modelnet_info.mat readers, the rotated tree
writer, item naming, the parity draw order against the reference loaders' logged draws (tests/golden/
{modelnet,redwood,3dmatch}_test_clouds.npz), the detector options and the refusals.  Also the numpy Philox4x32-10 that
the subsample restatement (tests/philox_ref.py) rests on, against Random123's known-answer vectors."""
import os

import numpy as np
import pytest

from tests import philox_ref as pr
from tests.util_gpu import golden, make_opt
from usip_b200.data.kitti_detector_loader import draw_subsample
from usip_b200.evaluation import indoor_test_loader as itl
from usip_b200.evaluation import modelnet_test_loader as mtl
from usip_b200.evaluation import repeatability as rep


# ------------------------------------------------------------------ the synthetic trees of tools/make_golden.py
def redwood_test_rows(s, f):
    return 5 + (37 * f + 11 * s) % 76               # make_golden.redwood_test_rows


def modelnet_tree(root, k=4, seed=7500, rows=1300):
    names = ["obj_%04d" % i for i in range(k)]
    os.makedirs(os.path.join(root, "normal"), exist_ok=True)
    mtl.write_synthetic_modelnet40_normal(os.path.join(root, "normal"), names, rows, seed=seed)
    Rs = mtl.write_rotated_modelnet(os.path.join(root, "normal"), os.path.join(root, "rotated_tree"), seed=seed)
    return os.path.join(root, "rotated_tree"), Rs


def redwood_tree(root, pairs=None, seed=7500):
    itl.write_synthetic_redwood(os.path.join(root, "npy"), os.path.join(root, "gt"), redwood_test_rows, pairs or {},
                                seed=seed)
    return os.path.join(root, "npy"), os.path.join(root, "gt")


def match3d_tree(root, pairs=None, seed=7500, frames=(0, 10, 3), rows=1300):
    itl.write_synthetic_3dmatch(os.path.join(root, "npy"), {s: frames for s in itl.MATCH3D_SCENES}, rows, pairs or {},
                                seed=seed)
    return os.path.join(root, "npy")


def golden_listing(g):
    return {s: [str(n) for n in g["listing/" + s]] for s in itl.MATCH3D_SCENES}


# ------------------------------------------------------------------ Philox
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = pr.philox4x32_10(*[[c] for c in ctr], *key)
        assert [int(x[0]) for x in got] == list(want)


def test_subset_restatement_rules():
    scan = np.random.RandomState(0).uniform(-40, 40, (500, 3)).astype(np.float32)
    rows, nv = pr.subset_rows(scan, 100, 1, 2, 3)
    assert nv == 500 and len(set(rows)) == 100 and (np.diff(rows) > 0).all()
    rows, nv = pr.subset_rows(scan[:30], 100, 1, 2, 3)       # 30 valid: every row 3 times, then 10 of them
    assert nv == 30
    np.testing.assert_array_equal(rows[:90], np.tile(np.arange(30), 3))
    assert len(set(rows[90:])) == 10 and (np.diff(rows[90:]) > 0).all()
    rows, nv = pr.subset_rows(scan, 100, 1, 2, 3, radius=-1.0)
    assert nv == 0 and (rows == 0).all()


# ------------------------------------------------------------------ ground truth
def test_read_gt_log(tmp_path):
    p = tmp_path / "gt.log"
    p.write_text("0\t1\t5\n1 0 0 0.5\n0 1 0 -1\n0 0 1 2\n0 0 0 1\n"
                 "  3 4 5\n" + " ".join(str(v) for v in range(16)) + "\n\n")
    anc, pos, T = rep.read_gt_log(str(p))
    np.testing.assert_array_equal(anc, [0, 3])
    np.testing.assert_array_equal(pos, [1, 4])
    np.testing.assert_array_equal(T[0], [[1, 0, 0, 0.5], [0, 1, 0, -1], [0, 0, 1, 2]])
    np.testing.assert_array_equal(T[1], np.arange(12.0).reshape(3, 4))
    p.write_text("0 1 5\n" + "1 " * 16 + "\n7 8\n")          # fewer than three integers left: the end
    assert len(rep.read_gt_log(str(p))[0]) == 1
    p.write_text("0 1 5\n1 2 3\n")
    with pytest.raises(ValueError, match="16 matrix values"):
        rep.read_gt_log(str(p))
    assert len(rep.read_gt_log(str(_empty(tmp_path)))[0]) == 0


def _empty(tmp_path):
    p = tmp_path / "empty.log"
    p.write_text("")
    return p


def test_eul2rotm_by_hand():
    np.testing.assert_allclose(mtl.eul2rotm([np.pi / 2, 0, 0]), [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-15)
    np.testing.assert_allclose(mtl.eul2rotm([0, np.pi / 2, 0]), [[0, 0, 1], [0, 1, 0], [-1, 0, 0]], atol=1e-15)
    np.testing.assert_allclose(mtl.eul2rotm([0, 0, np.pi / 2]), [[1, 0, 0], [0, 0, -1], [0, 1, 0]], atol=1e-15)
    # ZYX: Rz(a) Ry(b) Rx(c); a = pi/2, c = pi/2 maps x -> y and y -> z
    R = mtl.eul2rotm([np.pi / 2, 0, np.pi / 2])
    np.testing.assert_allclose(R @ [1, 0, 0], [0, 1, 0], atol=1e-15)
    np.testing.assert_allclose(R @ [0, 1, 0], [0, 0, 1], atol=1e-15)


def test_rotated_tree_and_modelnet_info(tmp_path):
    root, Rs = modelnet_tree(str(tmp_path), k=3, rows=50)
    T = rep.read_modelnet_info(os.path.join(root, "modelnet_info.mat"))
    assert T.shape == (3, 3, 4)
    np.testing.assert_array_equal(T[:, :, :3], Rs)
    np.testing.assert_array_equal(T[:, :, 3], 0)
    rng = np.random.RandomState(7500)
    for i in range(3):
        np.testing.assert_array_equal(Rs[i], mtl.eul2rotm((rng.rand(3) - 0.5) * 2 * np.pi))
        o = np.load(os.path.join(root, "original", "%d.npy" % i))
        r = np.load(os.path.join(root, "rotated", "%d.npy" % i))
        np.testing.assert_array_equal(o, np.load(os.path.join(str(tmp_path), "normal", "obj", "obj_%04d.npy" % i)))
        assert r.dtype == np.float32
        o64 = o.astype(np.float64)
        np.testing.assert_array_equal(r, np.concatenate([o64[:, :3] @ Rs[i], o64[:, 3:6] @ Rs[i]], 1).astype(np.float32))
        # [x 1] T' (eval_rep.m's apply_transform) maps rotated back onto original
        np.testing.assert_allclose(r[:, :3].astype(np.float64) @ T[i, :, :3].T + T[i, :, 3], o[:, :3], atol=1e-6)


def test_v73_mat_is_refused(tmp_path):
    p = tmp_path / "modelnet_info.mat"
    text = b"MATLAB 7.3 MAT-file, Platform: GLNXA64, Created on: Mon Jan  1 00:00:00 2018 HDF5 schema 1.00 ."
    p.write_bytes(text.ljust(116) + b"\x00" * 8 + b"\x00\x02IM" + b"\x00" * 400)      # version 0x0200, the v7.3 header
    with pytest.raises(ValueError, match="v7.3"):
        rep.read_modelnet_info(str(p))


# ------------------------------------------------------------------ sources
def test_redwood_item_mapping(tmp_path):
    src = itl.RedwoodTestLoader(str(tmp_path), make_opt(input_pc_num=32, node_num=8))
    assert len(src) == 207
    want = {0: ("livingroom1", 0), 56: ("livingroom1", 56), 57: ("livingroom2", 0), 104: ("office1", 0),
            206: ("office2", 49)}
    for i, k in want.items():
        assert src.key(i) == k
        assert src.paths[i] == os.path.join(str(tmp_path), k[0], "%d.npy" % k[1])
    assert src.keypoint_path("/o", 57) == "/o/livingroom2/0.bin"


def test_match3d_names(tmp_path):
    assert itl.match3d_frame("cloud_bin_0.npy") == 0
    assert itl.match3d_frame("cloud_bin_123.npy") == 123
    with pytest.raises(ValueError):
        itl.match3d_frame("cloud_0.npy")
    root = match3d_tree(str(tmp_path), rows=300)
    src = itl.Match3DTestLoader(root, make_opt(input_pc_num=256, node_num=16))
    s0 = itl.MATCH3D_SCENES[0]
    assert [src.key(i) for i in range(3)] == [(s0, 0), (s0, 3), (s0, 10)]
    assert src.keypoint_path("/o", 2) == "/o/%s/10.bin" % s0
    files = {s: ["cloud_bin_10.npy", "cloud_bin_0.npy"] for s in itl.MATCH3D_SCENES}
    src = itl.Match3DTestLoader(root, make_opt(input_pc_num=256, node_num=16), files=files)
    assert len(src) == 16 and src.key(0) == (s0, 10)


def test_modelnet_items(tmp_path):
    src = mtl.ModelNetRotatedTestLoader(str(tmp_path), make_opt(input_pc_num=512, node_num=32, surface_normal_len=3))
    assert len(src) == 2 * 2468
    assert src.key(0) == ("original", 0) and src.key(2468) == ("rotated", 0) and src.key(4935) == ("rotated", 2467)
    assert src.keypoint_path("/o", 2469) == "/o/rotated/1.bin"
    src = mtl.ModelNetRotatedTestLoader(str(tmp_path), make_opt(input_pc_num=512, node_num=32, surface_normal_len=3),
                                        n=4)
    assert src.paths[4] == os.path.join(str(tmp_path), "rotated", "0.npy")


def _parity_source(name, root, rng="numpy", **over):
    """The golden's source over the tree tools/make_golden.py wrote."""
    g = golden("%s_test_clouds.npz" % name)
    o = dict(input_pc_num=int(g["N"]), node_num=int(g["M"]))
    o.update(over)
    B = int(g["batch_size"])
    if name == "modelnet":
        tree, _ = modelnet_tree(root, k=int(g["objects"]))
        return g, mtl.ModelNetRotatedTestLoader(tree, make_opt(surface_normal_len=3, **o), rng=rng, batch_size=B,
                                                n=int(g["objects"]))
    if name == "redwood":
        return g, itl.RedwoodTestLoader(redwood_tree(root)[0], make_opt(**o), rng=rng, batch_size=B)
    return g, itl.Match3DTestLoader(match3d_tree(root), make_opt(**o), rng=rng, batch_size=B,
                                    files=golden_listing(g))


@pytest.mark.parametrize("name", ["modelnet", "redwood", "3dmatch"])
def test_parity_draw_order(name, tmp_path):
    g, src = _parity_source(name, str(tmp_path))
    short = 0
    for case in ("plain", "noise"):
        np.random.seed(int(g[case + "/case"][0]))
        if case + "/rows" in g:
            row_draws = list(g[case + "/rows"])
        else:
            row_draws = np.split(g[case + "/rows_flat"], np.cumsum(g[case + "/rows_len"])[:-1])
        for i in range(len(src)):
            n = len(src.load([i])[0])
            rows, cand, start = src.draw_item(np.random, n)
            if n >= src.N:
                np.testing.assert_array_equal(rows, row_draws[i])
            else:                                   # every row t times, then the logged remainder draw
                short += 1
                t = (src.N - len(row_draws[i])) // n
                np.testing.assert_array_equal(rows[:t * n], np.tile(np.arange(n), t))
                np.testing.assert_array_equal(rows[t * n:], row_draws[i])
            np.testing.assert_array_equal(cand, g[case + "/cand"][i])
            assert start == g[case + "/start"][i]
    assert (short > 0) == (name == "redwood")


def test_redwood_remainder_only_draw():
    """A scan of exactly N/2 rows is taken once and its remainder is a permutation of all its rows."""
    rng = np.random.RandomState(3)
    rows, cand, _ = draw_subsample(rng, 16, 32, 2)
    np.testing.assert_array_equal(rows[:16], np.arange(16))
    np.testing.assert_array_equal(np.sort(rows[16:]), np.arange(16))
    assert len(cand) == 16


def test_detector_opt_matches_option_files():
    """modelnet/, scenenn/ (Redwood) and match3d/options_detector.py."""
    want = {"modelnet": dict(input_pc_num=5000, surface_normal_len=3, node_num=512, node_knn_k_1=32,
                             loss_sigma_lower_bound=1e-4, scene="object", keypoint_on_pc_alpha=1.0, rot_3d=True,
                             rot_horizontal=False),
            "redwood": dict(input_pc_num=10240, surface_normal_len=4, node_num=512, node_knn_k_1=32,
                            loss_sigma_lower_bound=1e-4, scene="outdoor", keypoint_on_pc_alpha=100.0, rot_3d=True,
                            rot_horizontal=False),
            "3dmatch": dict(input_pc_num=10240, surface_normal_len=4, node_num=512, node_knn_k_1=32,
                            loss_sigma_lower_bound=1e-4, scene="outdoor", keypoint_on_pc_alpha=10.0, rot_3d=True,
                            rot_horizontal=False)}
    for d, w in want.items():
        o = rep.detector_opt(d)
        assert {k: getattr(o, k) for k in w} == w, d
    assert rep.detector_opt("kitti").loss_sigma_lower_bound == 1e-3
    assert rep.detector_opt("kitti").node_knn_k_1 == 16
    with pytest.raises(ValueError):
        rep.detector_opt("shrec")


# ------------------------------------------------------------------ refusals and evaluators
def test_refusals(tmp_path):
    with pytest.raises(ValueError, match="surface_normal_len must be 3"):
        mtl.ModelNetRotatedTestLoader(str(tmp_path), make_opt(input_pc_num=512, node_num=32))
    with pytest.raises(ValueError, match="surface_normal_len must be 4"):
        itl.RedwoodTestLoader(str(tmp_path), make_opt(surface_normal_len=3))
    root = match3d_tree(str(tmp_path / "m"), rows=300)
    src = itl.Match3DTestLoader(root, make_opt(input_pc_num=512, node_num=32))
    with pytest.raises(ValueError, match="300 rows"):
        src.load([0])
    mroot, _ = modelnet_tree(str(tmp_path / "mn"), k=2, rows=300)
    src = mtl.ModelNetRotatedTestLoader(mroot, make_opt(input_pc_num=512, node_num=32, surface_normal_len=3), n=2)
    with pytest.raises(ValueError, match="300 rows"):
        src.load([0])
    npy, gt = redwood_tree(str(tmp_path / "r"))
    src = itl.RedwoodTestLoader(npy, make_opt(input_pc_num=32, node_num=8))
    assert min(len(a) for a in src.load(list(range(len(src))))) < 32          # shorter scans are taken
    itl.write_gt_log(os.path.join(gt, "original", "office1-evaluation", "gt.log"),
                     [(0, 53, 53, np.eye(4))])
    with pytest.raises(KeyError, match="office1.*53"):
        rep.RedwoodRepeatability(npy, gt, make_opt(input_pc_num=32, node_num=8))


def test_evaluator_pairs_and_frames(tmp_path):
    s0, s1 = itl.MATCH3D_SCENES[:2]
    root = match3d_tree(str(tmp_path / "m"), pairs={s0: [(0, 10), (3, 0)], s1: [(10, 10)]})
    ev = rep.Match3DRepeatability(root, make_opt(input_pc_num=256, node_num=16))
    np.testing.assert_array_equal(ev.pairs, [[0, 2], [1, 0], [5, 5]])
    anc, pos, T = rep.read_gt_log(os.path.join(root, "%s-evaluation" % s0, "gt.log"))
    np.testing.assert_array_equal(ev.frames[:2, 2], T)
    np.testing.assert_array_equal(ev.frames[:, 0], np.broadcast_to(np.eye(3, 4), (3, 3, 4)))
    np.testing.assert_array_equal(ev.frames[:, 1], np.broadcast_to(np.eye(3, 4), (3, 3, 4)))
    np.testing.assert_array_equal(ev.frames[2, 2], np.eye(3, 4))

    mroot, Rs = modelnet_tree(str(tmp_path / "mn"), k=3, rows=600)
    ev = rep.ModelNetRepeatability(mroot, make_opt(input_pc_num=512, node_num=32, surface_normal_len=3))
    assert len(ev.source) == 6
    np.testing.assert_array_equal(ev.pairs, [[0, 3], [1, 4], [2, 5]])
    np.testing.assert_array_equal(ev.frames[:, 2, :, :3], Rs)

    npy, gt = redwood_tree(str(tmp_path / "r"), pairs={"livingroom2": [(0, 46)], "office2": [(49, 1)]})
    ev = rep.RedwoodRepeatability(npy, gt, make_opt(input_pc_num=32, node_num=8))
    np.testing.assert_array_equal(ev.pairs, [[57, 103], [206, 158]])
