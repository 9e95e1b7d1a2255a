"""Host side of the repeatability evaluation (usip_b200.evaluation.repeatability, .kitti_test_loader,
.oxford_test_loader): the float64 restatement of eval_rep.m on hand-computed cases, the ground-truth and calibration
parsers, the KITTI test list's dedupe order, the parity draw order against the reference loaders' logged draws
(tests/golden/kitti_test_clouds.npz, oxford_test_clouds.npz), and the argument checks."""
import os

import numpy as np
import pytest

from tests.rep_ref import pair_counts
from tests.util_gpu import golden, make_opt
from usip_b200.evaluation import kitti_test_loader as ktl
from usip_b200.evaluation import oxford_test_loader as otl
from usip_b200.evaluation import repeatability as rep

I34 = np.eye(3, 4)


def test_three_keypoints_rotation_translation():
    # T_gt: 90 degrees about z, then t = (1, 2, 3); positive keypoints chosen so that T_gt maps them near the anchors
    q = np.array([np.cos(np.pi / 4), 0, 0, np.sin(np.pi / 4)])
    T = rep.gt_transform([1, 2, 3], q)
    np.testing.assert_allclose(T[:, :3], [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-15)
    anc = np.array([[1.0, 2, 3], [11, 2, 3], [1, 12, 3]])
    # R p + t = a  ->  p = R^T (a - t); the second is moved 0.3 away, the third 0.7
    pos = np.array([[0.0, 0, 0], [0, -10, 0], [10, 0, 0]])
    pos[1] += [0.3, 0, 0]
    pos[2] += [0, 0, 0.7]
    inl, nanc = pair_counts(anc, pos, I34, I34, T, [1, 2, 3], 0.5)
    assert nanc == [1, 2, 3]
    # K=1: anchor 0 vs pos 0 -> 0;  K=2: anchors 0, 1 vs pos 0, 1: 0 and 0.3;  K=3: + anchor 2 at 0.7
    assert inl == [1, 2, 2]


def test_distance_exactly_r_is_not_an_inlier():
    anc = np.array([[0.0, 0, 0], [0.0, 0, 0]])
    pos = np.array([[0.5, 0, 0], [0.25, 0, 0]])
    assert pair_counts(anc[:1], pos[:1], I34, I34, I34, [1], 0.5)[0] == [0]
    assert pair_counts(anc, pos, I34, I34, I34, [2], 0.5)[0] == [2]


def test_quaternion_is_normalised():
    q = np.array([0.3, -0.2, 0.9, 0.1])
    np.testing.assert_allclose(rep.quat2rotm(q * 3.7), rep.quat2rotm(q / np.linalg.norm(q)), rtol=0, atol=4e-16)
    R = rep.quat2rotm(q * 3.7)
    np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-14)


def test_frames():
    p = np.array([[1.0, 2.0, 3.0]])
    from tests.rep_ref import apply_map
    np.testing.assert_array_equal(apply_map(rep.CAM_TO_ENU, p), [[1.0, 3.0, -2.0]])      # coord_cam2enu.m
    Tr = np.eye(4); Tr[:3, 3] = [1, 2, 3]
    np.testing.assert_array_equal(rep.cam_to_velodyne(Tr), np.concatenate([np.eye(3), [[-1], [-2], [-3]]], 1))


def _write(path, text):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(text)


def test_parsers(tmp_path):
    _write(str(tmp_path / "c.txt"), "idx1,idx2,t1,t2,t3,qw,qx,qy,qz\n3,7,0.5,-1,2,1,0,0,0\n4,9,1,1,1,0.5,0.5,0.5,0.5\n")
    np.testing.assert_array_equal(rep.read_correct_gt_kitti(str(tmp_path / "c.txt")),
                                  [[3, 7, 0.5, -1, 2, 1, 0, 0, 0], [4, 9, 1, 1, 1, .5, .5, .5, .5]])
    _write(str(tmp_path / "g.txt"), "h\th\th\th\th\th\th\th\th\th\th\n"
                                    "12\t40\ta.bin\tb.bin\t1.5\t2\t-3\t0.9\t0.1\t0.2\t0.3\n")
    np.testing.assert_array_equal(rep.read_gt_oxford(str(tmp_path / "g.txt")), [[12, 40, 1.5, 2, -3, .9, .1, .2, .3]])
    vals = " ".join(str(v) for v in range(12))
    _write(str(tmp_path / "calib.txt"), "".join("P%d: %s\n" % (k, vals) for k in range(4)) + "Tr: %s\n" % vals)
    Tr = rep.read_kitti_calib(str(tmp_path / "calib.txt"))["Tr"]
    np.testing.assert_array_equal(Tr, [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10, 11], [0, 0, 0, 1]])


def test_kitti_test_list_dedupe_order(tmp_path):
    _write(str(tmp_path / "01" / "groundtruths.txt"), "header\n5 6 x\n6 7 x\n8 5 x\n8 6 x\n")
    _write(str(tmp_path / "00" / "groundtruths.txt"), "header\n2 2 x\n")
    d = ktl.make_kitti_test_dataset(str(tmp_path))
    # both checks look at the list before the line adds anything, so a self-pair line adds its scan twice
    assert [(e["seq"], e["anc_idx"], e["pos_idx"]) for e in d] == [
        (0, 2, 2), (0, 2, 2), (1, 5, 6), (1, 6, 5), (1, 7, 6), (1, 8, 5)]


def _kitti_tree(root):
    ktl.write_synthetic_kitti_test(os.path.join(root, "txt"), os.path.join(root, "numpy"), os.path.join(root, "calib"),
                                   [3, 2], 1300, [[(0, 1), (2, 1), (0, 2)], [(1, 0)]], seed=7500)
    return os.path.join(root, "txt"), os.path.join(root, "numpy"), os.path.join(root, "calib")


@pytest.mark.parametrize("name", ["kitti", "oxford"])
def test_parity_draw_order(name, tmp_path):
    g = golden("%s_test_clouds.npz" % name)
    opt = make_opt(input_pc_num=int(g["N"]), node_num=int(g["M"]))
    if name == "kitti":
        src = ktl.KittiTestLoader(*_kitti_tree(str(tmp_path))[:2], opt, rng="numpy")
    else:
        otl.write_synthetic_oxford_test(str(tmp_path), range(5), 1300, [(0, 1)], str(tmp_path / "gt.txt"), seed=7500)
        src = otl.OxfordTestLoader(str(tmp_path), opt, rng="numpy", numbers=range(5))
    for case in ("plain", "noise"):
        np.random.seed(int(g[case + "/case"][0]))
        for i in range(len(src)):
            rows, cand, start = src.draw_item(np.random, len(src.load([i])[0]))
            np.testing.assert_array_equal(rows, g[case + "/rows"][i])
            np.testing.assert_array_equal(cand, g[case + "/cand"][i])
            assert start == g[case + "/start"][i]


def test_refusals(tmp_path):
    txt, num, cal = _kitti_tree(str(tmp_path))
    with pytest.raises(ValueError, match="surface_normal_len"):
        ktl.KittiTestLoader(txt, num, make_opt(surface_normal_len=3))
    src = ktl.KittiTestLoader(txt, num, make_opt(input_pc_num=2048, node_num=64))
    with pytest.raises(ValueError, match="1300 rows"):
        src.load([0])
    for ks, r in (([8, 4], 0.5), ([4, 4], 0.5), ([0, 4], 0.5), ([4, 8], 0.0), ([4, 8], -1.0)):
        with pytest.raises(ValueError):
            rep.check_sweep(ks, r)
    assert rep.check_sweep((4, 8), 0.5) == [4, 8]
    with open(os.path.join(txt, "01", "correct_gt.txt"), "a") as f:
        f.write("1,5,0,0,0,1,0,0,0\n")
    with pytest.raises(KeyError, match=r"\(1, 5\)"):
        rep.KittiRepeatability(txt, num, cal, make_opt(input_pc_num=1024, node_num=64))


def test_evaluator_pairs_and_frames(tmp_path):
    txt, num, cal = _kitti_tree(str(tmp_path))
    ev = rep.KittiRepeatability(txt, num, cal, make_opt(input_pc_num=1024, node_num=64))
    assert [ev.source.key(i) for i in range(len(ev.source))] == [(0, 0), (0, 1), (0, 2), (1, 1), (1, 0)]
    np.testing.assert_array_equal(ev.pairs, [[0, 1], [2, 1], [0, 2], [3, 4]])
    Tr = rep.read_kitti_calib(os.path.join(cal, "00", "calib.txt"))["Tr"]
    np.testing.assert_array_equal(ev.frames[0, 0], np.linalg.inv(Tr)[:3])
    assert ev.source.keypoint_path("/o", 4) == "/o/01/000000.bin"
