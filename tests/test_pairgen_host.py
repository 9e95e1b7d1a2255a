"""Host side of the detector pair builder (usip_b200.data.kitti_detector_loader), no GPU: the parity mode's draw order
against the reference loader's batches in tests/golden/detector_pairs.npz, the scan index mapping, argument checks."""
import os
import types

import numpy as np
import pytest

from usip_b200.data import kitti_detector_loader as kdl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detector_pairs.npz")


def golden_cases():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files if k.endswith("/case")})
    return g, names


def case_opt(g, name):
    index, seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    opt = types.SimpleNamespace(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S,
                                rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                translation_perturbation=bool(tp), radius_threshold=float(g[name + "/radius"]),
                                batch_size=1)
    return opt, str(g[name + "/mode"]), index, seed


def make_tree(g, root):
    kdl.write_synthetic_kitti(str(root), [int(c) for c in g["tree/counts"]], int(g["tree/Ns"]), seed=int(g["tree/seed"]))


def replay(g, name, root):
    """Parity-mode host draws for one golden item -> (rows (2,N), params (48,))."""
    opt, mode, index, seed = case_opt(g, name)
    pc = kdl.load_scan_npy(kdl.kitti_scan_path(str(root), mode, index), opt.surface_normal_len)
    r = opt.radius_threshold
    valid = np.nonzero(kdl.radius_mask(pc, r))[0] if r < 90 else np.arange(len(pc))
    np.random.seed(seed)
    rows = []
    for _ in range(2):
        choice, _, _ = kdl.draw_subsample(np.random, len(valid), opt.input_pc_num)
        rows.append(valid[choice])
    p, _ = kdl.draw_pair_scalars(np.random, opt, mode == "train", opt.input_pc_num, opt.node_num,
                                 opt.surface_normal_len, True)
    return pc, np.stack(rows), p


def test_parity_draw_order_matches_reference_scalars(tmp_path):
    g, names = golden_cases()
    assert len(names) == 6
    make_tree(g, tmp_path)
    for name in names:
        pc, rows, p = replay(g, name, tmp_path)
        np.testing.assert_array_equal(p[31:40].reshape(3, 3).astype(np.float32), g[name + "/R"], err_msg=name)
        np.testing.assert_array_equal(p[40:43].reshape(3, 1).astype(np.float32), g[name + "/shift"], err_msg=name)
        assert float(p[43]) == float(g[name + "/scale"]) == 1.0
        if str(g[name + "/mode"]) == "test":           # no augmentation: src is the selected rows themselves
            np.testing.assert_array_equal(pc[rows[0], 0:3].T, g[name + "/src_pc"])


def test_radius_case_takes_the_tiling_path(tmp_path):
    g, _ = golden_cases()
    make_tree(g, tmp_path)
    opt, mode, index, _ = case_opt(g, "radius")
    pc = kdl.load_scan_npy(kdl.kitti_scan_path(str(tmp_path), mode, index), 4)
    n_valid = int(kdl.radius_mask(pc, opt.radius_threshold).sum())
    assert 0 < n_valid < opt.input_pc_num
    _, rows, _ = replay(g, "radius", tmp_path)
    counts = np.bincount(rows[0], minlength=len(pc))
    inside = counts[kdl.radius_mask(pc, opt.radius_threshold)]
    assert counts.sum() == opt.input_pc_num and inside.max() - inside.min() <= 1
    assert counts[~kdl.radius_mask(pc, opt.radius_threshold)].sum() == 0


def test_scan_index_mapping(tmp_path):
    counts = [2, 0, 3, 1, 1, 1, 1, 1, 2, 1, 2]
    kdl.write_synthetic_kitti(str(tmp_path), counts, 16, seed=3)
    seqs, folders, nums, accs = kdl.make_dataset_kitti(str(tmp_path), "train")
    assert seqs == list(range(9)) and nums == counts[:9] and accs[-1] == sum(counts[:9])
    expect = [(s, i) for s in range(9) for i in range(counts[s])]
    for index, (s, i) in enumerate(expect):
        path = kdl.kitti_scan_path(str(tmp_path), "train", index)
        assert path.endswith(os.path.join("%02d" % s, kdl.KITTI_NP_FOLDER, "%06d.npy" % i))
    assert kdl.kitti_scan_path(str(tmp_path), "test", 2).endswith(os.path.join("10", kdl.KITTI_NP_FOLDER, "000001.npy"))
    with pytest.raises(IndexError):
        kdl.kitti_scan_path(str(tmp_path), "train", sum(counts[:9]))


def _opt(**kw):
    o = types.SimpleNamespace(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                              rot_perturbation=False, translation_perturbation=False, radius_threshold=100.0,
                              batch_size=2)
    o.__dict__.update(kw)
    return o


def test_builder_argument_validation():
    import torch
    b = kdl.DetectorPairBuilder(_opt(), device="cpu")
    scans = torch.zeros((10, 8))
    with pytest.raises(ValueError, match="no scans"):
        b.build(scans, np.array([0], np.int64), [0])
    with pytest.raises(ValueError, match="no points"):
        b.build(scans, np.array([0, 0, 10], np.int64), [0])
    with pytest.raises(IndexError):
        b.build(scans, np.array([0, 10], np.int64), [1])
    with pytest.raises(ValueError, match="8192"):
        kdl.DetectorPairBuilder(_opt(input_pc_num=3 * 8193), device="cpu")
    with pytest.raises(ValueError):
        kdl.DetectorPairBuilder(_opt(), device="cpu", rng="python")
