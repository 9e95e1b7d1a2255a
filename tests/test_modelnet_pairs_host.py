"""Host side of the ModelNet pair builder (usip_b200.data.modelnet_shrec_loader), no GPU: the parity mode's draw order
against the reference loader's batches in tests/golden/modelnet_pairs.npz, the tree index, argument checks."""
import os
import types

import numpy as np
import pytest

from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import modelnet_shrec_loader as mnl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "modelnet_pairs.npz")


def golden_cases():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files if k.endswith("/case")})
    return g, names


def case_opt(g, name):
    seed, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    opt = types.SimpleNamespace(dataset="modelnet", classes=40, input_pc_num=int(g["N"]), node_num=int(g["M"]),
                                surface_normal_len=3, rot_horizontal=bool(rh), rot_3d=bool(r3),
                                rot_perturbation=bool(rp), translation_perturbation=bool(tp), batch_size=1)
    return opt, str(g[name + "/mode"]), [int(i) for i in g[name + "/items"]], seed


def make_tree(g, root):
    n_train, n_test = (int(c) for c in g["tree/counts"])
    mnl.write_synthetic_modelnet(str(root), [str(s) for s in g["tree/shapes"]], n_train, n_test, int(g["tree/rows"]),
                                 seed=int(g["tree/seed"]))


def split_scans(root, mode, opt):
    """Every object of the split, in dataset order -> (list of (rows, 6) arrays, offsets)."""
    arrs = [kdl.load_scan_npy(path, 3) for path, _, _ in mnl.make_dataset_modelnet40_10k(str(root), mode, opt)]
    return arrs, np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)


def replay(g, name, root):
    """Parity-mode host draws for one golden case -> (objects, rows (B, 2, N), params (B, 48))."""
    opt, mode, items, seed = case_opt(g, name)
    arrs, _ = split_scans(root, mode, opt)
    np.random.seed(seed)
    rows, params = [], []
    for i in items:
        pair = []
        for _ in range(2):
            choice, cand, _ = kdl.draw_subsample(np.random, len(arrs[i]), opt.input_pc_num, mnl.MODELNET_DIVISOR)
            assert len(cand) == opt.input_pc_num // 4
            pair.append(choice)
        p, _ = mnl.draw_modelnet_pair_scalars(np.random, opt, mode == "train", opt.input_pc_num, opt.node_num, True)
        rows.append(pair)
        params.append(p)
    return arrs, np.array(rows), np.stack(params)


def test_parity_draw_order_matches_reference_scalars(tmp_path):
    g, names = golden_cases()
    assert len(names) == 5
    make_tree(g, tmp_path)
    for name in names:
        opt, mode, items, _ = case_opt(g, name)
        arrs, rows, p = replay(g, name, tmp_path)
        np.testing.assert_array_equal(p[:, 31:40].reshape(-1, 3, 3).astype(np.float32), g[name + "/R"], err_msg=name)
        np.testing.assert_array_equal(p[:, 40:43].reshape(-1, 3, 1).astype(np.float32), g[name + "/shift"],
                                      err_msg=name)
        np.testing.assert_array_equal(p[:, 43].astype(np.float32), g[name + "/scale"], err_msg=name)
        assert (np.abs(g[name + "/scale"] - 1) <= 0.2).all() and (g[name + "/scale"] != 1).all()
        if mode == "test":                               # no augmentation: src is the selected rows themselves
            for b, i in enumerate(items):
                np.testing.assert_array_equal(arrs[i][rows[b, 0], 0:3].T, g[name + "/src_pc"][b])
                np.testing.assert_array_equal(arrs[i][rows[b, 0], 3:6].T, g[name + "/src_sn"][b])
        else:
            assert 0.8 <= p[:, 27].min() and p[:, 27].max() <= 1.2 and (np.abs(p[:, 28:31]) <= 0.1).all()


def test_transform_drops_the_rotation_perturbation(tmp_path):
    """With rot_3d and rot_perturbation set, the transform's R is exactly Rz.Ry.Rx of three uniform angles: the
    perturbation's three randn draws would come between them and the scale."""
    g, _ = golden_cases()
    opt, _, _, seed = case_opt(g, "allrot")
    assert opt.rot_perturbation
    rng = np.random.RandomState(seed)
    p, _ = mnl.draw_modelnet_pair_scalars(rng, opt, True, 16, 4, True)
    rng = np.random.RandomState(seed)
    rng.uniform(); rng.rand(3); rng.randn(3); rng.randn(16, 3); rng.randn(16, 3); rng.randn(4, 3); rng.uniform()
    rng.uniform(size=(1, 3))
    angles = [rng.uniform() * 2 * np.pi for _ in range(3)]
    np.testing.assert_array_equal(p[31:40], kdl.angles2rotation_matrix(angles).astype(np.float32).ravel())
    assert p[43] == np.float32(rng.uniform(1 - 0.2, 1 + 0.2))


def test_make_dataset_orders_a_tree_like_the_reference(tmp_path):
    shapes = ["airplane", "night_stand", "cup"]
    mnl.write_synthetic_modelnet(str(tmp_path), shapes, 2, 1, 8, seed=3)
    opt = types.SimpleNamespace(classes=40, node_num=64)
    with open(os.path.join(tmp_path, "modelnet40_shape_names.txt")) as f:
        assert f.read().split() == list(reversed(shapes))
    train = mnl.make_dataset_modelnet40_10k(str(tmp_path), "train", opt)
    expect = [(s, i) for i in (1, 2) for s in shapes]           # the list file interleaves the shapes
    assert len(train) == len(expect)
    for (path, label, som), (s, i) in zip(train, expect):
        assert path == os.path.join(str(tmp_path), s, "%s_%04d.npy" % (s, i)) and os.path.isfile(path)
        assert label == 2 - shapes.index(s)                         # index among the (reversed) shape names
        assert som == os.path.join(str(tmp_path), "8x8_som_nodes", s, "%s_%04d.npy" % (s, i))
    test = mnl.make_dataset_modelnet40_10k(str(tmp_path), "test", opt)
    assert [os.path.basename(p) for p, _, _ in test] == ["%s_0003.npy" % s for s in shapes]
    a = np.load(train[0][0])
    assert a.shape == (8, 6) and a.dtype == np.float32
    np.testing.assert_allclose(np.linalg.norm(a[:, 3:6], axis=1), 1, rtol=1e-6)
    with pytest.raises(ValueError):
        mnl.make_dataset_modelnet40_10k(str(tmp_path), "val", opt)


def _opt(**kw):
    o = types.SimpleNamespace(dataset="modelnet", classes=40, input_pc_num=1000, node_num=64, surface_normal_len=3,
                              rot_horizontal=False, rot_3d=True, rot_perturbation=False, translation_perturbation=False,
                              batch_size=2)
    o.__dict__.update(kw)
    return o


def test_builder_argument_validation():
    import torch
    with pytest.raises(ValueError, match="must be 3"):
        mnl.ModelNetPairBuilder(_opt(surface_normal_len=4), device="cpu")
    with pytest.raises(ValueError, match="8192"):
        mnl.ModelNetPairBuilder(_opt(input_pc_num=4 * 8193), device="cpu")
    with pytest.raises(NotImplementedError, match="66-112"):
        mnl.ModelNetPairBuilder(_opt(dataset="shrec"), device="cpu")
    with pytest.raises(NotImplementedError, match="66-112"):
        mnl.ModelNetPairSource("/nonexistent", "train", _opt(dataset="shrec"), device="cpu")
    b = mnl.ModelNetPairBuilder(_opt(), device="cpu")
    scans = torch.zeros((2500, 6))
    with pytest.raises(ValueError, match="drawn without replacement"):
        b.build(scans, np.array([0, 1500, 2400], np.int64), [0, 1])
    with pytest.raises(IndexError):
        b.build(scans, np.array([0, 2500], np.int64), [1])
    with pytest.raises(ValueError, match="no items"):
        b.build(scans, np.array([0, 2500], np.int64), [])
    assert b.step == 0                                   # a refused build does not advance the step
