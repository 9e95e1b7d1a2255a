"""Host side of the indoor pair builders (usip_b200.data.match3d_detector_loader, scenenn_detector_loader), no GPU: the
tree listings, the parity mode's draw order against the reference loaders' batches in tests/golden/indoor_pairs.npz,
the draw laws, argument checks, and the C ABI's refusals of usip_indoor_pair_augment."""
import ctypes
import os
import pickle
import types

import numpy as np
import pytest

from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import match3d_detector_loader as m3l
from usip_b200.data import scenenn_detector_loader as snl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "indoor_pairs.npz")


def golden():
    return np.load(GOLDEN)


def case_names(g, prefix):
    return sorted({k.split("/")[0] for k in g.files if k.endswith("/case") and k.startswith(prefix)})


def m3_layout(g):
    layout = {}
    for entry in g["m3/layout"]:
        split, scene, sub, n = str(entry).split("/")
        layout.setdefault(split, {}).setdefault(scene, {})[sub] = int(n)
    return layout


def make_trees(g, root):
    """The golden's 3DMatch tree under root/3dmatch and SceneNN tree under root/scenenn -> (m3 root, sn root)."""
    m3, sn = os.path.join(str(root), "3dmatch"), os.path.join(str(root), "scenenn")
    rows = g["m3/rows"]
    m3l.write_synthetic_3dmatch_train(m3, m3_layout(g), lambda i: int(rows[i]), seed=int(g["tree/seed"]))
    counts = dict(zip(("train", "val", "test"), (int(c) for c in g["sn/counts"])))
    snl.write_synthetic_scenenn(sn, counts, lambda split, i: 600 if (split, i) == ("train", 1) else 1300,
                                seed=int(g["tree/seed"]))
    return m3, sn


def case_opt(g, name):
    seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    opt = types.SimpleNamespace(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S,
                                rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                translation_perturbation=bool(tp), batch_size=1)
    return opt, seed


def case_items(g, name, m3_root, sn_root):
    """-> (builder mode, divisor, fragment paths of the case's items, augment flags)."""
    modes = [str(m) for m in np.atleast_1d(g[name + "/mode"])]
    rel = [str(p) for p in g[name + "/paths"]]
    if name.startswith("m3"):
        return modes[0], m3l.MATCH3D_DIVISOR, [os.path.join(m3_root, r) for r in rel], [modes[0] == "train"] * len(rel)
    mode = "test" if modes == ["test"] else "train"
    return mode, snl.SCENENN_DIVISOR, [os.path.join(sn_root, r) for r in rel], [m == "train" for m in modes]


def replay(g, name, m3_root, sn_root):
    """Parity-mode host draws of one golden case through the builder's own draw order -> (arrays, sides, params)."""
    opt, seed = case_opt(g, name)
    mode, divisor, paths, aug = case_items(g, name, m3_root, sn_root)
    b = m3l.IndoorPairBuilder(opt, mode, "cpu", rng="numpy", divisor=divisor)
    arrs = [kdl.load_scan_npy(p, opt.surface_normal_len) for p in paths]
    np.random.seed(seed)
    b._pending = iter(aug)
    sides, params = [], []
    for a in arrs:
        s, (p, _) = b._draw_item(np.random, [len(a), len(a)])
        sides.append(s)
        params.append(p)
    return arrs, sides, np.stack(params), aug, mode


def test_golden_has_every_case():
    g = golden()
    assert case_names(g, "m3") == ["m3_default", "m3_horizontal", "m3_s3", "m3_test"]
    assert case_names(g, "sn") == ["sn_mixed", "sn_test", "sn_train", "sn_val"]
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_parity_draw_order_matches_reference_scalars(tmp_path):
    """R, scale and shift of every golden case, bit for bit, from the builder's draws: rows of src and dst, then
    candidates and start of each, then the augmentation (augmented items only), then the transform."""
    g = golden()
    m3_root, sn_root = make_trees(g, tmp_path)
    for name in case_names(g, ""):
        arrs, sides, p, aug, mode = replay(g, name, m3_root, sn_root)
        np.testing.assert_array_equal(p[:, 31:40].reshape(-1, 3, 3).astype(np.float32), g[name + "/R"], err_msg=name)
        np.testing.assert_array_equal(p[:, 40:43].reshape(-1, 3, 1).astype(np.float32), g[name + "/shift"],
                                      err_msg=name)
        np.testing.assert_array_equal(p[:, 43].astype(np.float32), g[name + "/scale"], err_msg=name)
        assert (np.abs(g[name + "/scale"] - 1) <= 0.1).all() and (g[name + "/scale"] != 1).all()
        for b, (a, a_aug) in enumerate(zip(arrs, aug)):
            if mode == "train":
                assert p[b, 45] == float(a_aug)
            if not a_aug:                        # no augmentation: src is the selected rows themselves
                S = int(g[name + "/case"][1])
                np.testing.assert_array_equal(a[sides[b][0][0], 0:3].T, g[name + "/src_pc"][b], err_msg=name)
                np.testing.assert_array_equal(a[sides[b][0][0], 3:3 + S].T, g[name + "/src_sn"][b], err_msg=name)
            else:
                assert 0.8 <= p[b, 27] <= 1.2 and (np.abs(p[b, 28:31]) <= 1).all()


def test_short_fragment_takes_the_tile_path(tmp_path):
    g = golden()
    m3_root, sn_root = make_trees(g, tmp_path)
    for name, b in (("m3_default", 0), ("sn_train", 0)):
        arrs, sides, _, _, _ = replay(g, name, m3_root, sn_root)
        n, N = len(arrs[b]), int(g["N"])
        assert n < N
        rows = sides[b][0][0]
        np.testing.assert_array_equal(rows[:n], np.arange(n))
        assert len(np.unique(rows[n:])) == N - n


def test_indoor_draws_follow_the_reference_laws():
    """draw_pair_scalars with the indoor laws consumes numpy like Match3DDetectorLoader.augment + transform_pc_pytorch."""
    opt = types.SimpleNamespace(rot_3d=False, rot_horizontal=True, rot_perturbation=True)
    N, M, S = 32, 8, 5
    p, jit = kdl.draw_pair_scalars(np.random.RandomState(5), opt, True, N, M, S, True, m3l.INDOOR_SCALE,
                                   m3l.INDOOR_PERTURBATION, m3l.INDOOR_JITTER, m3l.INDOOR_SCALE_THRE)
    r = np.random.RandomState(5)
    y = r.uniform() * 2 * np.pi
    a3 = r.rand(3) * np.pi * 2
    pert = np.clip(0.12 * r.randn(3), -0.36, 0.36)
    jpc = np.clip(0.01 * r.randn(2, N, 3), -0.02, 0.02)
    jsn = np.clip(0.01 * r.randn(2, N, S), -0.02, 0.02)
    jnd = np.clip(0.01 * r.randn(2, M, 3), -0.02, 0.02)
    scale = r.uniform(low=0.8, high=1.2)
    shift = r.uniform(-1, 1, (1, 3))
    np.testing.assert_array_equal(p[0:9], kdl.angles2rotation_matrix([0, y, 0]).ravel())
    np.testing.assert_array_equal(p[9:18], kdl.angles2rotation_matrix(a3).ravel())
    np.testing.assert_array_equal(p[18:27], kdl.angles2rotation_matrix(pert).ravel())
    for got, want in zip(jit, (jpc, jsn, jnd)):
        np.testing.assert_array_equal(got, want)
    assert p[27] == scale and (p[28:31] == shift.ravel()).all()
    x, ya = 0, r.uniform() * 2 * np.pi
    z = 0
    x += np.clip(0.06 * r.randn(), -0.18, 0.18)          # transform_pc_pytorch's own perturbation law
    ya += np.clip(0.06 * r.randn(), -0.18, 0.18)
    z += np.clip(0.06 * r.randn(), -0.18, 0.18)
    np.testing.assert_array_equal(p[31:40], kdl.angles2rotation_matrix([x, ya, z]).astype(np.float32).ravel())
    assert p[43] == np.float32(r.uniform(low=0.9, high=1.1))
    np.testing.assert_array_equal(p[40:43], r.uniform(-0.5, 0.5, (3, 1)).astype(np.float32).ravel())


def test_draw_pair_scalars_defaults_are_kittis():
    opt = types.SimpleNamespace(rot_3d=True, rot_horizontal=False, rot_perturbation=True)
    a = kdl.draw_pair_scalars(np.random.RandomState(9), opt, True, 16, 4, 4, True)
    b = kdl.draw_pair_scalars(np.random.RandomState(9), opt, True, 16, 4, 4, True, (0.9, 1.1), (0.06, 0.18),
                              ((0.04, 0.12), (0.01, 0.05), (0.04, 0.12)), 0.0)
    np.testing.assert_array_equal(a[0], b[0])
    for x, y in zip(a[1], b[1]):
        np.testing.assert_array_equal(x, y)
    assert np.abs(a[1][0]).max() <= 0.12 and np.abs(a[1][0]).max() > 0.02 and a[0][43] == 1.0


def test_3dmatch_listing_sorts_every_level(tmp_path):
    layout = {"train": {"b_scene": {"seq-02": 2, "seq-01": 11}, "a_scene": {"seq-01": 1}},
              "test": {"c_scene": {"seq-01": 1}}}
    m3l.write_synthetic_3dmatch_train(str(tmp_path), layout, 5, seed=1)
    with open(os.path.join(tmp_path, "training_list.txt")) as f:
        assert f.read().split() == ["b_scene", "a_scene"]              # the list file's order is kept
    train = [os.path.relpath(p, tmp_path) for p in m3l.make_3dmatch_dataset(str(tmp_path), "train")]
    names = sorted("%d.npy" % k for k in range(11))
    assert train == (["b_scene/seq-01/" + n for n in names] + ["b_scene/seq-02/0.npy", "b_scene/seq-02/1.npy",
                                                              "a_scene/seq-01/0.npy"])
    assert [os.path.relpath(p, tmp_path) for p in m3l.make_3dmatch_dataset(str(tmp_path), "test")] == \
        ["c_scene/seq-01/0.npy"]
    a = np.load(os.path.join(tmp_path, train[0]))
    assert a.shape == (5, 7) and a.dtype == np.float32
    with pytest.raises(ValueError):
        m3l.make_3dmatch_dataset(str(tmp_path), "val")


def test_scenenn_listing_and_train_plus_val(tmp_path):
    snl.write_synthetic_scenenn(str(tmp_path), {"train": 3, "val": 2, "test": 1}, 9, seed=2)
    with open(os.path.join(tmp_path, "info_val.pkl"), "rb") as f:
        info = pickle.load(f)
    assert set(info) == {"pairs_np", "icp_np", "positive_list", "sample_num"} and info["sample_num"] == 2
    assert snl.scenenn_sample_num(str(tmp_path), "train") == 3
    assert [os.path.relpath(p, tmp_path) for p in snl.make_scenenn_dataset(str(tmp_path), "train")] == \
        ["frames_train/%d.npy" % i for i in range(3)]
    with pytest.raises(ValueError):
        snl.make_scenenn_dataset(str(tmp_path), "train+val")
    src = object.__new__(snl.SceneNNPairSource)                    # the listing alone, without a device
    built = {}

    def fake_init(self, paths, mode, opt, divisor, device, seed, resident, rng, batch_size, drop_last, augment=None):
        built.update(paths=list(paths), mode=mode, divisor=divisor, augment=list(augment))

    orig = m3l._IndoorSource.__init__
    m3l._IndoorSource.__init__ = fake_init
    try:
        snl.SceneNNPairSource.__init__(src, str(tmp_path), "train+val", None)
    finally:
        m3l._IndoorSource.__init__ = orig
    assert [os.path.relpath(p, tmp_path) for p in built["paths"]] == \
        ["frames_train/%d.npy" % i for i in range(3)] + ["frames_val/0.npy", "frames_val/1.npy"]
    assert built["augment"] == [True, True, True, False, False]
    assert built["mode"] == "train" and built["divisor"] == snl.SCENENN_DIVISOR
    with pytest.raises(ValueError, match="mode must be"):
        snl.SceneNNPairSource(str(tmp_path), "trainval", None)


def _opt(**kw):
    o = types.SimpleNamespace(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=False, rot_3d=True,
                              rot_perturbation=False, translation_perturbation=False, batch_size=2)
    o.__dict__.update(kw)
    return o


def test_builder_argument_validation():
    import torch
    with pytest.raises(ValueError, match="8192"):
        m3l.IndoorPairBuilder(_opt(input_pc_num=10 * 8193), device="cpu")
    with pytest.raises(ValueError, match="FPS candidates"):
        m3l.IndoorPairBuilder(_opt(node_num=103), device="cpu")         # 1024 / 10 = 102 candidates
    m3l.IndoorPairBuilder(_opt(node_num=103), device="cpu", divisor=snl.SCENENN_DIVISOR)
    for S in (0, 9):
        with pytest.raises(ValueError, match="sn columns"):
            m3l.IndoorPairBuilder(_opt(surface_normal_len=S), device="cpu")
    with pytest.raises(ValueError, match="mode"):
        m3l.IndoorPairBuilder(_opt(), "val", device="cpu")
    b = m3l.IndoorPairBuilder(_opt(), device="cpu")
    scans = torch.zeros((2500, 7))
    with pytest.raises(ValueError, match="no points"):
        b.build(scans, np.array([0, 1500, 1500, 2500], np.int64), [0, 1])
    with pytest.raises(ValueError, match="one flag per item"):
        b.build(scans, np.array([0, 2500], np.int64), [0, 0], augment=[True])
    with pytest.raises(ValueError, match="columns"):
        m3l.IndoorPairBuilder(_opt(surface_normal_len=5), device="cpu").build(scans, np.array([0, 2500]), [0])
    with pytest.raises(ValueError, match="no items"):
        b.build(scans, np.array([0, 2500], np.int64), [])
    assert b.step == 0 and b._pending is None                      # a refused build changes nothing


def test_existing_sources_refuse_disk_residency(tmp_path):
    from usip_b200.data import modelnet_shrec_loader as mnl
    mnl.write_synthetic_modelnet(str(tmp_path), ("cup",), 1, 1, 8, seed=3)
    opt = types.SimpleNamespace(dataset="modelnet", classes=40, input_pc_num=8, node_num=2, surface_normal_len=3,
                                rot_horizontal=False, rot_3d=True, rot_perturbation=False,
                                translation_perturbation=False, batch_size=1)
    with pytest.raises(ValueError, match="resident='disk'"):
        mnl.ModelNetPairSource(str(tmp_path), "train", opt, device="cpu", resident="disk")


def test_indoor_pair_augment_refusals_before_any_launch():
    """Oxford flags, S outside 1..8, 3 + S > C and more than 32767 pairs: -1 and the reason, no launch (the pointers
    are never dereferenced)."""
    from usip_b200 import _lib, ops
    lib = _lib.load()
    a = [ctypes.c_void_p(0x100000 + 0x10000 * i) for i in range(10)]

    def call(C=7, flags=ops.PAIR_TRAIN, S=4, n_pairs=2):
        return lib.usip_indoor_pair_augment(a[0], C, a[0], a[0], a[0], a[0], a[0], None, None, None, 0, 0, flags, S,
                                            n_pairs, 16, 4, *a[1:10], None)

    for kw, msg in ((dict(flags=ops.PAIR_TRAIN | ops.PAIR_ENU_TO_CAM), "Oxford"),
                    (dict(flags=ops.PAIR_TRAIN | ops.PAIR_HEIGHT_SCALE), "Oxford"),
                    (dict(S=0), "3:3+S"), (dict(S=9, C=12), "3:3+S"), (dict(S=5, C=7), "3:3+S"),
                    (dict(n_pairs=32768), "at most 32767 pairs")):
        assert call(**kw) == -1, kw
        assert msg.encode() in lib.usip_last_error(), (kw, lib.usip_last_error())
