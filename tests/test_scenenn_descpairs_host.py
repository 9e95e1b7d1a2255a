"""Host side of the SceneNN descriptor pairs (usip_b200/data/scenenn_descriptor_loader.py): the listing and the
train+val kinds, the parity-mode draw order against the reference (tests/golden/scenenn_descpairs.npz), the synthetic
tree's rigid positives, argument checks, and the C ABI's refusals of the three new calls."""
import ctypes
import os
import pickle
import types

import numpy as np
import pytest

from usip_b200 import ops
from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import scenenn_descriptor_loader as sdl
from usip_b200.data import scenenn_detector_loader as snl

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scenenn_descpairs.npz")
CASES = ("train", "rot3d", "s3", "short", "val", "test", "seq", "wdiv")
KIND = {"train": ops.SCENENN_KIND_FULL, "val": ops.SCENENN_KIND_ROT, "test": ops.SCENENN_KIND_NONE}


def _opt(**kw):
    o = types.SimpleNamespace(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                              rot_perturbation=True, translation_perturbation=False, batch_size=2)
    o.__dict__.update(kw)
    return o


def _case_opt(g, name):
    seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    return seed, _opt(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S, rot_horizontal=bool(rh),
                      rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp))


def test_golden_has_every_case():
    g = np.load(GOLDEN)
    for name in CASES:
        for k in ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node", "R", "scale", "shift", "case",
                  "split", "item", "frames", "icp"):
            assert name + "/" + k in g, (name, k)
    assert not np.array_equal(g["wdiv/icp"][0, 3], [0, 0, 0, 1])       # the case that pins the w division
    assert list(g["test/frames"][0]) == [6, 7]                        # item 1 of the [::3] listing is pair 3


def test_parity_draws_reproduce_the_reference_transform():
    """Replaying __getitem__'s draws item by item (rows, candidates and starts, the kind's augmentation draws, the
    transform) gives the golden's R, scale and shift bit for bit: every draw is consumed in the reference's order."""
    g = np.load(GOLDEN)
    rows_of = lambda split, i: 600 if (split, i) in (("train", 4), ("train", 5)) else 1300
    for name in CASES:
        seed, opt = _case_opt(g, name)
        b = sdl.SceneNNDescriptorPairBuilder(opt, device="cpu", rng="numpy")
        splits = [str(s) for s in g[name + "/split"]]
        b._pending = iter([KIND[s] for s in splits])
        np.random.seed(seed)
        for j, split in enumerate(splits):
            a, p = (int(v) for v in g[name + "/frames"][j])
            sides, (params, jit) = b._draw_item(np.random, [rows_of(split, a), rows_of(split, p)])
            assert jit is None
            assert params[ops.PAIR_AUGMENT_SLOT] == KIND[split]
            np.testing.assert_array_equal(params[31:40].astype(np.float32).reshape(3, 3), g[name + "/R"][j], name)
            assert np.float32(params[43]) == g[name + "/scale"][j], name
            np.testing.assert_array_equal(params[40:43].astype(np.float32), g[name + "/shift"][j].ravel(), name)
            assert len(sides[0][1]) == opt.input_pc_num // 2 and 0 <= sides[0][2] < opt.input_pc_num // 2


def test_kinds_draw_what_their_split_draws():
    """Full: augment()'s rotations, scale and shift; rotations only: the three rotation matrices, no scale or shift;
    none: the transform alone.  No kind returns jitter to upload."""
    b = sdl.SceneNNDescriptorPairBuilder(_opt(input_pc_num=64, node_num=8), device="cpu", rng="numpy")
    for kind in (0, 1, 2):
        for per_point in (True, False):
            b._pending = iter([kind])
            p, jit = b._draw(np.random.RandomState(5), per_point)
            assert jit is None and p[45] == kind
            assert p[31:44].any()
            if kind == 0:
                assert not p[0:31].any()
            if kind == 1:
                assert p[0:27].any() and p[27] == 0 and not p[28:31].any()
            if kind == 2:
                assert 0.9 <= p[27] < 1.1 and p[28:31].any()


def test_device_mode_skips_exactly_the_jitter_draws():
    opt = _opt(input_pc_num=64, node_num=8)
    b = sdl.SceneNNDescriptorPairBuilder(opt, device="cpu")
    a, d = np.random.RandomState(9), np.random.RandomState(9)
    b._pending = iter([2]); pa, _ = b._draw(a, True)
    # replay by hand: the rotation draws, then the jitter the reference discards, then scale, shift and transform
    d.uniform(); d.rand(3); d.randn(3)
    d.randn(2, 64, 3); d.randn(2, 64, 4); d.randn(2, 8, 3)
    assert d.uniform(0.9, 1.1) == pa[27]
    b2 = sdl.SceneNNDescriptorPairBuilder(opt, device="cpu")
    e = np.random.RandomState(9)
    b2._pending = iter([2]); pd, _ = b2._draw(e, False)
    np.testing.assert_array_equal(pd[0:27], pa[0:27])
    f = np.random.RandomState(9)
    f.uniform(); f.rand(3); f.randn(3)
    assert f.uniform(0.9, 1.1) == pd[27]


def test_synthetic_positives_are_rigid_images(tmp_path):
    root = str(tmp_path)
    snl.write_synthetic_scenenn(root, {"train": 4, "val": 2}, 50, seed=3, pairs={"train": [(0, 1), (2, 3)]})
    pairs, icp = sdl.scenenn_pairs(root, "train")
    assert pairs.tolist() == [[0, 1], [2, 3]] and icp.shape == (2, 4, 4)
    for (a, p), T in zip(pairs, icp):
        A = np.load(os.path.join(root, "frames_train", "%d.npy" % a)).astype(np.float64)
        P = np.load(os.path.join(root, "frames_train", "%d.npy" % p)).astype(np.float64)
        np.testing.assert_allclose(A[:, 0:3] @ T[0:3, 0:3].T + T[0:3, 3], P[:, 0:3], atol=1e-6)
        np.testing.assert_allclose(A[:, 3:6] @ T[0:3, 0:3].T, P[:, 3:6], atol=1e-6)
        np.testing.assert_array_equal(A[:, 6:], P[:, 6:])
        np.testing.assert_allclose(T[0:3, 0:3] @ T[0:3, 0:3].T, np.eye(3), atol=1e-12)
        assert T[3].tolist() == [0, 0, 0, 1]
    v, _ = sdl.scenenn_pairs(root, "val")
    assert v.shape == (0, 2)
    with pytest.raises(ValueError, match="positive"):
        snl.write_synthetic_scenenn(root, {"train": 4}, 50, pairs={"train": [(0, 1), (1, 2)]})


def test_default_tree_is_unchanged(tmp_path):
    snl.write_synthetic_scenenn(str(tmp_path), {"train": 2}, 9, seed=2)
    with open(os.path.join(tmp_path, "info_train.pkl"), "rb") as f:
        info = pickle.load(f)
    assert info["pairs_np"].shape == (0, 2) and info["icp_np"].shape == (0, 4, 4) and info["sample_num"] == 2


def test_listing_test_split_and_train_plus_val(tmp_path):
    root = str(tmp_path)
    snl.write_synthetic_scenenn(root, {"train": 6, "val": 4, "test": 14}, 20, seed=4,
                                pairs={"train": [(4, 5), (0, 1)], "val": [(2, 3)],
                                       "test": [(2 * k, 2 * k + 1) for k in range(7)]})
    pairs, icp = sdl.scenenn_pairs(root, "test")
    assert pairs.tolist() == [[0, 1], [6, 7], [12, 13]] and icp.shape == (3, 4, 4)
    calls = []

    def fake_init(self, paths, mode, opt, builder, device, seed, resident, rng, batch_size, drop_last, n_items=None):
        calls.append(dict(paths=list(paths), mode=mode, builder=builder, n_items=n_items))

    orig = kdl._ScanSource.__init__
    kdl._ScanSource.__init__ = fake_init
    try:
        src = object.__new__(sdl.SceneNNDescriptorPairSource)     # the listing alone, without a device
        sdl.SceneNNDescriptorPairSource.__init__(src, root, "train+val", _opt(), detector=None)
        tst = object.__new__(sdl.SceneNNDescriptorPairSource)
        sdl.SceneNNDescriptorPairSource.__init__(tst, root, "test", _opt(), detector=None)
    finally:
        kdl._ScanSource.__init__ = orig
    built, built_test = calls
    rel = [os.path.relpath(q, root) for q in built["paths"]]
    assert rel == ["frames_train/%d.npy" % i for i in (0, 1, 4, 5)] + ["frames_val/2.npy", "frames_val/3.npy"]
    assert [rel[i] for i in src.anc] == ["frames_train/4.npy", "frames_train/0.npy", "frames_val/2.npy"]
    assert [rel[i] for i in src.pos] == ["frames_train/5.npy", "frames_train/1.npy", "frames_val/3.npy"]
    assert src.kinds.tolist() == [2, 2, 1] and src.icp.shape == (3, 4, 4)
    assert built["builder"] is sdl.SceneNNDescriptorPairBuilder
    assert built["mode"] == "train" and built["n_items"] == 3
    assert [os.path.relpath(q, root) for q in built_test["paths"]] == ["frames_test/%d.npy" % i for i in (0, 1, 6, 7, 12,
                                                                                                          13)]
    assert tst.kinds.tolist() == [0, 0, 0] and built_test["mode"] == "test" and built_test["n_items"] == 3
    with pytest.raises(ValueError, match="mode must be"):
        sdl.SceneNNDescriptorPairSource(root, "trainval", _opt(), None)


def test_builder_argument_validation():
    import torch
    for S in (2, 9):
        with pytest.raises(ValueError, match="sn columns"):
            sdl.SceneNNDescriptorPairBuilder(_opt(surface_normal_len=S), device="cpu")
    with pytest.raises(ValueError, match="FPS candidates"):
        sdl.SceneNNDescriptorPairBuilder(_opt(node_num=513), device="cpu")       # 1024 / 2 = 512 candidates
    with pytest.raises(ValueError, match="8192"):
        sdl.SceneNNDescriptorPairBuilder(_opt(input_pc_num=2 * 8193), device="cpu")
    b = sdl.SceneNNDescriptorPairBuilder(_opt(), device="cpu")
    assert not b.flags & ops.PAIR_TRAIN and b.divisor == 2
    scans, off = torch.zeros((2500, 7)), np.array([0, 1500, 2500], np.int64)
    eye = np.eye(4)[None]
    with pytest.raises(ValueError, match="icp"):
        b.build(scans, off, [0], [1], np.eye(4), [2])
    with pytest.raises(ValueError, match="one entry per pair"):
        b.build(scans, off, [0], [1], eye, [2, 2])
    with pytest.raises(ValueError, match="kinds must be"):
        b.build(scans, off, [0], [1], eye, [3])
    with pytest.raises(ValueError, match="anchors but"):
        b.build(scans, off, [0, 1], [1], np.concatenate([eye, eye]), [2, 2])
    assert b.step == 0 and b._pending is None and b._icp is None      # a refused build changes nothing


def test_c_abi_refusals_before_any_launch():
    """A null icp, S outside 3..8, 3 + S > C, the Oxford flags, M > n_cand and more than 32767 pairs: -1 and the
    reason, no launch (the pointers are never dereferenced)."""
    from usip_b200 import _lib
    lib = _lib.load()
    a = [ctypes.c_void_p(0x100000 + 0x10000 * i) for i in range(12)]

    def aug(C=7, flags=ops.PAIR_ROT_HORIZONTAL, S=4, n_pairs=2, icp=a[1], M=4, n_cand=8):
        return lib.usip_scenenn_desc_pair_augment(a[0], C, a[0], a[0], a[0], icp, a[2], a[3], a[4], flags, S, n_pairs,
                                                  16, M, n_cand, *a[3:12], None)

    for kw, msg in ((dict(icp=None), "null icp"), (dict(S=2), "3:3+S"), (dict(S=9, C=12), "3:3+S"),
                    (dict(S=5, C=7), "3:3+S"), (dict(flags=ops.PAIR_ENU_TO_CAM), "Oxford"),
                    (dict(flags=ops.PAIR_HEIGHT_SCALE), "Oxford"), (dict(M=9), "bad sizes"),
                    (dict(n_pairs=32768), "at most 32767 pairs")):
        assert aug(**kw) == -1, kw
        assert msg.encode() in lib.usip_last_error(), (kw, lib.usip_last_error())

    def gather(icp=a[1], n_pairs=2, n_cand=8):
        return lib.usip_cloud_gather_candidates_icp_f64(a[0], 7, a[0], a[0], a[0], a[0], icp, a[2], n_pairs, 16, n_cand,
                                                        None)

    for kw, msg in ((dict(icp=None), "null pointer"), (dict(n_pairs=32768), "at most 32767 pairs"),
                    (dict(n_cand=17), "bad sizes")):
        assert gather(**kw) == -1, kw
        assert msg.encode() in lib.usip_last_error(), (kw, lib.usip_last_error())
    assert lib.usip_fps_f64(a[0], a[0], a[0], None, 1, 8193, 4, None) == -1
    assert b"8192" in lib.usip_last_error()
    assert lib.usip_fps_f64(None, a[0], a[0], None, 1, 16, 4, None) == -1
