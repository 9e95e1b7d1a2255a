"""Host side of the Oxford pair builders (usip_b200.data.oxford_detector_loader, .oxford_descriptor_loader), no GPU:
the dataset parsing, the parity mode's draw order against the reference loaders' batches in
tests/golden/oxford_pairs.npz and oxford_descpairs.npz, the positives and negatives, argument checks."""
import os
import random
import types
import warnings

import numpy as np
import pytest

from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import oxford_descriptor_loader as odesc
from usip_b200.data import oxford_detector_loader as odet

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "oxford_pairs.npz")
GOLDEN_DESC = os.path.join(HERE, "golden", "oxford_descpairs.npz")


def golden_cases(path=GOLDEN):
    g = np.load(path)
    return g, sorted({k.split("/")[0] for k in g.files if k.endswith("/case")})


def make_tree(g, root):
    n_train, n_test = (int(c) for c in g["tree/counts"])
    odet.write_synthetic_oxford(str(root), n_train, int(g["tree/rows"]), n_test=n_test, seed=int(g["tree/seed"]))


def _parse(fn, root):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(str(root))


def case_opt(g, name):
    """Detector golden case -> (opt, mode, item, seed)."""
    index, seed, S, rh, r3, rp, tp, hsc = (int(v) for v in g[name + "/case"])
    opt = types.SimpleNamespace(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S,
                                rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                translation_perturbation=bool(tp), is_height_scaling=bool(hsc), batch_size=1)
    return opt, str(g[name + "/mode"]), index, seed


def desc_case_opt(g, name):
    """Descriptor golden case -> (opt, mode, items, seed)."""
    seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    opt = types.SimpleNamespace(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S,
                                rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                translation_perturbation=bool(tp), is_height_scaling=True,
                                batch_size=len(g[name + "/items"]))
    return opt, str(g[name + "/mode"]), [int(i) for i in g[name + "/items"]], seed


def item_scans(root, mode, make_dataset):
    """The scan of every item of the split, in dataset order -> list of (rows, 8) arrays."""
    ds = _parse(make_dataset, root)
    if mode == "train":
        return [kdl.load_scan_npy(odet.oxford_train_path(str(root), d["file"]), 3) for d in ds]
    return [kdl.load_scan_npy(odet.oxford_test_path(str(root), int(d["anc_idx"])), 3) for d in ds]


def enu_to_cam(a):
    """(n, 3) -> the reference's coordinate_ENU_to_cam_element, transposed to (3, n)."""
    return np.stack([a[:, 0], -a[:, 2], a[:, 1]])


def test_dataset_parsing_matches_the_reference(tmp_path):
    odet.write_synthetic_oxford(str(tmp_path), 12, 40, n_test=5, seed=3, invalid_at=4)
    with pytest.warns(UserWarning, match="line 4 is invalid"):
        det = odet.make_dataset_oxford_train(str(tmp_path))
    desc = _parse(odesc.make_dataset_oxford_train, tmp_path)
    assert len(det) == len(desc) == 12                   # 13 lines, the invalid one skipped
    # the line numbers index the parsed list: item 4 is the file after the invalid line, and lists name items
    assert det[4]["file"] == "000004.bin" and det[4]["pos_list"] == [2, 3, 5, 6]
    assert det[4]["nonneg_list"] == [0, 1, 7, 8]
    assert desc[4]["pos_line_list"] == [2, 3, 5, 6]
    assert desc[4]["nonneg_line_list"] == [0, 1, 7, 8, 2, 3, 5, 6]   # non-negatives, then the positives
    assert os.path.isfile(odet.oxford_train_path(str(tmp_path), det[11]["file"]))
    a = np.load(odet.oxford_train_path(str(tmp_path), det[0]["file"]))
    assert a.shape == (40, 8) and a.dtype == np.float32
    assert a[:, 2].std() < 0.2 * a[:, 1].std()               # ENU: z is up, the flat axis
    gt = odet.make_dataset_oxford_test(str(tmp_path))
    gtd = odesc.make_dataset_oxford_test(str(tmp_path))
    assert [d["anc_idx"] for d in gt] == [d["anc_idx"] for d in gtd] == [100, 103, 106, 109, 112]
    assert gtd[1]["pos_idx_list"] == [100, 106, 109] and set(gt[0]) == {"anc_idx", "pos_idx", "neg_idx", "t", "q"}
    for d in gt:
        assert os.path.isfile(odet.oxford_test_path(str(tmp_path), d["anc_idx"]))


def test_detector_parity_draw_order_matches_reference_scalars(tmp_path):
    g, names = golden_cases()
    assert len(names) == 6
    make_tree(g, tmp_path)
    for name in names:
        opt, mode, index, seed = case_opt(g, name)
        arr = item_scans(tmp_path, mode, odet.make_dataset_oxford_train if mode == "train"
                         else odet.make_dataset_oxford_test)[index]
        b = odet.OxfordPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        sides, (p, jit) = b._draw_item(np.random, [len(arr), len(arr)])
        np.testing.assert_array_equal(p[31:40].reshape(3, 3).astype(np.float32), g[name + "/R"], err_msg=name)
        np.testing.assert_array_equal(p[40:43].reshape(3, 1).astype(np.float32), g[name + "/shift"], err_msg=name)
        np.testing.assert_array_equal(np.float32(p[43]), g[name + "/scale"], err_msg=name)
        assert 0.25 <= p[44] <= 1.2 and len(sides[0][1]) == opt.input_pc_num // 8
        if mode == "test":                               # no augmentation, no height scale: the ENU rows in camera frame
            assert jit is None
            rows = arr[sides[0][0]]
            np.testing.assert_array_equal(enu_to_cam(rows[:, 0:3]), g[name + "/src_pc"])
            sn = rows[:, 3:3 + opt.surface_normal_len].T.copy()
            sn[1], sn[2] = -sn[2], sn[1].copy()
            np.testing.assert_array_equal(sn, g[name + "/src_sn"])
        else:
            assert 0.7 <= p[27] <= 1.3 and jit[0].shape == (2, opt.input_pc_num, 3)


def test_descriptor_parity_draw_order_and_test_mode_clouds(tmp_path):
    g, names = golden_cases(GOLDEN_DESC)
    make_tree(g, tmp_path)
    for name in names:
        opt, mode, items, seed = desc_case_opt(g, name)
        b = odesc.OxfordDescriptorPairBuilder(opt, mode, "cpu", rng="numpy")
        rows = np.random.RandomState(seed)
        p, jit = b._draw(np.random.RandomState(0), False)
        assert (p[:, 27] == (1.0 if mode == "train" else 0.0)).all()  # the scale is 1.0 and nothing is drawn for it
        if mode != "test":
            continue
        arrs = item_scans(tmp_path, mode, odesc.make_dataset_oxford_test)
        for k, i in enumerate(items):
            sides, d = b._draw_item(rows, [len(arrs[i]), len(arrs[i])])
            np.testing.assert_array_equal(enu_to_cam(arrs[i][sides[0][0], 0:3]), g[name + "/anc_pc"][k])
            assert d[1] is None


def _replay_pos_neg(ds, mode, items, seed, rng_cls=None):
    random.seed(seed)
    rng = random if rng_cls is None else rng_cls()
    pos = [odesc.pick_positive(ds, mode, i, rng) for i in items]
    return pos, odesc.mine_negative_sample(ds, mode, items, rng)


class _CountingRandom:
    """Python's global `random` with a count of randint calls."""

    def __init__(self):
        self.calls = 0

    def randint(self, a, b):
        self.calls += 1
        return random.randint(a, b)


def test_positives_and_negatives_replay_the_golden(tmp_path):
    g, names = golden_cases(GOLDEN_DESC)
    make_tree(g, tmp_path)
    assert set(names) == {"train", "noneg", "test"}
    for name in names:
        _, mode, items, seed = desc_case_opt(g, name)
        ds = _parse(odesc.make_dataset_oxford_train if mode == "train" else odesc.make_dataset_oxford_test, tmp_path)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            rng = _CountingRandom()
            pos, neg = _replay_pos_neg(ds, mode, items, seed, lambda: rng)
        np.testing.assert_array_equal(pos, g[name + "/pos_file"], err_msg=name)   # train: lines = file numbers here
        np.testing.assert_array_equal(neg.numpy(), g[name + "/neg_idx"], err_msg=name)
        np.testing.assert_array_equal(g[name + "/index"], items)
        B = len(items)
        if name == "noneg":
            assert any("anchor 2" in str(x.message) for x in w) and neg[2] == 0
        else:
            assert not w
        # one randint per positive, then one per anchor with a candidate in every pass: B passes in test mode
        passes = B if mode == "test" else 1
        assert len(w) % passes == 0
        assert rng.calls == B + passes * (B - len(w) // passes), (name, rng.calls)


def _opt(**kw):
    o = types.SimpleNamespace(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True,
                              rot_3d=False, rot_perturbation=False, translation_perturbation=False, batch_size=2)
    o.__dict__.update(kw)
    return o


@pytest.mark.parametrize("cls", [odet.OxfordPairBuilder, odesc.OxfordDescriptorPairBuilder])
def test_builder_argument_validation(cls):
    import torch
    div = odet.OXFORD_DET_DIVISOR if cls is odet.OxfordPairBuilder else odesc.OXFORD_DESC_DIVISOR
    with pytest.raises(ValueError, match="3..8"):
        cls(_opt(surface_normal_len=2), device="cpu")
    with pytest.raises(ValueError, match="8192"):
        cls(_opt(input_pc_num=div * 8193), device="cpu")
    with pytest.raises(ValueError, match="node_num"):
        cls(_opt(input_pc_num=1024, node_num=1024 // div + 1), device="cpu")
    b = cls(_opt(), device="cpu")
    scans = torch.zeros((2500, 8))
    args = ([0, 1],) if cls is odet.OxfordPairBuilder else ([0], [1])
    with pytest.raises(ValueError, match="drawn without replacement"):
        b.build(scans, np.array([0, 1500, 2400], np.int64), *args)
    assert b.step == 0                                   # a refused build does not advance the step
    assert b.flags & odet.ops.PAIR_ENU_TO_CAM


def test_height_scale_flag_follows_mode_and_option():
    assert odet.OxfordPairBuilder(_opt(), "train", "cpu").flags & odet.ops.PAIR_HEIGHT_SCALE
    assert not odet.OxfordPairBuilder(_opt(), "test", "cpu").flags & odet.ops.PAIR_HEIGHT_SCALE
    assert not odet.OxfordPairBuilder(_opt(is_height_scaling=False), "train", "cpu").flags & odet.ops.PAIR_HEIGHT_SCALE
    assert not odesc.OxfordDescriptorPairBuilder(_opt(), "train", "cpu").flags & odet.ops.PAIR_HEIGHT_SCALE
    b = odet.OxfordPairBuilder(_opt(), "train", "cpu")
    params = np.zeros((3, 48))
    params[:, 44] = [0.3, 0.7, 1.1]
    np.testing.assert_array_equal(b._z_scale(params), np.float32([0.3, 0.3, 0.7, 0.7, 1.1, 1.1]))
    assert odet.OxfordPairBuilder(_opt(), "test", "cpu")._z_scale(params) is None
