"""Oxford pair builders on the GPU (csrc/pairgen.cu USIP_PAIR_ENU_TO_CAM / USIP_PAIR_HEIGHT_SCALE,
usip_cloud_gather_candidates_zscaled, usip_scale_channel_f32; usip_b200.data.oxford_detector_loader and
.oxford_descriptor_loader).

Parity mode (the builders replay numpy's draws) against the reference loaders' own batches in
tests/golden/oxford_pairs.npz and oxford_descpairs.npz; device mode for the frame change, the height scaling,
determinism and the jitter law; end to end through both sources into ModelDetector / ModelDescriptor.optimize()."""
import math
import random

import numpy as np
import pytest
import torch

from tests.test_gpu_pairgen import _clipped_std, _ulps
from tests.test_oxford_pairs_host import (GOLDEN_DESC, _parse, case_opt, desc_case_opt, enu_to_cam, golden_cases,
                                          item_scans, make_tree)
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import ops
from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import oxford_descriptor_loader as odesc
from usip_b200.data import oxford_detector_loader as odet

pytestmark = pytest.mark.gpu
KEYS = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
DESC_KEYS = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node")


def _stack(arrs):
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off


def _compare(got, ref, name, exact, tally):
    got = got.reshape(ref.shape)
    if exact:
        np.testing.assert_array_equal(got, ref, err_msg=name)
    u = _ulps(got, ref)
    assert u.max() <= 2, (name, int(u.max()), float(np.abs(got - ref).max()))
    tally[0] += int((u == 0).sum()); tally[1] += u.size


def test_detector_parity_mode_reproduces_the_reference_loader(tmp_path):
    g, names = golden_cases()
    make_tree(g, tmp_path)
    tally = [0, 0]
    for name in names:
        opt, mode, index, seed = case_opt(g, name)
        scans, off = _stack(item_scans(tmp_path, mode, odet.make_dataset_oxford_train if mode == "train"
                                       else odet.make_dataset_oxford_test))
        b = odet.OxfordPairBuilder(opt, mode, dev(), rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, off, [index])
        for k, t in zip(KEYS, out):
            # the transform's scalars, and src before any augmentation, are copies of the reference's numbers
            exact = k in ("R", "scale", "shift") or (mode == "test" and k.startswith("src"))
            _compare(t[0].cpu().numpy(), g[name + "/" + k], name + "/" + k, exact, tally)
    print("oxford detector parity: %.5f of %d coordinates bit-identical" % (tally[0] / tally[1], tally[1]))
    assert tally[0] >= 0.99 * tally[1]


def _desc_scans(root, mode):
    """The scans of a split and the scan of an item / of a positive, as OxfordDescriptorPairSource indexes them."""
    if mode == "train":
        arrs = item_scans(root, mode, odesc.make_dataset_oxford_train)
        return arrs, (lambda i: i), (lambda p: p)
    ds = _parse(odesc.make_dataset_oxford_test, root)
    numbers = sorted({d["anc_idx"] for d in ds} | {p for d in ds for p in d["pos_idx_list"]})
    arrs = [kdl.load_scan_npy(odet.oxford_test_path(str(root), n), 3) for n in numbers]
    return arrs, (lambda i: numbers.index(ds[i]["anc_idx"])), numbers.index


def test_descriptor_parity_mode_reproduces_the_reference_loader(tmp_path):
    g, names = golden_cases(GOLDEN_DESC)
    make_tree(g, tmp_path)
    tally = [0, 0]
    for name in names:
        opt, mode, items, seed = desc_case_opt(g, name)
        ds = _parse(odesc.make_dataset_oxford_train if mode == "train" else odesc.make_dataset_oxford_test, tmp_path)
        arrs, scan_of_item, scan_of_pos = _desc_scans(tmp_path, mode)
        scans, off = _stack(arrs)
        b = odesc.OxfordDescriptorPairBuilder(opt, mode, dev(), rng="numpy")
        np.random.seed(seed)
        random.seed(seed)
        pos = [odesc.pick_positive(ds, mode, i, random) for i in items]
        with pytest.warns(UserWarning) if name == "noneg" else _nothing():
            neg = odesc.mine_negative_sample(ds, mode, items, random)
        out = b.build(scans, off, [scan_of_item(i) for i in items], [scan_of_pos(p) for p in pos])
        np.testing.assert_array_equal(pos, g[name + "/pos_file"], err_msg=name)
        np.testing.assert_array_equal(neg.numpy(), g[name + "/neg_idx"], err_msg=name)
        for k, t in zip(DESC_KEYS, out):
            _compare(t.cpu().numpy(), g[name + "/" + k], name + "/" + k, mode == "test", tally)
    print("oxford descriptor parity: %.5f of %d coordinates bit-identical" % (tally[0] / tally[1], tally[1]))
    assert tally[0] >= 0.99 * tally[1]


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _oopt(**kw):
    base = dict(input_pc_num=2048, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                rot_perturbation=False, translation_perturbation=False, is_height_scaling=True)
    base.update(kw)
    return make_opt(**base)


def _scans(ns, seed=0):
    arrs = [odet.synthetic_enu_scan(seed + i, n) for i, n in enumerate(ns)]
    scans, off = _stack(arrs)
    return scans, off, arrs


def test_test_mode_is_the_camera_frame_and_candidates_are_height_scaled():
    """Test mode: every output cloud is the gathered rows in the camera frame, exactly (dst after the transform of R,
    scale, shift); the nodes are FPS nodes of the unscaled candidates.  Train mode: the candidates' z is fl32(z * fl32(hs))
    with hs the pair's, shared by both clouds."""
    scans, off, arrs = _scans([3000, 2500, 4000], seed=70)
    opt = _oopt()
    b = odet.OxfordPairBuilder(opt, "test", dev(), seed=3)
    items = [2, 0, 1]
    out = b.build(scans, off, items, step=4)
    rows = b.last["rows"].cpu().numpy()
    for p, i in enumerate(items):
        a = arrs[i][rows[2 * p]]
        np.testing.assert_array_equal(out[0][p].cpu().numpy(), enu_to_cam(a[:, 0:3]))
        sn = a[:, 3:7].T.copy()
        sn[1], sn[2] = -sn[2], sn[1].copy()
        np.testing.assert_array_equal(out[1][p].cpu().numpy(), sn)
    _, nodes = ops.fps(b.last["candidates"], b.last["start"], opt.node_num)
    nd = nodes[0::2].cpu().numpy()
    np.testing.assert_array_equal(out[2].cpu().numpy(), np.stack([nd[:, 0], -nd[:, 2], nd[:, 1]], 1))

    bt = odet.OxfordPairBuilder(opt, "train", dev(), seed=3)
    bt.build(scans, off, items, step=4)
    hs = bt.last["params"][:, 44].cpu().numpy()
    assert ((0.25 <= hs) & (hs <= 1.2)).all() and len(np.unique(hs)) == 3
    rows, cand, pts = (bt.last[k].cpu().numpy() for k in ("rows", "cand", "candidates"))
    for c in range(6):
        raw = arrs[items[c // 2]][rows[c][cand[c]], 0:3]
        np.testing.assert_array_equal(pts[c][:, 0:2], raw[:, 0:2])
        np.testing.assert_array_equal(pts[c][:, 2], raw[:, 2] * np.float32(hs[c // 2]))   # float32 * float32
    off_b = odet.OxfordPairBuilder(_oopt(is_height_scaling=False), "train", dev(), seed=3)
    off_b.build(scans, off, items, step=4)
    assert off_b._z_scale(off_b.last["params"].cpu().numpy()) is None


def test_train_rows_are_height_scaled_before_the_frame_change():
    """Identity augmentation (uploaded zero jitter, identity rotations and transform, scale 1, no shift): src pc is
    (x, -fl32(z * fl32(hs)), y) exactly and sn is only moved; without USIP_PAIR_HEIGHT_SCALE pc is (x, -z, y)."""
    N, M, S = 1024, 32, 5
    a = odet.synthetic_enu_scan(5, N)
    scans = torch.from_numpy(a).to(dev())
    off = torch.tensor([0, N], dtype=torch.int64, device=dev())
    soc = torch.zeros(2, dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2, 1).contiguous()
    nodes = torch.from_numpy(np.ascontiguousarray(a[:M, :3].T)).to(dev()).repeat(2, 1, 1).contiguous()
    params = np.zeros((1, ops.PAIR_PARAM_STRIDE))
    params[:, 27], params[:, 43], params[:, 44] = 1.0, 1.0, 0.4321
    params[:, 31:40] = np.eye(3).ravel()
    zero = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev())
    jit = (zero(2, N, 3), zero(2, N, S), zero(2, M, 3))
    p = torch.from_numpy(params).to(dev())
    base = ops.PAIR_TRAIN | ops.PAIR_ENU_TO_CAM
    for flags, z in ((base | ops.PAIR_HEIGHT_SCALE, a[:, 2] * np.float32(0.4321)), (base, a[:, 2])):
        out = ops.pair_augment(scans, off, soc, rows, nodes, p, S, flags, 0, 0, *jit)
        for side in (0, 3):
            np.testing.assert_array_equal(out[side][0].cpu().numpy(), np.stack([a[:, 0], -z, a[:, 1]]))
            np.testing.assert_array_equal(out[side + 1][0].cpu().numpy(),
                                          np.stack([a[:, 3], -a[:, 5], a[:, 4], a[:, 6], a[:, 7]]))
            np.testing.assert_array_equal(out[side + 2][0].cpu().numpy(),
                                          np.stack([a[:M, 0], -a[:M, 2], a[:M, 1]]))


def test_descriptor_height_scaling_matches_torch():
    torch.manual_seed(0)
    B, N, M, hs = 3, 5000, 700, float(np.random.RandomState(1).uniform(0.25, 1.2))
    pc, kp, sn = (torch.randn(B, 3, N, device=dev()), torch.randn(B, 3, M, device=dev()),
                  torch.randn(B, 4, N, device=dev()))
    ref_pc, ref_kp, ref_sn = pc.clone(), kp.clone(), sn.clone()
    ref_pc[:, 1, :] *= hs
    ref_kp[:, 1, :] *= hs
    odesc.scale_height_(hs, pc, kp)
    assert torch.equal(pc, ref_pc) and torch.equal(kp, ref_kp) and torch.equal(sn, ref_sn)
    assert not torch.equal(pc[:, 1], ref_sn[:, 1])
    with pytest.raises(ValueError):
        ops.scale_channel_(pc, 3, 2.0)


def test_device_mode_is_deterministic_and_subsets_are_unique_rows():
    scans, off, arrs = _scans([3000, 2500, 4000, 2100], seed=10)
    opt = _oopt(rot_3d=True, rot_horizontal=False, rot_perturbation=True, translation_perturbation=True)
    b = odet.OxfordPairBuilder(opt, "train", dev(), seed=5)
    a1 = [t.clone() for t in b.build(scans, off, [0, 2, 3], step=7)]
    a2 = b.build(scans, off, [0, 2, 3], step=7)
    a3 = b.build(scans, off, [0, 2, 3], step=8)
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[6], a3[6])
    assert float(a1[7].min()) == 1.0 == float(a1[7].max()) and float(a1[8].abs().max()) <= 0.5
    d = odesc.OxfordDescriptorPairBuilder(opt, "train", dev(), seed=5)
    d1 = [t.clone() for t in d.build(scans, off, [0, 2], [1, 3], step=2)]
    d2 = d.build(scans, off, [0, 2], [1, 3], step=2)
    assert all(torch.equal(x, y) for x, y in zip(d1, d2))
    rows, cand = d.last["rows"].cpu().numpy(), d.last["cand"].cpu().numpy()
    for c, scan in enumerate([0, 1, 2, 3]):
        r = rows[c]
        assert len(np.unique(r)) == len(r) and r.max() < len(arrs[scan])
        assert len(np.unique(cand[c])) == cand.shape[1] == opt.input_pc_num // 4


def test_device_jitter_is_clipped_normal_in_the_camera_frame():
    """Identity rotations, scale 1, no shift: the descriptor's output minus the camera-frame input is the jitter,
    N(0, 0.04^2) clipped at 0.12 for pc and nodes, N(0, 0.01^2) clipped at 0.05 for sn."""
    N, M, S = 16384, 512, 4
    a = odet.synthetic_enu_scan(9, N)
    scans = torch.from_numpy(a).to(dev())
    off = torch.tensor([0, N], dtype=torch.int64, device=dev())
    soc = torch.zeros(2, dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2, 1).contiguous()
    nodes = torch.from_numpy(np.ascontiguousarray(a[:M, :3].T)).to(dev()).repeat(2, 1, 1).contiguous()
    params = np.zeros((2, ops.DESC_PARAM_STRIDE))
    params[:, 27] = 1.0
    out = ops.desc_pair_augment(scans, off, soc, rows, nodes, torch.from_numpy(params).to(dev()), S,
                                ops.PAIR_TRAIN | ops.PAIR_ENU_TO_CAM, seed=4, step=1)
    o = [t[0].cpu().numpy().astype(np.float64) for t in out]
    sn = a[:, 3:7].T.astype(np.float64)
    sn[1], sn[2] = -sn[2], sn[1].copy()
    cam = lambda x: np.stack([x[:, 0], -x[:, 2], x[:, 1]]).astype(np.float64)
    for j, sigma, clip in ((o[0] - cam(a[:, 0:3]), 0.04, 0.12), (o[1] - sn, 0.01, 0.05),
                           (o[2] - cam(a[:M, 0:3]), 0.04, 0.12)):
        assert np.abs(j).max() <= clip * (1 + 1e-4)
        sd = _clipped_std(sigma, clip)
        n = j.size
        assert abs(j.mean()) < 5 * sd / math.sqrt(n) + 1e-6
        assert abs(j.std() / sd - 1) < 6 / math.sqrt(2 * n) + 2e-3, (j.std(), sd)


# ------------------------------------------------------------------------------------------------ end to end
def test_pair_source_feeds_detector_optimize(tmp_path):
    """The Oxford detector shape: B=2, N=16384, M=512, S=4, rot_horizontal, height scaling."""
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    odet.write_synthetic_oxford(str(tmp_path), 5, 20480, seed=90)
    opt = _oopt(input_pc_num=16384, node_num=512, batch_size=2)
    src = odet.OxfordPairSource(str(tmp_path), "train", opt, dev(), seed=1)
    md = ModelDetector(opt)
    load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    losses = []
    for _ in src.feed(md):
        md.optimize(epoch=0)
        losses.append(float(md.loss))
    assert len(src) == 2 and len(losses) == 2 and all(math.isfinite(v) for v in losses)


def _desc_source(tmp_path, mode, N, M, B, n_train, rows, **kw):
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    from usip_b200.models.keypoint_detector import ModelDetector
    odet.write_synthetic_oxford(str(tmp_path), n_train, rows, n_test=6, seed=91)
    opt = _oopt(input_pc_num=N, node_num=M, batch_size=B, **kw)
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    det.freeze_model()
    src = odesc.OxfordDescriptorPairSource(str(tmp_path), mode, opt, det, dev(), seed=1)
    torch.manual_seed(3)
    return src, det, ModelDescriptor(opt)


def test_descriptor_source_scales_after_the_detector(tmp_path):
    """The keypoints are the frozen detector's on the unscaled clouds, then camera y of clouds and keypoints is scaled
    by the batch's height scale; sn and sigmas are not.  Test mode scales nothing."""
    src, det, md = _desc_source(tmp_path, "train", 1024, 64, 3, 9, 1300, ball_nsamples=32)
    for out in src.feed(md):
        info = src.last
        c, hs = info["clouds"], info["height_scale"]
        assert 0.25 <= hs <= 1.2
        # the same batch again, unscaled: device mode is a pure function of (seed, step)
        u = src.builder.build(src.scans, src.offsets, src.item_scan[info["items"]],
                              [src.scan_of_positive(p) for p in info["positives"]], step=info["step"])
        (kp_a, kp_p), (sg_a, sg_p) = det.run_model_siamese((u[0], u[3]), (u[1], u[4]), (u[2], u[5]))
        assert torch.equal(out[3], sg_a) and torch.equal(out[7], sg_p)
        assert out[0] is c[0] and out[4] is c[3] and torch.equal(out[1], u[1]) and torch.equal(out[5], u[4])
        for got, ref in ((out[2], kp_a), (out[6], kp_p), (out[0], u[0]), (out[4], u[3])):
            ref = ref.clone()
            ref[:, 1, :] *= hs
            assert torch.equal(got, ref)
        md.optimize(epoch=0)
        assert math.isfinite(float(md.loss.detach()))
    ts, tdet, tmd = _desc_source(tmp_path / "t", "test", 1024, 64, 3, 3, 1300, ball_nsamples=32)
    for out in ts.feed(tmd):
        c = ts.last["clouds"]
        assert ts.last["height_scale"] is None
        (kp_a, _), _ = tdet.run_model_siamese((c[0], c[3]), (c[1], c[4]), (c[2], c[5]))
        assert torch.equal(out[2], kp_a)
        pos = ts.last["positives"]
        assert all(p in ts.dataset[i]["pos_idx_list"] for i, p in zip(ts.last["items"], pos))


def test_descriptor_source_full_oxford_shape_step(tmp_path):
    """BASELINE configs[3]: 8 pairs, N=16384, 1024 keypoints, ball_query r=1.0, Kb=64."""
    src, det, md = _desc_source(tmp_path, "train", 16384, 1024, 8, 12, 20480, ball_radius=1.0, ball_nsamples=64)
    n = 0
    for _ in src.feed(md):
        np.random.seed(n)
        md.optimize(epoch=0)
        assert math.isfinite(float(md.loss.detach()))
        for d in (md.anc_descriptors, md.pos_descriptors):
            norm = d.detach().norm(dim=1)
            assert float((norm - 1).abs().max()) < 1e-4
        n += 1
    assert n == 1
