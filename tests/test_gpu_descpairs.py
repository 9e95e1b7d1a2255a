"""Descriptor pair builder on the GPU (csrc/pairgen.cu, usip_b200.data.kitti_descriptor_loader).

Parity mode (the builder replays numpy's draws) against the reference loader's own batches in
tests/golden/descriptor_pairs.npz; device mode (Philox) for determinism and the distributions it must have; end to end
through KittiDescriptorPairSource and a frozen ModelDetector into ModelDescriptor.optimize()."""
import math
import random

import numpy as np
import pytest
import torch

from tests.test_descpairs_host import case_opt, golden_cases, make_tree
from tests.test_gpu_pairgen import _clipped_std, _ulps
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import ops
from usip_b200.data import kitti_descriptor_loader as kdesc
from usip_b200.data import kitti_detector_loader as kdl

pytestmark = pytest.mark.gpu
KEYS = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node")


def _tree_scans(root, mode, S):
    _, _, _, accs = kdl.make_dataset_kitti(str(root), mode)
    arrs = [kdl.load_scan_npy(kdl.kitti_scan_path(str(root), mode, i), S) for i in range(accs[-1])]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off


def test_parity_mode_reproduces_the_reference_loader(tmp_path):
    g, names = golden_cases()
    make_tree(g, tmp_path)
    same = total = 0
    for name in names:
        opt, mode, anchors, seed = case_opt(g, name)
        scans, off = _tree_scans(tmp_path, mode, opt.surface_normal_len)
        _, _, nums, accs = kdl.make_dataset_kitti(str(tmp_path), mode)
        seq, poses = kdesc.load_kitti_poses(str(tmp_path), mode)
        b = kdesc.DescriptorPairBuilder(opt, mode, dev(), rng="numpy")
        np.random.seed(seed)
        random.seed(seed)
        pos = [kdesc.nearby_index(a, poses, accs, nums, opt.positive_radius_threshold, random) for a in anchors]
        out = b.build(scans, off, anchors, pos)
        with pytest.warns(UserWarning) if name == "s5" else _nothing():
            neg = kdesc.mine_negative_sample(seq[anchors], poses[anchors].astype(np.float32),
                                             opt.negative_radius_threshold)
        np.testing.assert_array_equal(seq[pos], g[name + "/pos_seq"], err_msg=name)
        np.testing.assert_array_equal(neg.numpy(), g[name + "/neg_idx"], err_msg=name)
        for k, t in zip(KEYS, out):
            got, ref = t.cpu().numpy(), g[name + "/" + k]
            assert got.shape == ref.shape, (name, k, got.shape, ref.shape)
            if mode == "test":
                np.testing.assert_array_equal(got, ref, err_msg=name + "/" + k)
            u = _ulps(got, ref)
            assert u.max() <= 2, (name, k, int(u.max()), float(np.abs(got - ref).max()))
            same += int((u == 0).sum()); total += u.size
    frac = same / total
    print("descpairs parity: %.5f of %d coordinates bit-identical" % (frac, total))
    assert frac >= 0.99


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _kopt(**kw):
    base = dict(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                rot_perturbation=False, translation_perturbation=False, positive_radius_threshold=5.0,
                negative_radius_threshold=50.0)
    base.update(kw)
    return make_opt(**base)


def _scans(ns, seed=0):
    arrs = [kdl.synthetic_scan(seed + i, n) for i, n in enumerate(ns)]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off, arrs


def _device_builder(opt, mode="train", seed=5):
    return kdesc.DescriptorPairBuilder(opt, mode, dev(), seed=seed, rng="device")


def test_device_mode_is_deterministic_per_step():
    scans, off, _ = _scans([3000, 2500, 4000, 1100])
    b = _device_builder(_kopt(rot_3d=True, rot_perturbation=True, translation_perturbation=True))
    a1 = [t.clone() for t in b.build(scans, off, [0, 2], [1, 3], step=7)]
    a2 = b.build(scans, off, [0, 2], [1, 3], step=7)
    a3 = b.build(scans, off, [0, 2], [1, 3], step=8)
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[5], a3[5])


def test_device_subsets_unique_and_from_their_own_scan():
    ns = [3000, 1500, 1024, 2600]
    scans, off, arrs = _scans(ns, seed=40)
    opt = _kopt()
    b = _device_builder(opt, mode="test")
    anc, pos = [0, 2], [1, 3]
    out = b.build(scans, off, anc, pos, step=1)
    rows, cand, start = (b.last[k].cpu().numpy() for k in ("rows", "cand", "start"))
    for c in range(4):
        pc = arrs[(anc if c % 2 == 0 else pos)[c // 2]]
        r = rows[c]
        assert r.min() >= 0 and r.max() < len(pc)
        assert len(np.unique(r)) == len(r) and (np.diff(r) > 0).all()
        assert len(np.unique(cand[c])) == cand.shape[1] == opt.input_pc_num // 4 and (np.diff(cand[c]) > 0).all()
        assert 0 <= start[c] < cand.shape[1]
        got_pc = out[0 if c % 2 == 0 else 3][c // 2].cpu().numpy()
        got_sn = out[1 if c % 2 == 0 else 4][c // 2].cpu().numpy()
        np.testing.assert_array_equal(got_pc, pc[r, 0:3].T)               # test mode: the rows as they are
        np.testing.assert_array_equal(got_sn, pc[r, 3:7].T)


def test_device_subset_frequencies_chi_square():
    from scipy import stats
    scans, off, _ = _scans([64, 80], seed=3)
    opt = _kopt(input_pc_num=48, node_num=4)
    b = _device_builder(opt, seed=123)
    steps, B = 50, 8
    counts = [np.zeros(64), np.zeros(80)]
    for s in range(steps):
        b.build(scans, off, [0] * B, [1] * B, step=s)
        rows = b.last["rows"].cpu().numpy()
        counts[0] += np.bincount(rows[0::2].ravel(), minlength=64)
        counts[1] += np.bincount(rows[1::2].ravel(), minlength=80)
    for n, cnt in zip((64, 80), counts):
        expect = steps * B * 48 / n
        chi2 = float(((cnt - expect) ** 2 / expect).sum())
        p = stats.chi2.sf(chi2 / ((n - 48) / (n - 1)), n - 1)   # draws without replacement: scaled statistic
        assert p > 1e-4, (n, chi2, p)


def test_device_jitter_is_clipped_normal_with_the_scale_in_params():
    """With no rotation flag, scale 1 and no shift, output - input is the jitter (to fp32 rounding)."""
    N, M, S = 16384, 512, 4
    pc = np.random.RandomState(0).uniform(-1, 1, (2 * N, 8)).astype(np.float32)
    scans = torch.from_numpy(pc).to(dev())
    off = torch.tensor([0, N, 2 * N], dtype=torch.int64, device=dev())
    soc = torch.tensor([0, 1], dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2, 1).contiguous()
    nodes = torch.from_numpy(np.stack([pc[:M, :3].T, pc[N:N + M, :3].T])).to(dev()).contiguous()
    params = torch.zeros((2, ops.DESC_PARAM_STRIDE), dtype=torch.float64, device=dev())
    params[:, 27] = 1
    out = ops.desc_pair_augment(scans, off, soc, rows, nodes, params, S, ops.PAIR_TRAIN, seed=9, step=2)
    got = [t.cpu().numpy()[0].astype(np.float64) for t in out]
    j_pc = [got[0] - pc[:N, 0:3].T, got[3] - pc[N:, 0:3].T]
    j_sn = [got[1] - pc[:N, 3:3 + S].T, got[4] - pc[N:, 3:3 + S].T]
    j_nd = [got[2] - pc[:M, 0:3].T, got[5] - pc[N:N + M, 0:3].T]
    for j, sigma, clip in ((np.stack(j_pc), 0.04, 0.12), (np.stack(j_sn), 0.01, 0.05), (np.stack(j_nd), 0.04, 0.12)):
        assert np.abs(j).max() <= clip * (1 + 1e-5)
        sd = _clipped_std(sigma, clip)
        n = j.size
        assert abs(j.mean()) < 5 * sd / math.sqrt(n)
        assert abs(j.std() / sd - 1) < 6 / math.sqrt(2 * n) + 1e-3, (j.std(), sd)
    assert np.abs(j_pc[0] - j_pc[1]).max() > 1e-3                       # anchor and positive draw their own jitter


def test_device_nodes_are_fps_of_the_candidates():
    scans, off, _ = _scans([20480, 20480, 17000], seed=60)
    opt = _kopt(input_pc_num=16384, node_num=256)
    b = _device_builder(opt, mode="test")
    out = b.build(scans, off, [1, 0], [2, 1], step=3)
    _, nodes = ops.fps(b.last["candidates"], b.last["start"], 256, want_nodes=True)
    assert torch.equal(out[2], nodes[0::2]) and torch.equal(out[5], nodes[1::2])


def test_anchor_and_positive_share_the_scale_and_rotate_independently():
    scans, off, arrs = _scans([3000, 3000, 3000], seed=70)
    opt = _kopt()
    b = _device_builder(opt, seed=11)
    out = b.build(scans, off, [0, 2, 1], [1, 0, 2], step=4)
    P = b.last["params"].cpu().numpy()
    scale = b.last["scale"].cpu().numpy()
    rows = b.last["rows"].cpu().numpy()
    assert np.all((0.9 <= scale) & (scale <= 1.1)) and len(np.unique(scale)) == 3
    for pair in range(3):
        assert P[2 * pair, 27] == P[2 * pair + 1, 27] == scale[pair]
        assert np.abs(P[2 * pair, 0:9] - P[2 * pair + 1, 0:9]).max() > 1e-3
        for side, scan in ((0, [0, 2, 1][pair]), (1, [1, 0, 2][pair])):
            c = 2 * pair + side
            R = P[c, 0:9].reshape(3, 3)
            np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-12)
            xyz = arrs[scan][rows[c], 0:3].astype(np.float64)
            got = out[3 * side][pair].cpu().numpy().T.astype(np.float64)
            resid = got / scale[pair] - xyz @ R                             # the jitter, scaled back
            assert np.abs(resid).max() <= 0.12 + 1e-4, (pair, side, np.abs(resid).max())


# ------------------------------------------------------------------------------------------------ end to end
def _trajectory(counts):
    poses = []
    for s, n in enumerate(counts):
        ps = []
        for i in range(n):
            P = np.eye(4)
            P[:3, 3] = [1000.0 * s + 2.0 * i, 0.0, 0.0]
            ps.append(P)
        poses.append(ps)
    return poses


def _source_models(tmp_path, N, M, B, counts, Ns, **kw):
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    from usip_b200.models.keypoint_detector import ModelDetector
    kdl.write_synthetic_kitti(str(tmp_path), counts, Ns, seed=90, poses=_trajectory(counts))
    opt = _kopt(input_pc_num=N, node_num=M, batch_size=B, **kw)
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    det.freeze_model()
    src = kdesc.KittiDescriptorPairSource(str(tmp_path), "train", opt, det, dev(), seed=1)
    torch.manual_seed(3)
    md = ModelDescriptor(opt)
    return src, det, md, opt


def _check_source(src, det, md, opt, epochs):
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    losses, first = [], None
    for _ in range(epochs):
        for out in src.feed(md):
            c = src.last["clouds"]
            (kp_a, kp_p), (sg_a, sg_p) = det.run_model_siamese((c[0], c[3]), (c[1], c[4]), (c[2], c[5]))
            for got, ref in zip((out[2], out[6], out[3], out[7]), (kp_a, kp_p, sg_a, sg_p)):
                assert torch.equal(got, ref)                        # same keypoints as on the default stream
            assert out[8].dtype == torch.int64 and torch.equal(out[8].cpu(), src.last["neg_idx"])
            if first is None:
                first = [t.clone() for t in out]
            np.random.seed(len(losses))                            # the descriptor forward draws a permutation
            md.optimize(epoch=0)
            losses.append(float(md.loss.detach()))
    assert len(losses) == epochs * len(src) and all(math.isfinite(v) for v in losses)
    torch.manual_seed(3)
    md2 = ModelDescriptor(opt)
    md2.set_input(*first)
    np.random.seed(0)
    md2.optimize(epoch=0)
    assert float(md2.loss.detach()) == losses[0], (float(md2.loss.detach()), losses[0])   # the hand-over changes nothing
    return losses


def test_descriptor_source_feeds_optimize(tmp_path):
    src, det, md, opt = _source_models(tmp_path, 1024, 64, 2, [6, 2, 2, 0, 0, 0, 0, 0, 2, 0, 0], 1300,
                                       ball_nsamples=32)
    _check_source(src, det, md, opt, epochs=2)


def test_descriptor_source_full_kitti_shape_step(tmp_path):
    src, det, md, opt = _source_models(tmp_path, 16384, 256, 8, [10, 6, 0, 0, 0, 0, 0, 0, 0, 0, 0], 20480,
                                       ball_radius=2.0, ball_nsamples=64)
    _check_source(src, det, md, opt, epochs=1)
