"""Detector pair builder on the GPU (csrc/pairgen.cu, usip_b200.data.kitti_detector_loader).

Parity mode (the builder replays numpy's draws) against the reference loader's own batches in
tests/golden/detector_pairs.npz; device mode (Philox) for determinism and the distributions it must have; end to end
through KittiPairSource into ModelDetector.optimize()."""
import math
import os

import numpy as np
import pytest
import torch

from tests.test_pairgen_host import GOLDEN, case_opt, make_tree
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import ops
from usip_b200.data import kitti_detector_loader as kdl

pytestmark = pytest.mark.gpu
KEYS = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")


def _ulps(a, b):
    """fp32 ulp distance (sign-magnitude ordered)."""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))


def _one_scan(root, mode, index, S):
    pc = kdl.load_scan_npy(kdl.kitti_scan_path(str(root), mode, index), S)
    return torch.from_numpy(pc).to(dev()), np.array([0, len(pc)], np.int64)


def test_parity_mode_reproduces_the_reference_loader(tmp_path):
    g = np.load(GOLDEN)
    make_tree(g, tmp_path)
    names = sorted({k.split("/")[0] for k in g.files if k.endswith("/case")})
    same = total = 0
    for name in names:
        opt, mode, index, seed = case_opt(g, name)
        scans, offsets = _one_scan(tmp_path, mode, index, opt.surface_normal_len)
        b = kdl.DetectorPairBuilder(opt, mode, dev(), rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, offsets, [0])
        for k, t in zip(KEYS, out):
            got, ref = t[0].cpu().numpy(), g[name + "/" + k]
            if k in ("R", "scale", "shift") or mode == "test" and k.startswith("src"):
                np.testing.assert_array_equal(got.reshape(ref.shape), ref, err_msg=name + "/" + k)
            u = _ulps(got.reshape(ref.shape), ref)
            assert u.max() <= 2, (name, k, int(u.max()), float(np.abs(got.reshape(ref.shape) - ref).max()))
            same += int((u == 0).sum()); total += u.size
    frac = same / total
    print("pairgen parity: %.4f of %d coordinates bit-identical" % (frac, total))
    assert frac >= 0.99


def _device_builder(opt, mode="train", seed=5):
    return kdl.DetectorPairBuilder(opt, mode, dev(), seed=seed, rng="device")


def _kopt(**kw):
    base = dict(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                rot_perturbation=False, translation_perturbation=False, radius_threshold=100.0)
    base.update(kw)
    return make_opt(**base)


def _scans(ns, seed=0):
    arrs = [kdl.synthetic_scan(seed + i, n) for i, n in enumerate(ns)]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off, arrs


def test_device_mode_is_deterministic_per_step():
    scans, off, _ = _scans([3000, 2500, 4000])
    b = _device_builder(_kopt(rot_3d=True, rot_perturbation=True, translation_perturbation=True))
    a1 = [t.clone() for t in b.build(scans, off, [0, 2, 1], step=7)]
    a2 = b.build(scans, off, [0, 2, 1], step=7)
    a3 = b.build(scans, off, [0, 2, 1], step=8)
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[6], a3[6])
    R = a1[6].double()
    eye = torch.eye(3, dtype=torch.float64, device=R.device)
    assert float((R @ R.transpose(1, 2) - eye).abs().max()) < 1e-6
    assert float((torch.linalg.det(R) - 1).abs().max()) < 1e-6


def test_device_subsets_unique_inside_radius_and_tiled_evenly():
    ns = [8000, 1300]                                # ~1570 and ~255 points inside r = 20
    scans, off, arrs = _scans(ns, seed=40)
    opt = _kopt(radius_threshold=20.0)
    b = _device_builder(opt)
    b.build(scans, off, [0, 1], step=1)
    rows = b.last["rows"].cpu().numpy()
    cand = b.last["cand"].cpu().numpy()
    start = b.last["start"].cpu().numpy()
    for c in range(4):
        pc = arrs[c // 2]
        inside = kdl.radius_mask(pc, 20.0)
        r = rows[c]
        assert r.min() >= 0 and r.max() < len(pc) and inside[r].all()
        if inside.sum() >= opt.input_pc_num:
            assert len(np.unique(r)) == len(r)
            assert (np.diff(r) > 0).all()                              # ascending row index
        else:
            counts = np.bincount(r, minlength=len(pc))[inside]
            assert counts.sum() == opt.input_pc_num and counts.max() - counts.min() <= 1
        assert len(np.unique(cand[c])) == cand.shape[1] and (np.diff(cand[c]) > 0).all()
        assert 0 <= start[c] < cand.shape[1]


def test_device_subset_frequencies_chi_square():
    from scipy import stats
    scans, off, _ = _scans([64], seed=3)
    opt = _kopt(input_pc_num=48, node_num=4)
    b = _device_builder(opt, seed=123)
    counts = np.zeros(64)
    steps, B = 50, 8
    for s in range(steps):
        b.build(scans, off, [0] * B, step=s)
        counts += np.bincount(b.last["rows"].cpu().numpy().ravel(), minlength=64)
    expect = steps * 2 * B * 48 / 64
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    # without replacement each draw's counts are negatively correlated: the statistic is scaled by (64-48)/(64-1)
    p = stats.chi2.sf(chi2 / ((64 - 48) / 63), 63)
    assert p > 1e-4, (chi2, p)


def _clipped_std(sigma, clip):
    c = clip / sigma
    phi, Phi = math.exp(-c * c / 2) / math.sqrt(2 * math.pi), 0.5 * (1 + math.erf(c / math.sqrt(2)))
    return sigma * math.sqrt((2 * Phi - 1) - 2 * c * phi + c * c * 2 * (1 - Phi))


def test_device_jitter_is_clipped_normal_with_a_cloud_map():
    """With identity rotations, scale 1 and no shift, output - input is the jitter (to fp32 rounding)."""
    N, M, S = 16384, 512, 4
    pc = np.random.RandomState(0).uniform(-1, 1, (N, 8)).astype(np.float32)
    scans = torch.from_numpy(pc).to(dev())
    off = torch.tensor([0, N], dtype=torch.int64, device=dev())
    sp = torch.zeros(2, dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2, 1).contiguous()
    nodes = torch.from_numpy(np.ascontiguousarray(pc[:M, :3].T)).to(dev()).repeat(2, 1, 1).contiguous()
    params = np.zeros((1, ops.PAIR_PARAM_STRIDE))
    params[0, 27] = 1.0
    params[0, 31:40] = np.eye(3).ravel()
    params[0, 43] = 1.0
    out = ops.pair_augment(scans, off, sp, rows, nodes, torch.from_numpy(params).to(dev()), S, ops.PAIR_TRAIN,
                           seed=9, step=2)
    with pytest.raises(ValueError, match="both clouds"):               # a map with one entry per pair is refused
        ops.pair_augment(scans, off, sp[:1], rows, nodes, torch.from_numpy(params).to(dev()), S, ops.PAIR_TRAIN)
    src_pc, src_sn, src_node = (t.cpu().numpy()[0].astype(np.float64) for t in out[:3])
    j_pc = src_pc - pc[:, 0:3].T
    j_sn = src_sn - pc[:, 3:3 + S].T
    j_nd = src_node - pc[:M, 0:3].T
    for j, sigma, clip in ((j_pc, 0.04, 0.12), (j_sn, 0.01, 0.05), (j_nd, 0.04, 0.12)):
        assert np.abs(j).max() <= clip * (1 + 1e-5)
        sd = _clipped_std(sigma, clip)
        n = j.size
        assert abs(j.mean()) < 5 * sd / math.sqrt(n)
        assert abs(j.std() / sd - 1) < 6 / math.sqrt(2 * n) + 1e-3, (j.std(), sd)
    dst = out[3].cpu().numpy()[0] - pc[:, 0:3].T
    assert np.abs(dst - j_pc).max() > 1e-3                              # src and dst draw independent jitter


def test_device_nodes_are_fps_of_the_candidates():
    scans, off, _ = _scans([20480, 20480], seed=60)
    opt = _kopt(input_pc_num=16384, node_num=512)
    b = _device_builder(opt, mode="test")
    out = b.build(scans, off, [1, 0], step=3)
    _, nodes = ops.fps(b.last["candidates"], b.last["start"], 512, want_nodes=True)
    assert torch.equal(out[2], nodes[0::2])


def _source_model(tmp_path, N, M, B, counts, Ns):
    kdl.write_synthetic_kitti(str(tmp_path), counts, Ns, seed=90)
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    opt = _kopt(input_pc_num=N, node_num=M, batch_size=B)
    src = kdl.KittiPairSource(str(tmp_path), "train", opt, dev(), seed=1)
    md = ModelDetector(opt)
    load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
    return src, md, opt


def test_pair_source_feeds_optimize(tmp_path):
    src, md, _ = _source_model(tmp_path, 1024, 64, 2, [2, 2, 1, 1, 1, 1, 1, 1, 2, 0, 0], 1500)
    losses = []
    for _ in range(2):
        for _ in src.feed(md):
            md.optimize(epoch=0)
            losses.append(float(md.loss))
    assert len(losses) == 2 * len(src) and all(math.isfinite(v) for v in losses)


def test_pair_source_full_kitti_shape_step(tmp_path):
    src, md, _ = _source_model(tmp_path, 16384, 512, 2, [2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0], 20480)
    n = 0
    for _ in src.feed(md):
        md.optimize(epoch=0)
        assert math.isfinite(float(md.loss))
        n += 1
    assert n == 1


def test_graph_and_eager_train_steps_agree_on_a_built_batch(tmp_path):
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    scans, off, _ = _scans([5000, 6000], seed=80)
    opt = _kopt(input_pc_num=2048, node_num=64, batch_size=2)
    batch = _device_builder(opt).build(scans, off, [0, 1], step=0)
    losses = {}
    for graph in (False, True):
        md = ModelDetector(opt)
        load_params(md.detector, orc.init_detector_params(S=4, seed=1, randomize_bn=True))
        md.use_cuda_graph = graph
        ls = []
        for _ in range(2):
            md.set_input(*batch)
            md.optimize(epoch=0)
            ls.append(float(md.loss))
        losses[graph] = ls
    for x, y in zip(losses[False], losses[True]):
        assert abs(x - y) <= 5e-4 * abs(x), losses
