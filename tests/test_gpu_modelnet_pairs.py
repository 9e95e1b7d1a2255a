"""ModelNet pair builder on the GPU (csrc/pairgen.cu usip_modelnet_pair_augment, usip_b200.data.modelnet_shrec_loader).

Parity mode (the builder replays numpy's draws) against the reference loader's own batches in
tests/golden/modelnet_pairs.npz; device mode (Philox) for determinism, the shared jitter and its laws, the sn arithmetic;
end to end through ModelNetPairSource into ModelDetector.optimize()."""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_pairgen import _clipped_std, _ulps
from tests.test_modelnet_pairs_host import case_opt, golden_cases, make_tree, split_scans
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import _lib, ops
from usip_b200.data import modelnet_shrec_loader as mnl

pytestmark = pytest.mark.gpu
KEYS = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")


def test_parity_mode_reproduces_the_reference_loader(tmp_path):
    g, names = golden_cases()
    make_tree(g, tmp_path)
    same = total = 0
    for name in names:
        opt, mode, items, seed = case_opt(g, name)
        arrs, off = split_scans(tmp_path, mode, opt)
        scans = torch.from_numpy(np.concatenate(arrs)).to(dev())
        b = mnl.ModelNetPairBuilder(opt, mode, dev(), rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, off, items)
        for k, t in zip(KEYS, out):
            got, ref = t.cpu().numpy(), g[name + "/" + k]
            got = got.reshape(ref.shape)
            if k in ("R", "scale", "shift") or mode == "test" and k.startswith("src"):
                np.testing.assert_array_equal(got, ref, err_msg=name + "/" + k)
            u = _ulps(got, ref)
            assert u.max() <= 2, (name, k, int(u.max()), float(np.abs(got - ref).max()))
            same += int((u == 0).sum()); total += u.size
    frac = same / total
    print("modelnet pairgen parity: %.4f of %d coordinates bit-identical" % (frac, total))
    assert frac >= 0.99


def _mopt(**kw):
    base = dict(dataset="modelnet", classes=40, input_pc_num=1000, node_num=64, surface_normal_len=3, node_knn_k_1=32,
                rot_horizontal=False, rot_3d=True, rot_perturbation=False, translation_perturbation=False,
                scene="object", loss_sigma_lower_bound=1e-4, keypoint_on_pc_alpha=1.0)
    base.update(kw)
    return make_opt(**base)


def _objects(ns, seed=0):
    arrs = [mnl.synthetic_object(seed + i, n) for i, n in enumerate(ns)]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off, arrs


def test_device_mode_is_deterministic_per_step():
    scans, off, _ = _objects([3000, 2500, 4000])
    b = mnl.ModelNetPairBuilder(_mopt(rot_horizontal=True, rot_perturbation=True, translation_perturbation=True),
                                "train", dev(), seed=5)
    a1 = [t.clone() for t in b.build(scans, off, [0, 2, 1], step=7)]
    a2 = b.build(scans, off, [0, 2, 1], step=7)
    a3 = b.build(scans, off, [0, 2, 1], step=8)
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[6], a3[6])
    R = a1[6].double()
    eye = torch.eye(3, dtype=torch.float64, device=R.device)
    assert float((R @ R.transpose(1, 2) - eye).abs().max()) < 1e-6
    assert float((a1[7] - 1).abs().max()) <= 0.2 and float(a1[8].abs().max()) <= 0.5


def _identity_inputs(N, M, B=1, seed=0):
    """One object whose rows are taken in order by both clouds of B pairs, its first M points as both clouds' nodes,
    and params with identity rotations, scale 1 and no shift."""
    pc = np.random.RandomState(seed).uniform(-1, 1, (N, 6)).astype(np.float32)
    scans = torch.from_numpy(pc).to(dev())
    off = torch.tensor([0, N], dtype=torch.int64, device=dev())
    soc = torch.zeros(2 * B, dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2 * B, 1).contiguous()
    nodes = torch.from_numpy(np.ascontiguousarray(pc[:M, :3].T)).to(dev()).repeat(2 * B, 1, 1).contiguous()
    params = np.zeros((B, ops.PAIR_PARAM_STRIDE))
    for r in range(3):
        params[:, 9 * r:9 * r + 9] = np.eye(3).ravel()
    params[:, 27] = 1.0
    params[:, 31:40] = np.eye(3).ravel()
    params[:, 43] = 1.0
    return pc, scans, off, soc, rows, nodes, params


def test_device_jitter_is_shared_by_both_clouds_and_clipped_normal():
    """Identical rows in both clouds and identity params: src - input == dst - input exactly, and the difference follows
    the reference's laws (sigma 0.01 / clip 0.05 for pc and sn, 0.04 / 0.1 for nodes).  Two pairs draw different
    jitter."""
    N, M = 16384, 512
    pc, scans, off, soc, rows, nodes, params = _identity_inputs(N, M, B=2)
    out = ops.modelnet_pair_augment(scans, off, soc, rows, nodes, torch.from_numpy(params).to(dev()), ops.PAIR_TRAIN,
                                    seed=9, step=2)
    o = [t.cpu().numpy().astype(np.float64) for t in out]
    j_pc, j_sn, j_nd = o[0] - pc[:, 0:3].T, o[1] - pc[:, 3:6].T, o[2] - pc[:M, 0:3].T
    np.testing.assert_array_equal(o[3] - pc[:, 0:3].T, j_pc)
    np.testing.assert_array_equal(o[4] - pc[:, 3:6].T, j_sn)
    np.testing.assert_array_equal(o[5] - pc[:M, 0:3].T, j_nd)
    for j, sigma, clip in ((j_pc, 0.01, 0.05), (j_sn, 0.01, 0.05), (j_nd, 0.04, 0.1)):
        assert np.abs(j).max() <= clip * (1 + 1e-5)
        assert np.abs(j[0] - j[1]).max() > sigma                       # pairs draw independently
        sd = _clipped_std(sigma, clip)
        n = j.size
        assert abs(j.mean()) < 5 * sd / math.sqrt(n)
        assert abs(j.std() / sd - 1) < 6 / math.sqrt(2 * n) + 1e-3, (j.std(), sd)


@pytest.mark.parametrize("flags", [ops.PAIR_ROT_3D | ops.PAIR_TRANSLATION, ops.PAIR_TRANSLATION])
def test_sn_is_jittered_and_scaled_never_shifted(flags):
    """Uploaded jitter, identity rotations, scale 1.15, shift 0.05: after a rotation (float64 chain) sn is
    fl32((sn + j) * s); without one (the float32 slice) fl32(fl32(sn + j) * fl32(s)).  pc is shifted, sn is not."""
    N, M, s = 4096, 64, 1.15
    pc, scans, off, soc, rows, nodes, params = _identity_inputs(N, M, seed=1)
    params[:, 27] = s
    params[:, 28:31] = 0.05
    rng = np.random.RandomState(3)
    jit = [np.clip(sd * rng.randn(1, n, 3), -c, c) for sd, c, n in ((0.01, 0.05, N), (0.01, 0.05, N), (0.04, 0.1, M))]
    out = ops.modelnet_pair_augment(scans, off, soc, rows, nodes, torch.from_numpy(params).to(dev()),
                                    ops.PAIR_TRAIN | flags, 0, 0, *[torch.from_numpy(j).to(dev()) for j in jit])
    sn, j_sn = pc[:, 3:6].astype(np.float64), jit[1][0]
    if flags & ops.PAIR_ROT_3D:
        expect = ((sn + j_sn) * s).astype(np.float32)
        expect_pc = ((pc[:, 0:3].astype(np.float64) + jit[0][0]) * s + 0.05).astype(np.float32)
    else:
        expect = (sn + j_sn).astype(np.float32) * np.float32(s)
        expect_pc = (((pc[:, 0:3] + jit[0][0]).astype(np.float32) * np.float32(s)).astype(np.float64) + 0.05)
        expect_pc = expect_pc.astype(np.float32)
    for side in (1, 4):                                             # src_sn, dst_sn (identity transform)
        np.testing.assert_array_equal(out[side][0].cpu().numpy(), expect.T)
    np.testing.assert_array_equal(out[0][0].cpu().numpy(), expect_pc.T)


def test_argument_checks():
    N, M = 256, 16
    _, scans, off, soc, rows, nodes, params = _identity_inputs(N, M)
    p = torch.from_numpy(params).to(dev())
    with pytest.raises(ValueError, match="one array per pair"):          # a per-cloud array is refused
        ops.modelnet_pair_augment(scans, off, soc, rows, nodes, p, ops.PAIR_TRAIN,
                                  jit_pc=torch.zeros((2, N, 3), dtype=torch.float64, device=dev()))
    with pytest.raises(_lib.UsipB200Error, match="columns 3:6"):
        ops.modelnet_pair_augment(scans[:, :5].contiguous(), off, soc, rows, nodes, p, ops.PAIR_TRAIN)


def test_device_subsets_candidates_and_nodes():
    scans, off, arrs = _objects([10000, 5000], seed=60)
    opt = _mopt(input_pc_num=5000, node_num=512)
    b = mnl.ModelNetPairBuilder(opt, "train", dev(), seed=3)
    out = b.build(scans, off, [1, 0], step=3)
    rows, cand = b.last["rows"].cpu().numpy(), b.last["cand"].cpu().numpy()
    assert cand.shape == (4, 5000 // 4)
    for c in range(4):
        r = rows[c]
        assert len(np.unique(r)) == len(r) and (np.diff(r) > 0).all() and r.max() < len(arrs[1 - c // 2])
        assert len(np.unique(cand[c])) == cand.shape[1] and (np.diff(cand[c]) > 0).all()
    assert not np.array_equal(rows[2], rows[3])                          # the two clouds subsample independently
    b2 = mnl.ModelNetPairBuilder(opt, "test", dev(), seed=3)
    out = b2.build(scans, off, [1, 0], step=3)
    _, nodes = ops.fps(b2.last["candidates"], b2.last["start"], 512, want_nodes=True)
    assert torch.equal(out[2], nodes[0::2])


def _source_model(tmp_path, N, M, B, n_train, rows):
    mnl.write_synthetic_modelnet(str(tmp_path), ("airplane", "night_stand", "cup"), n_train, 1, rows, seed=90)
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    opt = _mopt(input_pc_num=N, node_num=M, batch_size=B)
    src = mnl.ModelNetPairSource(str(tmp_path), "train", opt, dev(), seed=1)
    md = ModelDetector(opt)
    load_params(md.detector, orc.init_detector_params(S=3, seed=1, randomize_bn=True))
    return src, md


def test_pair_source_feeds_optimize(tmp_path):
    src, md = _source_model(tmp_path, 1000, 64, 2, 2, 1500)
    losses = []
    for _ in range(2):
        for _ in src.feed(md):
            md.optimize(epoch=0)
            losses.append(float(md.loss))
    assert len(src) == 3 and len(losses) == 6 and all(math.isfinite(v) for v in losses)


def test_pair_source_full_modelnet_shape_step(tmp_path):
    """BASELINE configs[1]: B=24, N=5000, M=512, S=3, Kn=32, scene 'object'."""
    src, md = _source_model(tmp_path, 5000, 512, 24, 9, 10000)
    n = 0
    for _ in src.feed(md):
        md.optimize(epoch=0)
        assert math.isfinite(float(md.loss))
        n += 1
    assert n == 1


def test_graph_and_eager_train_steps_agree_on_a_built_batch():
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    scans, off, _ = _objects([5000, 6000], seed=80)
    opt = _mopt(input_pc_num=2048, node_num=64, batch_size=2)
    batch = mnl.ModelNetPairBuilder(opt, "train", dev(), seed=5).build(scans, off, [0, 1], step=0)
    losses = {}
    for graph in (False, True):
        md = ModelDetector(opt)
        load_params(md.detector, orc.init_detector_params(S=3, seed=1, randomize_bn=True))
        md.use_cuda_graph = graph
        ls = []
        for _ in range(2):
            md.set_input(*batch)
            md.optimize(epoch=0)
            ls.append(float(md.loss))
        losses[graph] = ls
    for x, y in zip(losses[False], losses[True]):
        assert abs(x - y) <= 5e-4 * abs(x), losses
