"""Repeatability on the GPU (csrc/repeatability.cu usip_repeatability_f64, csrc/pairgen.cu usip_test_cloud_gather,
usip_b200.evaluation.repeatability / kitti_test_loader / oxford_test_loader).

The kernel's counts against the float64 restatement of eval_rep.m (tests/rep_ref.py), exactly; the test clouds in
parity mode against the reference loaders' own batches (tests/golden/kitti_test_clouds.npz, oxford_test_clouds.npz),
bit for bit; device mode's determinism, subsets and frame; the selection order against save_keypoints.select_keypoints;
and the evaluator end to end against the restatement run on the keypoint files it writes."""
import os

import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests.rep_ref import pair_counts, repeatability_ref
from tests.test_repeatability_host import _kitti_tree
from tests.util_gpu import dev, golden, load_params, make_opt
from usip_b200 import ops
from usip_b200.evaluation import kitti_test_loader as ktl
from usip_b200.evaluation import oxford_test_loader as otl
from usip_b200.evaluation import repeatability as rep
from usip_b200.evaluation.save_keypoints import read_keypoints_bin, select_keypoints

pytestmark = pytest.mark.gpu


def _small_motion(rng):
    q = np.concatenate([[1.0], rng.normal(0, 0.02, 3)])
    return rep.gt_transform(rng.uniform(-0.2, 0.2, 3), q)


def _kernel_case(rng, S, M, P, oxford_frames):
    kp = rng.uniform(-1.5, 1.5, (S, 3, M)).astype(np.float32)
    order = np.stack([rng.permutation(M) for _ in range(S)]).astype(np.int32)
    count = rng.randint(1, M + 1, S).astype(np.int32)
    count[:3] = [1, M, 2]
    pairs = rng.randint(0, S, (P, 2)).astype(np.int32)
    frames = np.empty((P, 3, 3, 4))
    for p in range(P):
        if oxford_frames:
            F = rep.CAM_TO_ENU
        else:
            F = rep.cam_to_velodyne(np.concatenate([_small_motion(rng) * [1, 1, 1, 10], [[0, 0, 0, 1]]]))
        frames[p] = [F, F, _small_motion(rng)]
    return kp, order, count, pairs, frames


@pytest.mark.parametrize("oxford_frames", [False, True])
def test_kernel_matches_restatement(oxford_frames):
    rng = np.random.RandomState(11 + oxford_frames)
    S, M, P = 40, 77, 3000
    ks = [1, 5, 16, 40, 77, 100]
    kp, order, count, pairs, frames = _kernel_case(rng, S, M, P, oxford_frames)
    d = lambda a: torch.from_numpy(a).to(dev())
    inl, n_anc = ops.repeatability(d(kp), d(order), d(count), d(pairs), d(frames), ks, 0.5)
    ref_inl, ref_n = repeatability_ref(kp, order, count, pairs, frames, ks, 0.5)
    np.testing.assert_array_equal(n_anc.cpu().numpy(), ref_n)
    np.testing.assert_array_equal(inl.cpu().numpy(), ref_inl)
    assert 0 < ref_inl.sum() < ref_n.sum()            # neither all nor none are inliers


def test_identity_pairs_score_one():
    rng = np.random.RandomState(3)
    S, M = 6, 512
    kp, order, count, _, _ = _kernel_case(rng, S, M, 1, False)
    pairs = np.stack([np.arange(S), np.arange(S)], 1).astype(np.int32)
    F = rep.cam_to_velodyne(np.concatenate([_small_motion(rng), [[0, 0, 0, 1]]]))
    frames = np.stack([np.stack([F, F, np.eye(3, 4)])] * S)
    d = lambda a: torch.from_numpy(a).to(dev())
    ks = [4, 8, 16, 32, 64, 128, 256, 512]
    inl, n_anc = ops.repeatability(d(kp), d(order), d(count), d(pairs), d(frames), ks, 0.5)
    np.testing.assert_array_equal(inl.cpu().numpy(), n_anc.cpu().numpy())
    np.testing.assert_array_equal(n_anc.cpu().numpy(), np.minimum(np.array(ks)[None], count[:, None]))


def test_kernel_refusals():
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    kp = d(np.zeros((2, 3, 8), np.float32)); order = d(np.zeros((2, 8), np.int32)); cnt = d(np.ones(2, np.int32))
    pairs = d(np.zeros((1, 2), np.int32)); frames = d(np.zeros((1, 3, 3, 4)))
    for ks, r in (([8, 4], 0.5), ([0, 4], 0.5), ([4], 0.0)):
        with pytest.raises(RuntimeError):
            ops.repeatability(kp, order, cnt, pairs, frames, ks, r)
    big = d(np.zeros((1, 3, 5000), np.float32))
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.repeatability(big, d(np.zeros((1, 5000), np.int32)), d(np.ones(1, np.int32)), pairs, frames, [5000], 0.5)


# ----------------------------------------------------------------------------------------------- test clouds
def _source(name, root, rng_mode, batch_size=2, **opt_over):
    if name == "kitti":
        txt, num, _ = _kitti_tree(root)
        return ktl.KittiTestLoader(txt, num, make_opt(**opt_over), rng=rng_mode, batch_size=batch_size)
    otl.write_synthetic_oxford_test(root, range(5), 1300, [(0, 1)], os.path.join(root, "gt.txt"), seed=7500)
    return otl.OxfordTestLoader(root, make_opt(**opt_over), rng=rng_mode, batch_size=batch_size, numbers=range(5))


@pytest.mark.parametrize("name", ["kitti", "oxford"])
def test_parity_mode_matches_reference_loader(name, tmp_path):
    g = golden("%s_test_clouds.npz" % name)
    src = _source(name, str(tmp_path), "numpy", int(g["batch_size"]), input_pc_num=int(g["N"]), node_num=int(g["M"]))
    for case in ("plain", "noise"):
        seed = int(g[case + "/case"][0])
        np.random.seed(seed)
        torch.manual_seed(seed)
        got = {"pc": [], "sn": [], "node": []}
        for _, out in src.batches(float(g[case + "/noise_sigma"])):
            for k, v in zip(("pc", "sn", "node"), out):
                got[k].append(v.cpu().numpy())
        for k in got:
            np.testing.assert_array_equal(np.concatenate(got[k]), g[case + "/" + k], err_msg="%s %s" % (case, k))


@pytest.mark.parametrize("name", ["kitti", "oxford"])
def test_device_mode(name, tmp_path):
    src = _source(name, str(tmp_path), "device", 3, input_pc_num=1024, node_num=64)
    a = src.build([0, 1, 2], noise_sigma=0.1, step=5)
    last = {k: v.cpu().numpy() for k, v in src.last.items()}
    b = src.build([0, 1, 2], noise_sigma=0.1, step=5)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    plain = src.build([0, 1, 2], step=5)
    assert torch.equal(plain[1], a[1]) and torch.equal(plain[2], a[2]) and not torch.equal(plain[0], a[0])
    noise = (a[0] - plain[0]).cpu().numpy() / 0.1
    assert abs(noise.mean()) < 0.05 and abs(noise.std() - 1) < 0.05
    scans = src.load([0, 1, 2])
    for c in range(3):
        rows = last["rows"][c]
        assert len(np.unique(rows)) == len(rows) and rows.max() < len(scans[c])
        pts = last["candidates"][c]
        np.testing.assert_array_equal(pts, scans[c][rows[last["cand"][c]], :3])
        node = plain[2][c].cpu().numpy().T
        cand = pts if name == "kitti" else np.stack([pts[:, 0], -pts[:, 2], pts[:, 1]], 1)
        assert {tuple(p) for p in node} <= {tuple(p) for p in cand}
        raw = scans[c][rows]
        pc, sn = plain[0][c].cpu().numpy().T, plain[1][c].cpu().numpy().T
        if name == "oxford":                           # exact camera frame: (x, y, z) -> (x, -z, y)
            np.testing.assert_array_equal(pc, np.stack([raw[:, 0], -raw[:, 2], raw[:, 1]], 1))
            np.testing.assert_array_equal(sn[:, :3], np.stack([raw[:, 3], -raw[:, 5], raw[:, 4]], 1))
            np.testing.assert_array_equal(sn[:, 3], raw[:, 6])
        else:
            np.testing.assert_array_equal(pc, raw[:, :3])
            np.testing.assert_array_equal(sn, raw[:, 3:7])


# ----------------------------------------------------------------------------------------------- selection
@pytest.mark.parametrize("nms_radius", [0.0, 0.4])
def test_selection_prefix(nms_radius):
    g = torch.Generator().manual_seed(5)
    kp = (torch.rand((5, 3, 200), generator=g) * 4).to(dev())
    sg = torch.rand((5, 200), generator=g).to(dev())
    sg[:, 10:20] = sg[:, 0:1]                          # ties
    order, count = rep.select_order(kp, sg, nms_radius)
    for K in (4, 64, 200):
        ref = select_keypoints(kp, sg, nms_radius, K)
        for s in range(5):
            n = min(K, int(count[s]))
            assert torch.equal(kp[s][:, order[s, :n].long()].t(), ref[s])


# ----------------------------------------------------------------------------------------------- end to end
def _model(N, M, B):
    from usip_b200.models.keypoint_detector import ModelDetector
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M)
    md = ModelDetector(opt)
    P = orc.init_detector_params(S=4, seed=21, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    load_params(md.detector, P)
    return md, opt


@pytest.mark.parametrize("name", ["kitti", "oxford"])
@pytest.mark.parametrize("nms_radius", [0.0, 1.0])
def test_end_to_end_against_keypoint_files(name, nms_radius, tmp_path):
    root = str(tmp_path)
    N, M, B = 1024, 64, 2
    md, opt = _model(N, M, B)
    if name == "kitti":
        txt, num, cal = os.path.join(root, "txt"), os.path.join(root, "numpy"), os.path.join(root, "calib")
        ktl.write_synthetic_kitti_test(txt, num, cal, [4, 3], 1500,
                                       [[(0, 1), (1, 2), (2, 2), (3, 0)], [(0, 1), (2, 2), (1, 2)]], seed=3)
        ev = rep.KittiRepeatability(txt, num, cal, opt, seed=9, batch_size=B)
    else:
        gt = os.path.join(root, "groundtruths.txt")
        otl.write_synthetic_oxford_test(root, [0, 1, 2, 3, 4], 1500, [(0, 1), (2, 2), (3, 4), (4, 4), (1, 3)], gt, seed=4)
        ev = rep.OxfordRepeatability(root, gt, opt, seed=9, batch_size=B, numbers=range(5))
    ks = [4, 16, 64, 100]
    res = ev.run(md, ks, nms_radius=nms_radius, noise_sigma=0.01)
    out = os.path.join(root, "kp")
    for k, K in enumerate(ks):
        ev.write_keypoint_tree(out, K)
        for p, ((a, b), f) in enumerate(zip(ev.pairs, ev.frames)):
            anc = read_keypoints_bin(ev.source.keypoint_path(out, a))
            pos = read_keypoints_bin(ev.source.keypoint_path(out, b))
            inl, n = pair_counts(anc, pos, f[0], f[1], f[2], [K], 0.5)
            assert (res.inliers[p, k], res.n_anc[p, k]) == (inl[0], n[0]), (p, K)
            if a == b:
                assert res.repeatability[p, k] == 1.0
    assert len(res.lines()) == 2 * len(ks)
