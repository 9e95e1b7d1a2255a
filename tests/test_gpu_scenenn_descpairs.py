"""SceneNN descriptor pairs on the GPU (usip_b200/data/scenenn_descriptor_loader.py, csrc/pairgen.cu's
usip_cloud_gather_candidates_icp_f64 and usip_scenenn_desc_pair_augment, csrc/fps.cu's usip_fps_f64): parity mode
against the unmodified reference loader (tests/golden/scenenn_descpairs.npz), usip_fps_f64 against usip_fps_f32 and a
float64 FarthestSampler, device mode against the float64 restatement of tests/scenenn_desc_ref.py, determinism, full
coverage of the outputs, the three residencies, the geometric hand-over to the loss, and the source feeding
ModelDescriptorIndoor."""
import math
import os

import numpy as np
import pytest
import torch

from tests import scenenn_desc_ref as pr
from tests.test_gpu_pairgen import _ulps
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import ops
from usip_b200.data import scenenn_descriptor_loader as sdl
from usip_b200.data import scenenn_detector_loader as snl

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scenenn_descpairs.npz")
KEYS = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node", "R", "scale", "shift")
KIND = {"train": 2, "val": 1, "test": 0}


def _sopt(**kw):
    base = dict(input_pc_num=1024, node_num=64, surface_normal_len=4, node_knn_k_1=4, k=1, rot_horizontal=True,
                rot_3d=False, rot_perturbation=True, translation_perturbation=False, scene="indoor",
                loss_sigma_lower_bound=1e-4, keypoint_on_pc_alpha=10.0, batch_size=2, ball_radius=0.6,
                ball_nsamples=64, descriptor_len=128, CGF_radius=0.3, triple_loss_gamma=0.5, sigma_max=3.0)
    base.update(kw)
    return make_opt(**base)


def _golden_tree(root, g):
    counts = dict(zip(("train", "val", "test"), (int(v) for v in g["tree/counts"])))
    pairs = {s: [tuple(int(x) for x in p) for p in g["tree/pairs_" + s]] for s in counts}
    rows = lambda split, i: 600 if (split, i) in (("train", 4), ("train", 5)) else 1300
    snl.write_synthetic_scenenn(root, counts, rows, seed=int(g["tree/seed"]), pairs=pairs)


def _frames(root, splits, frames):
    """Host scans of the items' frames, anchor and positive of each item in turn -> (scans, offsets)."""
    arrs = [np.load(os.path.join(root, "frames_" + s, "%d.npy" % int(f))) for s, fr in zip(splits, frames) for f in fr]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)), off


def test_parity_mode_matches_the_reference(tmp_path):
    g = np.load(GOLDEN)
    _golden_tree(str(tmp_path), g)
    differing = total = 0
    for name in ("train", "rot3d", "s3", "short", "val", "test", "seq", "wdiv"):
        seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
        opt = _sopt(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S, rot_horizontal=bool(rh),
                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp))
        splits = [str(s) for s in g[name + "/split"]]
        scans, off = _frames(str(tmp_path), splits, g[name + "/frames"])
        n = len(splits)
        b = sdl.SceneNNDescriptorPairBuilder(opt, device=dev(), rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, off, 2 * np.arange(n), 2 * np.arange(n) + 1, g[name + "/icp"], [KIND[s] for s in splits])
        torch.cuda.synchronize()
        for k, t in zip(KEYS, out):
            got, ref = t.cpu().numpy(), g[name + "/" + k].reshape(t.shape)
            u = _ulps(got, ref)
            assert u.max() <= 1, (name, k, int(u.max()))
            differing += int((u > 0).sum()); total += u.size
    print("scenenn_descpairs parity: %d of %d elements differ from the reference (each by 1 fp32 ulp)"
          % (differing, total))


def test_parity_nodes_are_the_reference_fps_selection(tmp_path):
    """The anchor's node i is the ICP'd candidate the float64 FarthestSampler picks, restated on the host from the
    builder's own candidates and start; with no augmentation (test) the nodes are those points cast."""
    g = np.load(GOLDEN)
    _golden_tree(str(tmp_path), g)
    for name in ("test", "wdiv", "short"):
        seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
        opt = _sopt(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S, rot_horizontal=bool(rh),
                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp))
        splits = [str(s) for s in g[name + "/split"]]
        scans, off = _frames(str(tmp_path), splits, g[name + "/frames"])
        b = sdl.SceneNNDescriptorPairBuilder(opt, device=dev(), rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, off, [0], [1], g[name + "/icp"], [KIND[s] for s in splits])
        pts = b.last["candidates"].cpu().numpy()
        idx = b.last["node_idx"].cpu().numpy()
        start = b.last["start"].cpu().numpy()
        for c in range(2):
            np.testing.assert_array_equal(idx[c], pr.farthest_sampler(pts[c], start[c], opt.node_num))
        if name == "test":
            np.testing.assert_array_equal(out[2][0].cpu().numpy(), pts[0][idx[0]].T.astype(np.float32))
        np.testing.assert_array_equal(_ulps(out[2][0].cpu().numpy(), g[name + "/anc_node"][0]) <= 1, True)


# ------------------------------------------------------------------------------------------------- usip_fps_f64
@pytest.mark.parametrize("Ns,k", [(1, 1), (3000, 1), (3000, 200), (8192, 256), (5000, 512)])
def test_fps_f64_matches_f32_and_the_float64_sampler(Ns, k):
    r = np.random.RandomState(Ns + k)
    p32 = r.uniform(-3, 3, (3, Ns, 3)).astype(np.float32)
    start = r.randint(0, Ns, 3).astype(np.int32)
    i32, n32 = ops.fps(torch.from_numpy(p32).to(dev()), torch.from_numpy(start).to(dev()), k)
    i64, n64 = ops.fps_f64(torch.from_numpy(p32.astype(np.float64)).to(dev()), torch.from_numpy(start).to(dev()), k,
                           want_nodes=True)
    assert torch.equal(i32, i64) and torch.equal(n32, n64)
    T = np.eye(4)
    c, s = math.cos(0.7), math.sin(0.7)
    T[0:3, 0:3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
    T[0:3, 3] = [0.3, -0.2, 0.1]
    p64 = np.stack([pr.icp_map(T, p) for p in p32])                 # ICP'd: not float32 values
    i64, _ = ops.fps_f64(torch.from_numpy(p64).to(dev()), torch.from_numpy(start).to(dev()), k)
    i64 = i64.cpu().numpy()
    for b in range(3):
        np.testing.assert_array_equal(i64[b], pr.farthest_sampler(p64[b], start[b], k))


# ------------------------------------------------------------------------------------------------- device mode
def _device_tree(root, counts=None, rows=1500):
    counts = counts or {"train": 8, "val": 4, "test": 14}
    pairs = {"train": [(0, 1), (2, 3), (4, 5), (6, 7)], "val": [(0, 1), (2, 3)],
             "test": [(2 * k, 2 * k + 1) for k in range(7)]}             # the listing keeps pairs 0, 3 and 6
    snl.write_synthetic_scenenn(root, counts, rows, seed=11, pairs=pairs)


def _device_batch(root, opt, items, step=3, seed=5):
    pairs = {s: sdl.scenenn_pairs(root, s) for s in ("train", "val", "test")}
    splits = [s for s, _ in items]
    frames = [pairs[s][0][i] for s, i in items]
    icp = np.stack([pairs[s][1][i] for s, i in items])
    scans, off = _frames(root, splits, frames)
    b = sdl.SceneNNDescriptorPairBuilder(opt, device=dev(), seed=seed)
    n = len(items)
    out = b.build(scans.to(dev()), off, 2 * np.arange(n), 2 * np.arange(n) + 1, icp, [KIND[s] for s in splits],
                  step=step)
    return b, out, scans.numpy(), off, icp


@pytest.mark.parametrize("kw", [dict(), dict(rot_horizontal=False, rot_3d=True, translation_perturbation=True),
                                dict(rot_horizontal=False, rot_perturbation=False, translation_perturbation=True,
                                     surface_normal_len=3)])
def test_device_mode_matches_the_float64_restatement(tmp_path, kw):
    root = str(tmp_path)
    _device_tree(root)
    opt = _sopt(**kw)
    items = [("train", 0), ("val", 1), ("test", 2), ("train", 3)]
    b, out, scans, off, icp = _device_batch(root, opt, items)
    L = {k: v.cpu().numpy() for k, v in b.last.items() if torch.is_tensor(v)}
    soc = np.arange(2 * len(items))
    cand = pr.gather_candidates_icp(scans, off, soc, L["rows"], L["cand"], icp)
    np.testing.assert_allclose(L["candidates"], cand, rtol=0, atol=1e-12)
    for c in range(len(soc)):
        np.testing.assert_array_equal(L["node_idx"][c], pr.farthest_sampler(L["candidates"][c], L["start"][c],
                                                                            opt.node_num))
    ref = pr.scenenn_desc_pair_augment(scans, off, soc, L["rows"], icp, L["candidates"], L["node_idx"], L["params"],
                                       opt.surface_normal_len, b.flags)
    for k, t, r in zip(KEYS, out, ref):
        u = _ulps(t.cpu().numpy(), np.asarray(r).reshape(t.shape))
        assert u.max() <= 1, (k, int(u.max()))


def test_device_mode_is_deterministic_per_step(tmp_path):
    root = str(tmp_path)
    _device_tree(root)
    items = [("train", 0), ("val", 0), ("train", 2)]
    _, a1, *_ = _device_batch(root, _sopt(), items, step=7)
    a1 = [t.clone() for t in a1]
    _, a2, *_ = _device_batch(root, _sopt(), items, step=7)
    _, a3, *_ = _device_batch(root, _sopt(), items, step=8)
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[6], a3[6])


def test_every_output_element_is_written(tmp_path):
    """17 pairs over 4 shared frame pairs of every kind, built into memory that held NaN: no output element is left
    unwritten."""
    root = str(tmp_path)
    _device_tree(root)
    pairs = {s: sdl.scenenn_pairs(root, s) for s in ("train", "val", "test")}
    shared = [("train", 0), ("val", 1), ("test", 2), ("train", 3)]
    scans, off = _frames(root, [s for s, _ in shared], [pairs[s][0][i] for s, i in shared])
    which = np.arange(17) % 4
    icp = np.stack([pairs[shared[w][0]][1][shared[w][1]] for w in which])
    junk = torch.full((64 << 20,), float("nan"), device=dev())
    del junk
    b = sdl.SceneNNDescriptorPairBuilder(_sopt(), device=dev(), seed=1)
    out = b.build(scans.to(dev()), off, 2 * which, 2 * which + 1, icp, [KIND[shared[w][0]] for w in which], step=2)
    assert out[0].shape == (17, 3, 1024)
    for k, t in zip(KEYS, out):
        assert torch.isfinite(t).all(), k


def test_geometric_invariant(tmp_path):
    """Every anchor row, mapped by the batch's (R, scale, shift), lands on the positive row that came from the same
    source point -- in every kind: the ICP direction, the pair-shared augmentation and the transform the loss's
    _transform_anchor_keypoints applies all agree."""
    root = str(tmp_path)
    _device_tree(root, rows=900)
    for kw in (dict(), dict(rot_horizontal=False, rot_3d=True, translation_perturbation=True)):
        b, out, *_ = _device_batch(root, _sopt(**kw), [("train", 1), ("val", 0), ("test", 1), ("train", 2)])
        anc_pc, pos_pc, R, scale, shift = (out[0].double(), out[3].double(), out[6].double(), out[7].double(),
                                           out[8].double())
        mapped = (R @ anc_pc * scale[:, None, None] + shift).cpu().numpy()
        rows = b.last["rows"].cpu().numpy()
        pos = pos_pc.cpu().numpy()
        for p in range(len(rows) // 2):
            _, ia, ip = np.intersect1d(rows[2 * p], rows[2 * p + 1], return_indices=True)
            assert len(ia) > 100
            err = np.abs(mapped[p][:, ia] - pos[p][:, ip]).max()
            assert err < 2e-5 * max(1.0, np.abs(pos[p]).max()), (kw, p, err)


# ------------------------------------------------------------------------------------------------- the source
def _detector(opt):
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    det = ModelDetector(opt)
    load_params(det.detector, orc.init_detector_params(S=opt.surface_normal_len, seed=1, C1=64, C2=256,  # indoor
                                                       randomize_bn=True))
    det.freeze_model()
    return det


def test_residencies_give_the_same_batches(tmp_path):
    root = str(tmp_path)
    _device_tree(root)
    opt = _sopt()
    det = _detector(opt)
    got = []
    for resident in ("host", "device", "disk"):
        src = sdl.SceneNNDescriptorPairSource(root, "train+val", opt, det, dev(), seed=4, resident=resident)
        got.append([[t.clone() for t in out] for out, ev in src.batches()])
        torch.cuda.synchronize()
    assert len(got[0]) == 3
    for other in got[1:]:
        for x, y in zip(got[0], other):
            for a, b in zip(x, y):
                assert torch.equal(a, b)


def test_source_feeds_model_descriptor_indoor(tmp_path):
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    root = str(tmp_path)
    _device_tree(root)
    opt = _sopt()
    det = _detector(opt)
    src = sdl.SceneNNDescriptorPairSource(root, "train+val", opt, det, dev(), seed=2)
    assert len(src) == 3 and sorted(src.kinds.tolist()) == [1, 1, 2, 2, 2, 2]
    torch.manual_seed(3)
    md = ModelDescriptorIndoor(opt)
    losses, first = [], None
    for epoch in range(2):
        for out in src.feed(md):
            assert [tuple(t.shape) for t in out[8:]] == [(2, 3, 3), (2,), (2, 3, 1)]
            c = src.last["clouds"]
            (kp_a, kp_p), (sg_a, sg_p) = det.run_model_siamese((c[0], c[3]), (c[1], c[4]), (c[2], c[5]))
            for got, ref in zip((out[2], out[6], out[3], out[7]), (kp_a, kp_p, sg_a, sg_p)):
                assert torch.equal(got, ref)                        # same keypoints as on the default stream
            if first is None:
                first = [t.clone() for t in out]
                torch.cuda.manual_seed(11)
            np.random.seed(len(losses))
            md.optimize(epoch=epoch)
            losses.append(float(md.loss.detach()))
    assert len(losses) == 6 and all(math.isfinite(v) for v in losses)
    torch.manual_seed(3)
    md2 = ModelDescriptorIndoor(opt)
    md2.set_input(*first)
    torch.cuda.manual_seed(11)
    np.random.seed(0)
    md2.optimize(epoch=0)
    assert float(md2.loss.detach()) == losses[0], (float(md2.loss.detach()), losses[0])  # the hand-over changes nothing
    test = sdl.SceneNNDescriptorPairSource(root, "test", opt, det, dev(), seed=2, drop_last=False)
    assert len(test) == 2 and test.kinds.tolist() == [0, 0, 0]
    for _ in test.feed(md):
        md.test_model()
        assert math.isfinite(float(md.loss))
