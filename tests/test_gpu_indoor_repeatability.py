"""Repeatability on the rotated ModelNet40, Redwood and 3DMatch test sets on the GPU (usip_b200.evaluation
.modelnet_test_loader / indoor_test_loader / repeatability).

The test clouds in parity mode against the reference loaders' own batches (tests/golden/{modelnet,redwood,3dmatch}
_test_clouds.npz), bit for bit, with and without noise; device mode's determinism, Redwood's tiling of short scans, the
surface-normal columns and the FPS nodes; and each evaluator end to end against the float64 restatement of eval_rep.m
(tests/rep_ref.py) run on the keypoint files it writes, including a 3DMatch fragment longer than the one-CTA subsample
kernel takes."""
import os

import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests.rep_ref import pair_counts
from tests.test_indoor_repeatability_host import _parity_source, match3d_tree, modelnet_tree, redwood_tree
from tests.util_gpu import load_params, make_opt
from usip_b200 import ops
from usip_b200.evaluation import indoor_test_loader as itl
from usip_b200.evaluation import modelnet_test_loader as mtl
from usip_b200.evaluation import repeatability as rep
from usip_b200.evaluation.save_keypoints import read_keypoints_bin

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["modelnet", "redwood", "3dmatch"])
def test_parity_mode_matches_reference_loader(name, tmp_path):
    g, src = _parity_source(name, str(tmp_path))
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


def _device_source(name, root):
    if name == "modelnet":
        tree, _ = modelnet_tree(root, k=3, rows=1500)
        return mtl.ModelNetRotatedTestLoader(tree, make_opt(input_pc_num=1024, node_num=64, surface_normal_len=3),
                                             batch_size=3, n=3)
    if name == "redwood":
        return itl.RedwoodTestLoader(redwood_tree(root)[0], make_opt(input_pc_num=64, node_num=8), batch_size=3)
    return itl.Match3DTestLoader(match3d_tree(root), make_opt(input_pc_num=1024, node_num=64), batch_size=3)


@pytest.mark.parametrize("name", ["modelnet", "redwood", "3dmatch"])
def test_device_mode(name, tmp_path):
    src = _device_source(name, str(tmp_path))
    items = [0, 1, 2] if name != "redwood" else [0, 1, 4]          # Redwood frames of 5, 42 and 77 rows
    a = src.build(items, noise_sigma=0.1, step=5)
    last = {k: v.cpu().numpy() for k, v in src.last.items()}
    b = src.build(items, noise_sigma=0.1, step=5)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    plain = src.build(items, step=5)
    assert torch.equal(plain[1], a[1]) and torch.equal(plain[2], a[2]) and not torch.equal(plain[0], a[0])
    assert plain[1].shape[1] == (3 if name == "modelnet" else 4)
    scans = src.load(items)
    for c in range(3):
        rows, n = last["rows"][c], len(scans[c])
        if n >= src.N:
            assert len(np.unique(rows)) == len(rows) and rows.max() < n
        else:                                        # every row t times, ascending, then an ascending remainder
            t = max(1, -(-src.N // n) - 1)
            np.testing.assert_array_equal(rows[:t * n], np.tile(np.arange(n), t))
            rest = rows[t * n:]
            assert len(np.unique(rest)) == len(rest) == src.N - t * n and (np.diff(rest) > 0).all()
        pts = last["candidates"][c]
        np.testing.assert_array_equal(pts, scans[c][rows[last["cand"][c]], :3])
        node = plain[2][c].cpu().numpy().T
        assert {tuple(p) for p in node} <= {tuple(p) for p in pts}
        raw = scans[c][rows]
        np.testing.assert_array_equal(plain[0][c].cpu().numpy().T, raw[:, :3])
        np.testing.assert_array_equal(plain[1][c].cpu().numpy().T, raw[:, 3:3 + src.S])
    if name == "redwood":
        assert min(len(s) for s in scans) < src.N


def _model(N, M, B, S):
    from usip_b200.models.keypoint_detector import ModelDetector
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S)
    md = ModelDetector(opt)
    P = orc.init_detector_params(S=S, seed=21, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    load_params(md.detector, P)
    return md, opt


@pytest.mark.parametrize("name", ["modelnet", "redwood", "3dmatch"])
@pytest.mark.parametrize("nms_radius", [0.0, 0.3])
def test_end_to_end_against_keypoint_files(name, nms_radius, tmp_path):
    root = str(tmp_path)
    N, M, B = 1024, 64, 2
    md, opt = _model(N, M, B, 3 if name == "modelnet" else 4)
    if name == "modelnet":
        tree, _ = modelnet_tree(root, k=3, rows=1500)
        ev = rep.ModelNetRepeatability(tree, opt, seed=9, batch_size=B)
    elif name == "redwood":
        scenes = [("livingroom1", 4), ("office2", 3)]
        npy, gt = os.path.join(root, "npy"), os.path.join(root, "gt")
        itl.write_synthetic_redwood(npy, gt, lambda s, f: (300, 1500, 2000, 700)[f % 4],
                                    {"livingroom1": [(0, 1), (2, 2), (3, 0)], "office2": [(1, 2), (0, 1)]}, seed=4,
                                    scenes=scenes)
        ev = rep.RedwoodRepeatability(npy, gt, opt, seed=9, batch_size=B, scenes=scenes)
    else:
        scenes = itl.MATCH3D_SCENES[:2]
        n_long = ops.pair_max_scan_rows() + 3000                      # the cluster kernel draws this batch's rows
        itl.write_synthetic_3dmatch(root, {scenes[0]: (0, 1, 2), scenes[1]: (0, 5)},
                                    lambda s, k: n_long if (s, k) == (0, 1) else 1500,
                                    {scenes[0]: [(0, 1), (1, 2), (2, 2)], scenes[1]: [(5, 0)]}, seed=5)
        ev = rep.Match3DRepeatability(root, opt, seed=9, batch_size=B, scenes=scenes)
        assert max(len(a) for a in ev.source.load(list(range(len(ev.source))))) > ops.pair_max_scan_rows()
    ks = [4, 16, 64]
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
    if name == "modelnet":
        assert sorted(os.listdir(out)) == ["original", "rotated"]
