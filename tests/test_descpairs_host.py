"""Host side of the descriptor pair builder (usip_b200.data.kitti_descriptor_loader), no GPU: the positive search, the
parity mode's numpy draw order and negative mining against the reference loader's batches in
tests/golden/descriptor_pairs.npz, argument checks, and ModelDescriptor's prefetch hand-over."""
import contextlib
import os
import random
import types

import numpy as np
import pytest
import torch

from usip_b200.data import kitti_descriptor_loader as kdesc
from usip_b200.data import kitti_detector_loader as kdl

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "descriptor_pairs.npz")


def golden_cases():
    g = np.load(GOLDEN)
    return g, sorted({k.split("/")[0] for k in g.files if k.endswith("/case")})


def case_opt(g, name):
    seed, S, rh, r3, rp, tp = (int(v) for v in g[name + "/case"])
    anchors = [int(a) for a in g[name + "/anchors"]]
    opt = types.SimpleNamespace(input_pc_num=int(g["N"]), node_num=int(g["M"]), surface_normal_len=S,
                                rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                translation_perturbation=bool(tp), positive_radius_threshold=5.0,
                                negative_radius_threshold=50.0, batch_size=len(anchors))
    return opt, str(g[name + "/mode"]), anchors, seed


def make_tree(g, root):
    counts = [int(c) for c in g["tree/counts"]]
    flat = g["tree/poses"]
    acc = np.concatenate([[0], np.cumsum(counts)])
    poses = [flat[acc[s]:acc[s + 1]] for s in range(len(counts))]
    kdl.write_synthetic_kitti(str(root), counts, int(g["tree/Ns"]), seed=int(g["tree/seed"]), poses=poses)


def replay(g, name, root):
    """The host draws of one golden batch, in the reference's order -> (positives, neg_idx, seq, poses)."""
    opt, mode, anchors, seed = case_opt(g, name)
    _, _, nums, accs = kdl.make_dataset_kitti(str(root), mode)
    seq, poses = kdesc.load_kitti_poses(str(root), mode)
    N, M, S = opt.input_pc_num, opt.node_num, opt.surface_normal_len
    np.random.seed(seed)
    random.seed(seed)
    pos = []
    for a in anchors:                                        # KittiDescriptorLoader.__getitem__
        kdl.draw_subsample(np.random, int(g["tree/Ns"]), N, kdesc.DESC_DIVISOR)
        pos.append(kdesc.nearby_index(a, poses, accs, nums, opt.positive_radius_threshold, random))
        kdl.draw_subsample(np.random, int(g["tree/Ns"]), N, kdesc.DESC_DIVISOR)
        kdesc.draw_desc_pair_scalars(np.random, mode == "train", N, M, S, True)
    neg = kdesc.mine_negative_sample(seq[anchors], poses[anchors].astype(np.float32), opt.negative_radius_threshold)
    return pos, neg, seq, poses


def test_positive_search_and_mining_replay_the_reference(tmp_path):
    g, names = golden_cases()
    assert len(names) == 5
    make_tree(g, tmp_path)
    no_negative = 0
    for name in names:
        with pytest.warns(UserWarning) if name == "s5" else contextlib.nullcontext() as w:
            pos, neg, seq, poses = replay(g, name, tmp_path)
        if name == "s5":
            no_negative = sum("no negative" in str(x.message) for x in w)
        np.testing.assert_array_equal(seq[pos], g[name + "/pos_seq"], err_msg=name)
        np.testing.assert_array_equal(poses[pos].astype(np.float32), g[name + "/pos_pose"], err_msg=name)
        np.testing.assert_array_equal(neg.numpy(), g[name + "/neg_idx"], err_msg=name)
        _, _, anchors, _ = case_opt(g, name)
        np.testing.assert_array_equal(poses[anchors].astype(np.float32), g[name + "/anc_pose"], err_msg=name)
    assert no_negative == 2
    # the batches do exercise the search: positives other than the anchor itself, in the anchor's sequence
    assert sum(int((g[n + "/pos_pose"] != g[n + "/anc_pose"]).any(axis=(1, 2)).sum()) for n in names) >= 10


def test_nearby_index_stays_in_the_sequence_and_radius():
    poses = np.tile(np.eye(4), (30, 1, 1))
    poses[:, 0, 3] = 100.0 * np.arange(30)                   # no other scan within reach: the anchor itself
    rng = random.Random(0)
    assert kdesc.nearby_index(7, poses, [30], [30], 5.0, rng) == 7
    poses[:, 0, 3] = 0.5 * np.arange(30)
    got = {kdesc.nearby_index(20, poses, [10, 30], [10, 20], 5.0, rng) for _ in range(200)}
    assert got <= set(range(10, 30)) and min(got) >= 11 and len(got) > 5


def _opt(**kw):
    o = types.SimpleNamespace(input_pc_num=1024, node_num=64, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                              rot_perturbation=False, translation_perturbation=False, batch_size=2)
    o.__dict__.update(kw)
    return o


def test_builder_argument_validation():
    b = kdesc.DescriptorPairBuilder(_opt(), device="cpu")
    scans = torch.zeros((4000, 8))
    off = np.array([0, 1500, 1500, 2000, 4000], np.int64)
    with pytest.raises(ValueError, match="no scans"):
        b.build(scans, np.array([0], np.int64), [0], [0])
    with pytest.raises(ValueError, match="no points"):
        b.build(scans, off, [0], [1])
    with pytest.raises(ValueError, match="500 rows"):                 # shorter than input_pc_num
        b.build(scans, off, [0], [2])
    with pytest.raises(IndexError):
        b.build(scans, off, [0], [4])
    with pytest.raises(ValueError, match="positives"):
        b.build(scans, off, [0, 3], [3])
    with pytest.raises(ValueError, match="columns"):
        kdesc.DescriptorPairBuilder(_opt(surface_normal_len=5), device="cpu").build(torch.zeros((4000, 7)), off, [0],
                                                                                    [3])
    with pytest.raises(ValueError, match="8192"):
        kdesc.DescriptorPairBuilder(_opt(input_pc_num=4 * 8193), device="cpu")
    with pytest.raises(ValueError, match="node_num"):
        kdesc.DescriptorPairBuilder(_opt(input_pc_num=200, node_num=64), device="cpu")
    with pytest.raises(ValueError):
        kdesc.DescriptorPairBuilder(_opt(), device="cpu", rng="python")


def test_set_input_after_prefetch_never_synchronises(monkeypatch):
    """The staged tensors are adopted with a stream-side wait; a plain set_input() still synchronises."""
    from usip_b200.models.keypoint_descriptor import ModelDescriptor

    class _Stream:
        waited = []

        def __init__(self, *a, **k):
            pass

        def wait_event(self, ev):
            _Stream.waited.append(ev)

    class _Event:
        def record(self, stream=None):
            pass

    def _no_sync(*a, **k):
        raise AssertionError("torch.cuda.synchronize called")

    monkeypatch.setattr(torch.cuda, "Stream", _Stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _Stream())
    monkeypatch.setattr(torch.cuda, "synchronize", _no_sync)
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, s: None)
    md = ModelDescriptor.__new__(ModelDescriptor)
    md.opt = types.SimpleNamespace(device=torch.device("cpu"))
    B, N, M = 2, 16, 4
    args = (torch.rand(B, 3, N), torch.rand(B, 4, N), torch.rand(B, 3, M), torch.rand(B, M), torch.rand(B, 3, N),
            torch.rand(B, 4, N), torch.rand(B, 3, M), torch.rand(B, M), torch.tensor([1, 0]))
    done = _Event()
    md.prefetch_input(*args, after=done)
    assert _Stream.waited[-1] is done
    md.set_input(*args)
    for k, a in zip(ModelDescriptor._INPUT_FIELDS, args):
        assert torch.equal(getattr(md, k), a), k
    assert md.neg_idx.dtype == torch.int64 and md.anc_pc.dtype == torch.float32
    with pytest.raises(AssertionError, match="synchronize"):          # no prefetch: the reference's behaviour
        md.set_input(*args)
