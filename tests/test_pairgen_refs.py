"""The numpy restatement of csrc/pairgen.cu (tests/pairgen_ref.py) on the CPU: Philox's published known answers, the
Box-Muller edges, the uniqueness of the stream counters, and the restated per-point arithmetic against the reference
loaders' own batches.  The pair builders run here in parity mode with their device calls replaced by the restatement
(and FPS by the oracle's), so every golden batch is recomputed from the builders' host draws alone."""
import contextlib
import itertools
import os
import random

import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests import pairgen_ref as ref
from tests.philox_ref import pg_random, philox4x32_10
from usip_b200 import ops

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ulps(a, b):
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))


# ---------------------------------------------------------------------------------------------------- the stream
@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32_10."""
    got = philox4x32_10(*ctr, *key)
    assert tuple(int(x) for x in got) == want


def test_pg_random_is_philox_of_the_stated_counter():
    for seed, step, cloud, item, purpose, sub in [(0, 0, 0, 0, 3, 0), (2 ** 32 + 5, 2 ** 32 + 7, 65535, 2 ** 24 - 1, 4, 1),
                                                  (2 ** 64 - 1, 2 ** 48 - 1, 3, 17, 6, 0)]:
        c = ref.counter(seed, step, cloud, item, purpose, sub)
        want = [int(x) for x in philox4x32_10(*c)]
        got = [int(x[0]) for x in pg_random(seed, step, cloud, [item], purpose, sub)]
        assert got == want


def test_box_muller_edges():
    # a = 0xffffffff: u1 = 1, r = 0 exactly, whatever b is
    z0, z1 = ref.normal2(np.full(4, 0xffffffff, np.uint32), np.array([0, 1, 2 ** 30, 0xffffffff], np.uint32))
    assert np.all(z0 == 0) and np.all(z1 == 0)
    # a = 0: u1 = 2^-32, the largest radius, finite (u1 = a 2^-32 would take log(0))
    z0, z1 = ref.normal2(np.zeros(1, np.uint32), np.zeros(1, np.uint32))
    assert np.isfinite(z0).all() and z0[0] == np.sqrt(64 * np.log(2.0)) and z1[0] == 0
    # exact quadrants: b = k 2^30 puts 2 u2 on a multiple of 1/2, where sinpi / cospi are 0 or +-1 exactly
    r = np.sqrt(-2 * np.log(0.5))
    z0, z1 = ref.normal2(np.full(4, 2 ** 31 - 1, np.uint32), np.array([0, 2 ** 30, 2 ** 31, 3 * 2 ** 30], np.uint32))
    np.testing.assert_array_equal(z0, r * np.array([1, 0, -1, 0]))
    np.testing.assert_array_equal(z1, r * np.array([0, 1, 0, -1]))
    # and the reduction agrees with sin / cos of 2 pi u2 away from those points
    b = np.random.RandomState(0).randint(0, 2 ** 32, 10000, dtype=np.uint64).astype(np.uint32)
    z0, z1 = ref.normal2(np.full(b.shape, 2 ** 31 - 1, np.uint32), b)
    th = 2 * np.pi * b.astype(np.float64) * 2.0 ** -32
    np.testing.assert_allclose(z0, r * np.cos(th), rtol=0, atol=1e-9)
    np.testing.assert_allclose(z1, r * np.sin(th), rtol=0, atol=1e-9)


def test_counters_never_collide():
    """Two (purpose, sub, cloud or pair, item, step) tuples never share a counter for item < 2^24, cloud < 2^16 and
    step < 2^48: the counter words hold item, cloud, the step's low word and purpose | sub << 8 | step_hi << 16."""
    items = [0, 1, 2 ** 16, 2 ** 24 - 1]
    clouds = [0, 1, 2 ** 15, 2 ** 16 - 1]
    steps = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7, 2 ** 40, 2 ** 48 - 1]
    slots = [(p, 0) for p in range(7)] + [(ref.PURPOSE_JIT_SN, 1)]
    seen = {}
    for (p, sub), c, i, s in itertools.product(slots, clouds, items, steps):
        ctr = ref.counter(7, s, c, i, p, sub)[:4]
        assert ctr not in seen, ((p, sub, c, i, s), seen.get(ctr))
        seen[ctr] = (p, sub, c, i, s)
    # the counter is injective: every field reads back
    rng = np.random.RandomState(1)
    for _ in range(2000):
        p, sub = slots[rng.randint(len(slots))]
        c, i, s = rng.randint(2 ** 16), rng.randint(2 ** 24), int(rng.randint(2 ** 24)) << 24 | rng.randint(2 ** 24)
        c0, c1, c2, c3, _, _ = ref.counter(7, s, c, i, p, sub)
        assert (c0, c1, c2 | (c3 >> 16) << 32, c3 & 0xff, (c3 >> 8) & 0xff) == (i, c, s, p, sub)


def test_jitter_streams_are_keyed_as_stated():
    """Distinct keys give distinct draws: positions, clouds, purposes, sn blocks, steps and the seed's high word."""
    base = ref.normals(5, 3, 2, np.arange(64), ref.PURPOSE_JIT_PC)
    for other in (ref.normals(5, 3, 2, np.arange(1, 65), ref.PURPOSE_JIT_PC),
                  ref.normals(5, 3, 3, np.arange(64), ref.PURPOSE_JIT_PC),
                  ref.normals(5, 3, 2, np.arange(64), ref.PURPOSE_JIT_NODE),
                  ref.normals(5, 3, 2, np.arange(64), ref.PURPOSE_JIT_PC, 1),
                  ref.normals(5, 3 + 2 ** 32, 2, np.arange(64), ref.PURPOSE_JIT_PC),
                  ref.normals(5 + 2 ** 32, 3, 2, np.arange(64), ref.PURPOSE_JIT_PC)):
        assert not np.any(other == base)
    sn = ref.jitter_sn(5, 3, 2, 64, 8)
    assert not np.any(sn[:, 0:4] == sn[:, 4:8])
    assert np.abs(ref.jitter_xyz(5, 3, 2, 8192, ref.PURPOSE_JIT_PC, ref.PC_LAW)).max() == 0.12   # clipped: exactly


def test_ulp_shift():
    v = np.array([0.0, -0.0, 1.0, -1.0, 5e-324, np.inf * 0 + 3.5])
    for k in (-8, -1, 1, 8):
        w = v.copy()
        for _ in range(abs(k)):
            w = np.nextafter(w, np.sign(k) * np.inf)
        got = ref.ulp_shift(v, k)
        np.testing.assert_array_equal(got, w)


# ------------------------------------------------------------------------------- the arithmetic against goldens
def _t(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else a


def _wrap(fn):
    """A device call restated: tensors in, numpy through the restatement, CPU tensors out."""
    def call(*args, **kw):
        out = fn(*[_t(a) for a in args], **{k: _t(v) for k, v in kw.items()})
        return tuple(torch.from_numpy(np.ascontiguousarray(o)) for o in out) if isinstance(out, tuple) \
            else torch.from_numpy(out)
    return call


def _fps(pts, start, k, want_nodes=True):
    pts, start = _t(pts), _t(start)
    idx = np.stack([orc.fps(pts[c], int(start[c]), k) for c in range(len(pts))])
    nodes = np.stack([pts[c][idx[c]].T for c in range(len(pts))])
    return torch.from_numpy(idx), torch.from_numpy(np.ascontiguousarray(nodes))


def _strip(fn, n_arrays):
    """ops.* signature (seed, step after flags) -> the restatement's (jitter only)."""
    def call(*args, **kw):
        args = list(args)
        seed_step_at = n_arrays
        del args[seed_step_at:seed_step_at + 2]
        kw.pop("seed", None), kw.pop("step", None)
        return fn(*args, **kw)
    return call


@pytest.fixture
def restated(monkeypatch):
    """The builders on the CPU: their device calls replaced by the restatement, FPS by the oracle."""
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(ops, "cloud_gather_candidates", _wrap(ref.gather_candidates))
    monkeypatch.setattr(ops, "fps", _fps)
    monkeypatch.setattr(ops, "pair_augment", _wrap(_strip(ref.pair_augment, 8)))
    monkeypatch.setattr(ops, "modelnet_pair_augment", _wrap(_strip(ref.modelnet_pair_augment, 7)))
    monkeypatch.setattr(ops, "desc_pair_augment", _wrap(_strip(ref.desc_pair_augment, 8)))

    def cloud_gather(scans, offsets, scan_of_cloud, rows, nodes, S, flags=0, noise_sigma=0.0, noise=None, seed=0,
                     step=0):
        return _wrap(ref.cloud_gather)(scans, offsets, scan_of_cloud, rows, nodes, S, flags, noise_sigma, noise)
    monkeypatch.setattr(ops, "test_cloud_gather", cloud_gather)
    monkeypatch.setattr(ops, "scale_channel_", lambda t, k, f: t.__setitem__(
        (slice(None), k), torch.from_numpy((t[:, k].numpy().astype(np.float64) * np.float32(f)).astype(np.float32)))
        or t)


def _check(got, want, what, worst):
    got = np.asarray(got).reshape(want.shape)
    u = _ulps(got, want)
    worst[0] = max(worst[0], int(u.max()))
    assert u.max() <= 1, (what, int(u.max()), float(np.abs(got.astype(np.float64) - want).max()))


KEYS = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
DESC_KEYS = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node")


def test_restated_detector_pairs_reproduce_the_golden(restated, tmp_path):
    from tests.test_pairgen_host import case_opt, golden_cases, make_tree
    from usip_b200.data import kitti_detector_loader as kdl
    g, names = golden_cases()
    make_tree(g, tmp_path)
    worst = [0]
    for name in names:
        opt, mode, index, seed = case_opt(g, name)
        pc = kdl.load_scan_npy(kdl.kitti_scan_path(str(tmp_path), mode, index), opt.surface_normal_len)
        b = kdl.DetectorPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        out = b.build(torch.from_numpy(pc), np.array([0, len(pc)], np.int64), [0])
        for k, t in zip(KEYS, out):
            _check(t[0].numpy(), g[name + "/" + k], name + "/" + k, worst)
    print("detector pairs: worst %d fp32 ulp from the golden" % worst[0])


def test_restated_modelnet_pairs_reproduce_the_golden(restated, tmp_path):
    from tests.test_modelnet_pairs_host import case_opt, golden_cases, make_tree, split_scans
    from usip_b200.data import modelnet_shrec_loader as mnl
    g, names = golden_cases()
    make_tree(g, tmp_path)
    worst = [0]
    for name in names:
        opt, mode, items, seed = case_opt(g, name)
        arrs, off = split_scans(tmp_path, mode, opt)
        b = mnl.ModelNetPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        out = b.build(torch.from_numpy(np.concatenate(arrs)), off, items)
        for k, t in zip(KEYS, out):
            _check(t.numpy(), g[name + "/" + k], name + "/" + k, worst)
    print("modelnet pairs: worst %d fp32 ulp from the golden" % worst[0])


def test_restated_descriptor_pairs_reproduce_the_golden(restated, tmp_path):
    from tests.test_descpairs_host import case_opt, golden_cases, make_tree
    from usip_b200.data import kitti_descriptor_loader as kdesc
    from usip_b200.data import kitti_detector_loader as kdl
    g, names = golden_cases()
    make_tree(g, tmp_path)
    worst = [0]
    for name in names:
        opt, mode, anchors, seed = case_opt(g, name)
        _, _, nums, accs = kdl.make_dataset_kitti(str(tmp_path), mode)
        arrs = [kdl.load_scan_npy(kdl.kitti_scan_path(str(tmp_path), mode, i), opt.surface_normal_len)
                for i in range(accs[-1])]
        off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
        _, poses = kdesc.load_kitti_poses(str(tmp_path), mode)
        b = kdesc.DescriptorPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        random.seed(seed)
        pos = [kdesc.nearby_index(a, poses, accs, nums, opt.positive_radius_threshold, random) for a in anchors]
        out = b.build(torch.from_numpy(np.concatenate(arrs)), off, anchors, pos)
        for k, t in zip(DESC_KEYS, out):
            _check(t.numpy(), g[name + "/" + k], name + "/" + k, worst)
    print("descriptor pairs: worst %d fp32 ulp from the golden" % worst[0])


def test_restated_oxford_pairs_reproduce_the_golden(restated, tmp_path):
    from tests.test_oxford_pairs_host import (GOLDEN_DESC, _parse, case_opt, desc_case_opt, golden_cases, item_scans,
                                              make_tree)
    from usip_b200.data import kitti_detector_loader as kdl
    from usip_b200.data import oxford_descriptor_loader as odesc
    from usip_b200.data import oxford_detector_loader as odet
    stack = lambda arrs: (torch.from_numpy(np.concatenate(arrs)),
                          np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64))
    g, names = golden_cases()
    make_tree(g, tmp_path)
    worst = [0]
    for name in names:
        opt, mode, index, seed = case_opt(g, name)
        scans, off = stack(item_scans(tmp_path, mode, odet.make_dataset_oxford_train if mode == "train"
                                      else odet.make_dataset_oxford_test))
        b = odet.OxfordPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        out = b.build(scans, off, [index])
        for k, t in zip(KEYS, out):
            _check(t[0].numpy(), g[name + "/" + k], "oxford " + name + "/" + k, worst)
    g, names = golden_cases(GOLDEN_DESC)
    for name in names:
        opt, mode, items, seed = desc_case_opt(g, name)
        ds = _parse(odesc.make_dataset_oxford_train if mode == "train" else odesc.make_dataset_oxford_test, tmp_path)
        if mode == "train":
            arrs = item_scans(tmp_path, mode, odesc.make_dataset_oxford_train)
            scan_of_item = scan_of_pos = lambda i: i
        else:
            numbers = sorted({d["anc_idx"] for d in ds} | {p for d in ds for p in d["pos_idx_list"]})
            arrs = [kdl.load_scan_npy(odet.oxford_test_path(str(tmp_path), n), 3) for n in numbers]
            scan_of_item, scan_of_pos = (lambda i: numbers.index(ds[i]["anc_idx"])), numbers.index
        scans, off = stack(arrs)
        b = odesc.OxfordDescriptorPairBuilder(opt, mode, "cpu", rng="numpy")
        np.random.seed(seed)
        random.seed(seed)
        pos = [odesc.pick_positive(ds, mode, i, random) for i in items]
        out = b.build(scans, off, [scan_of_item(i) for i in items], [scan_of_pos(p) for p in pos])
        for k, t in zip(DESC_KEYS, out):
            _check(t.numpy(), g[name + "/" + k], "oxford_desc " + name + "/" + k, worst)
    print("oxford pairs: worst %d fp32 ulp from the golden" % worst[0])


def test_restated_kitti_test_clouds_reproduce_the_golden(restated, tmp_path):
    from tests.test_repeatability_host import _kitti_tree
    from tests.util_gpu import make_opt
    from usip_b200.evaluation import kitti_test_loader as ktl
    g = np.load(os.path.join(GOLDEN, "kitti_test_clouds.npz"))
    txt, num, _ = _kitti_tree(str(tmp_path))
    src = ktl.KittiTestLoader(txt, num, make_opt(input_pc_num=int(g["N"]), node_num=int(g["M"])), device="cpu",
                              rng="numpy", batch_size=int(g["batch_size"]))
    worst = [0]
    for case in ("plain", "noise"):
        seed = int(g[case + "/case"][0])
        np.random.seed(seed)
        torch.manual_seed(seed)
        got = {"pc": [], "sn": [], "node": []}
        for _, out in src.batches(float(g[case + "/noise_sigma"])):
            for k, v in zip(("pc", "sn", "node"), out):
                got[k].append(v.numpy())
        for k in got:
            _check(np.concatenate(got[k]), g[case + "/" + k], case + "/" + k, worst)
    print("kitti test clouds: worst %d fp32 ulp from the golden" % worst[0])
