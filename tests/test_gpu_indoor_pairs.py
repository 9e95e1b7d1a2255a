"""Indoor pair builders on the GPU (csrc/pairgen.cu usip_indoor_pair_augment, usip_b200.data.match3d_detector_loader
and scenenn_detector_loader).

Parity mode (the builder replays numpy's draws) against the reference loaders' own batches in
tests/golden/indoor_pairs.npz; device mode against the Philox restatement of tests/pairgen_ref.py with the indoor laws
(the bracket rule of test_gpu_pairgen_streams.py); determinism, the laws, the per-pair augmentation switch, fragments
longer than the one-CTA subsample kernel, the three residencies; end to end through both sources into
ModelDetector.optimize()."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import pairgen_ref as ref
from tests.test_gpu_pairgen import _clipped_std, _ulps
from tests.test_gpu_pairgen_streams import CORNERS, _bracket, _case, _d, _nan
from tests.test_indoor_pairs_host import case_items, case_names, case_opt, golden, make_trees
from tests.util_gpu import dev, load_params, make_opt
from usip_b200 import _lib, ops
from usip_b200.data import kitti_detector_loader as kdl
from usip_b200.data import match3d_detector_loader as m3l
from usip_b200.data import scenenn_detector_loader as snl
from usip_b200.ops import _p, _stream, check

pytestmark = pytest.mark.gpu
KEYS = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
T, H, D3, PERT, TR = (ops.PAIR_TRAIN, ops.PAIR_ROT_HORIZONTAL, ops.PAIR_ROT_3D, ops.PAIR_ROT_PERTURBATION,
                      ops.PAIR_TRANSLATION)
LAW = (0.01, 0.02)                               # match3d_detector_loader.py:125-132, pc, sn and node


# ------------------------------------------------------------------------------------------- the indoor restatement
def indoor_jitter(seed, step, n_clouds, N, M, S, ulps=0):
    """Device-mode jitter of usip_indoor_pair_augment in upload layout, (2B, N, 3), (2B, N, S), (2B, M, 3): the keys of
    pairgen_ref.kitti_jitter (cloud, point, purpose; sn block q from sub q / 4) with sigma 0.01, clip 0.02 for all."""
    u = np.broadcast_to(np.asarray(ulps, np.int64), (4,))
    pc = np.stack([ref.jitter_xyz(seed, step, c, N, ref.PURPOSE_JIT_PC, LAW, ulps) for c in range(n_clouds)])
    sn = np.stack([np.concatenate([ref.clip(LAW[0] * ref.normals(seed, step, c, np.arange(N), ref.PURPOSE_JIT_SN,
                                                                 q // 4, u), LAW[1]) for q in range(0, S, 4)],
                                  axis=1)[:, :S] for c in range(n_clouds)])
    nd = np.stack([ref.jitter_xyz(seed, step, c, M, ref.PURPOSE_JIT_NODE, LAW, ulps) for c in range(n_clouds)])
    return pc, sn, nd


def indoor_pair_augment(scans, offsets, scan_of_cloud, rows, nodes, params, S, flags, jit_pc, jit_sn, jit_node):
    """pair_augment_kernel with usip_indoor_pair_augment's arguments: pairgen_ref.pair_augment with sn = columns 3:3+S
    (its S = 1 column is the last, so the scans are cut to 4 columns) and pair b augmented only where
    params[b, 45] != 0."""
    cut = scans[:, :4] if S == 1 else scans
    args = (cut, offsets, scan_of_cloud, rows, nodes, params, S)
    on = ref.pair_augment(*args, flags, jit_pc, jit_sn, jit_node)
    off = ref.pair_augment(*args, flags & ~T)
    keep = params[:, ops.PAIR_AUGMENT_SLOT] != 0
    if not flags & T:
        return off
    return tuple(np.where(keep.reshape((-1,) + (1,) * (a.ndim - 1)), a, b) for a, b in zip(on, off))


def _run(cs, jit=None, seed=None, step=None):
    """One usip_indoor_pair_augment call with NaN-filled outputs -> numpy outputs."""
    B, N, M, S = cs["B"], cs["N"], cs["M"], cs["S"]
    ins = [_d(cs[k]) for k in ("scans", "off", "soc", "rows", "nodes", "params")]
    jt = [None if j is None else _d(j) for j in (jit or (None, None, None))]
    outs = [_nan(B, 3, N), _nan(B, S, N), _nan(B, 3, M), _nan(B, 3, N), _nan(B, S, N), _nan(B, 3, M), _nan(B, 3, 3),
            _nan(B), _nan(B, 3, 1)]
    seed = cs["seed"] if seed is None else seed
    step = cs["step"] if step is None else step
    rc = _lib.load().usip_indoor_pair_augment(
        _p(ins[0]), cs["scans"].shape[1], *[_p(t) for t in ins[1:]], *[_p(t) for t in jt],
        ctypes.c_uint64(seed & (2 ** 64 - 1)), ctypes.c_uint64(step & (2 ** 64 - 1)), int(cs["flags"]), S, B, N, M,
        *[_p(t) for t in outs], _stream())
    check(rc, "indoor")
    return [o.cpu().numpy() for o in outs]


# ------------------------------------------------------------------------------------------------ parity mode
def test_parity_mode_reproduces_the_reference_loaders(tmp_path):
    g = golden()
    m3_root, sn_root = make_trees(g, tmp_path)
    same = total = 0
    for name in case_names(g, ""):
        opt, seed = case_opt(g, name)
        mode, divisor, paths, aug = case_items(g, name, m3_root, sn_root)
        arrs = [kdl.load_scan_npy(p, opt.surface_normal_len) for p in paths]
        off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
        scans = torch.from_numpy(np.concatenate(arrs)).to(dev())
        b = m3l.IndoorPairBuilder(opt, mode, dev(), rng="numpy", divisor=divisor)
        np.random.seed(seed)
        out = b.build(scans, off, np.arange(len(arrs)), augment=aug)
        for k, t in zip(KEYS, out):
            got, want = t.cpu().numpy(), g[name + "/" + k]
            got = got.reshape(want.shape)
            if k in ("R", "scale", "shift"):
                np.testing.assert_array_equal(got, want, err_msg=name + "/" + k)
            if k.startswith("src"):              # an un-augmented pair's src is the gathered rows themselves
                for i in np.nonzero(~np.array(aug) | (mode == "test"))[0]:
                    np.testing.assert_array_equal(got[i], want[i], err_msg=name + "/" + k)
            u = _ulps(got, want)
            assert u.max() <= 2, (name, k, int(u.max()), float(np.abs(got - want).max()))
            same += int((u == 0).sum()); total += u.size
    frac = same / total
    print("indoor pairgen parity: %.4f of %d coordinates bit-identical" % (frac, total))
    assert frac >= 0.99


# ------------------------------------------------------------------------------------ device mode vs restatement
CASES = [  # (S, C, flags, N, M, augment pattern of the pairs, extra)
    (1, 4, T, 1, 1, [1, 1], {}),
    (1, 7, T | H, 257, 300, [1, 0], {}),
    (4, 7, T | D3, 16384, 512, [1, 1], {"seed": 2 ** 32 + 5}),
    (3, 7, T | H | PERT | TR, 255, 64, [0, 1, 1], {"n_pairs": 3, "step": 2 ** 32 + 7}),
    (5, 8, T | D3 | PERT | TR, 257, 300, [1, 0, 1], {"n_pairs": 3, "step": 0}),
    (8, 11, T | H | TR, 255, 64, [1] * 9 + [0] * 8, {"n_pairs": 17, "seed": 2 ** 40 + 3}),
    (4, 7, T | D3, 4096, 64, [1, 1], {"zero": True}),
    (4, 7, D3, 257, 64, [1, 0], {}),                           # test mode: the switch does not matter
]


@pytest.mark.parametrize("c", CASES, ids=lambda c: "S%d-C%d-f%d-N%d-M%d-a%s%s" % (
    c[0], c[1], c[2], c[3], c[4], "".join(map(str, c[5])), "".join("-%s%s" % kv for kv in sorted(c[6].items()))))
def test_device_jitter_equals_restated_upload(c):
    S, C, flags, N, M, aug, extra = c
    cs = _case("det", N, M, S, C, flags, **extra)
    cs["params"][:, ops.PAIR_AUGMENT_SLOT] = aug
    got = _run(cs)
    jit = lambda u: indoor_jitter(cs["seed"], cs["step"], 2 * cs["B"], N, M, S, u)
    nominal_jit = jit(0)
    nominal = _run(cs, nominal_jit)
    runs = [_run(cs, jit(u)) for u in CORNERS] + [nominal]
    n = nb = 0
    for k, gk in enumerate(got):
        a, b = _bracket(gk, [r[k] for r in runs], "indoor output %d" % k)
        n += a; nb += b
    print("indoor device vs upload: %d elements, %d non-empty brackets" % (n, nb))
    want = indoor_pair_augment(*[cs[k] for k in ("scans", "off", "soc", "rows", "nodes", "params")], S, flags,
                               *nominal_jit)
    for k, (gk, w) in enumerate(zip(nominal, want)):
        assert _ulps(gk, w.reshape(gk.shape)).max() <= 1, ("upload vs restatement", k)
    if flags & T:                                 # un-augmented pairs: the gather, then the dst transform, bit for bit
        for b in np.nonzero(np.array(aug) == 0)[0]:
            test_mode = _run(dict(cs, flags=flags & ~T))
            for k in range(6):
                np.testing.assert_array_equal(got[k][b], test_mode[k][b])


# --------------------------------------------------------------------------------------------- device builders
def _iopt(**kw):
    base = dict(input_pc_num=10240, node_num=512, surface_normal_len=4, node_knn_k_1=32, rot_horizontal=False,
                rot_3d=True, rot_perturbation=False, translation_perturbation=False, scene="indoor",
                loss_sigma_lower_bound=1e-4, keypoint_on_pc_alpha=10.0, batch_size=2)
    base.update(kw)
    return make_opt(**base)


def _fragments(ns, seed=0):
    from usip_b200.evaluation.indoor_test_loader import synthetic_fragment
    arrs = [synthetic_fragment(seed + i, n) for i, n in enumerate(ns)]
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return torch.from_numpy(np.concatenate(arrs)).to(dev()), off, arrs


def test_device_mode_is_deterministic_per_step():
    scans, off, _ = _fragments([30000, 8000, 12000])
    b = m3l.IndoorPairBuilder(_iopt(input_pc_num=4096, node_num=128, rot_perturbation=True,
                                    translation_perturbation=True), "train", dev(), seed=5)
    a1 = [t.clone() for t in b.build(scans, off, [0, 2, 1], step=7, augment=[True, False, True])]
    a2 = b.build(scans, off, [0, 2, 1], step=7, augment=[True, False, True])
    a3 = b.build(scans, off, [0, 2, 1], step=8, augment=[True, False, True])
    for x, y in zip(a1, a2):
        assert torch.equal(x, y)
    assert not torch.equal(a1[0], a3[0]) and not torch.equal(a1[6], a3[6])
    R = a1[6].double()
    eye = torch.eye(3, dtype=torch.float64, device=R.device)
    assert float((R @ R.transpose(1, 2) - eye).abs().max()) < 1e-6
    assert float((a1[7] - 1).abs().max()) <= 0.1 and float(a1[8].abs().max()) <= 0.5


def test_device_jitter_laws():
    """Identity params, rows and nodes taken in order: src - input is the jitter itself, clipped at 0.02, with the
    clipped standard deviation of N(0, 0.01^2), for pc, every sn column and nodes."""
    N, M, S, B = 16384, 2048, 4, 2
    pc = np.random.RandomState(0).uniform(-2, 2, (N, 7)).astype(np.float32)
    scans = torch.from_numpy(pc).to(dev())
    off = torch.tensor([0, N], dtype=torch.int64, device=dev())
    soc = torch.zeros(2 * B, dtype=torch.int32, device=dev())
    rows = torch.arange(N, dtype=torch.int32, device=dev()).repeat(2 * B, 1).contiguous()
    nodes = torch.from_numpy(np.ascontiguousarray(pc[:M, :3].T)).to(dev()).repeat(2 * B, 1, 1).contiguous()
    params = np.zeros((B, ops.PAIR_PARAM_STRIDE))
    params[:, 27] = 1.0
    params[:, 31:40] = np.eye(3).ravel()
    params[:, 43] = 1.0
    params[:, ops.PAIR_AUGMENT_SLOT] = 1.0
    out = ops.indoor_pair_augment(scans, off, soc, rows, nodes, torch.from_numpy(params).to(dev()), S, T, seed=9,
                                  step=2)
    o = [t.cpu().numpy().astype(np.float64) for t in out]
    sd = _clipped_std(*LAW)
    for j in (o[0] - pc[:, 0:3].T, o[1] - pc[:, 3:3 + S].T, o[2] - pc[:M, 0:3].T,
              o[3] - pc[:, 0:3].T, o[4] - pc[:, 3:3 + S].T, o[5] - pc[:M, 0:3].T):
        assert np.abs(j).max() <= LAW[1] * (1 + 1e-4)
        assert (np.abs(j) >= LAW[1] * (1 - 1e-4)).any()         # some draws are clipped
        n = j.size
        assert abs(j.mean()) < 5 * sd / math.sqrt(n) + 1e-7
        assert abs(j.std() / sd - 1) < 6 / math.sqrt(2 * n) + 1e-3, (j.std(), sd)
    assert np.abs((o[0] - pc[:, 0:3].T) - (o[3] - pc[:, 0:3].T)).max() > LAW[0]   # every cloud draws its own


def test_per_pair_switch_in_a_mixed_batch():
    scans, off, arrs = _fragments([20000, 15000], seed=30)
    opt = _iopt(input_pc_num=4096, node_num=128, translation_perturbation=True)
    b = m3l.IndoorPairBuilder(opt, "train", dev(), seed=4, divisor=snl.SCENENN_DIVISOR)
    mixed = [t.clone() for t in b.build(scans, off, [0, 1], step=3, augment=[True, False])]
    last = b.last
    both = b.build(scans, off, [0, 1], step=3, augment=[True, True])
    for k in range(9):                            # the augmented pair does not depend on its neighbour
        assert torch.equal(mixed[k][0], both[k][0]), KEYS[k]
    assert not torch.equal(mixed[0][1], both[0][1])
    rows = last["rows"].cpu().numpy()
    _, nodes = ops.fps(last["candidates"], last["start"], opt.node_num, want_nodes=True)
    a = arrs[1]
    np.testing.assert_array_equal(mixed[0][1].cpu().numpy(), a[rows[2], 0:3].T)
    np.testing.assert_array_equal(mixed[1][1].cpu().numpy(), a[rows[2], 3:7].T)
    assert torch.equal(mixed[2][1], nodes[2])
    P = last["params"].cpu().numpy()[1]
    assert P[ops.PAIR_AUGMENT_SLOT] == 0 and last["params"].cpu().numpy()[0, ops.PAIR_AUGMENT_SLOT] == 1
    src = np.ascontiguousarray(a[rows[3], 0:3])
    want = ref._dst_transform(P, src)
    assert _ulps(mixed[3][1].cpu().numpy(), want.T).max() <= 1
    want_nd = ref._dst_transform(P, np.ascontiguousarray(nodes[3].cpu().numpy().T))
    assert _ulps(mixed[5][1].cpu().numpy(), want_nd.T).max() <= 1
    # the un-augmented pair equals a test-mode build of the same rows and params
    soc = torch.tensor([0, 0, 1, 1], dtype=torch.int32, device=dev())
    test = ops.indoor_pair_augment(scans, torch.from_numpy(off).to(dev()), soc, last["rows"], nodes, last["params"], 4,
                                   b.flags & ~T)
    for k in range(9):
        assert torch.equal(test[k][1], mixed[k][1]), KEYS[k]


def test_long_fragments_build_through_the_cluster_kernel():
    """A 250,000-row fragment (above the one-CTA kernel's limit) and a 20,000-row one build, and their rows are
    ops.cloud_subsample's on the same inputs."""
    assert 250000 > ops.pair_max_scan_rows()
    scans, off, _ = _fragments([250000, 20000], seed=50)
    opt = _iopt()
    b = m3l.IndoorPairBuilder(opt, "train", dev(), seed=6)
    out = b.build(scans, off, [0, 1], step=11)
    assert all(bool(torch.isfinite(t).all()) for t in out)
    soc = torch.tensor([0, 0, 1, 1], dtype=torch.int32, device=dev())
    rows, cand, start, _ = ops.cloud_subsample(scans, torch.from_numpy(off).to(dev()), soc, 250000, opt.input_pc_num,
                                               opt.input_pc_num // 10, None, 6, 11)
    assert torch.equal(rows, b.last["rows"]) and torch.equal(cand, b.last["cand"])
    assert torch.equal(start, b.last["start"])
    r = rows.cpu().numpy()
    assert (np.diff(r, axis=1) > 0).all() and r[:2].max() < 250000 and r[2:].max() < 20000


def _m3_tree(root, n_files=5, rows=30000, seed=0):
    layout = {"train": {"kitchen": {"seq-01": n_files - 2, "seq-02": 2}}}
    m3l.write_synthetic_3dmatch_train(str(root), layout, rows, seed=seed)


def test_disk_host_and_device_residency_give_the_same_batches(tmp_path):
    _m3_tree(tmp_path, rows=lambda i: 60000 if i == 1 else 9000 + 1000 * i)
    opt = _iopt(input_pc_num=4096, node_num=128, batch_size=2)
    got = {}
    for resident in ("disk", "host", "device"):
        src = m3l.Match3DPairSource(str(tmp_path), "train", opt, dev(), seed=3, resident=resident)
        got[resident] = [[t.clone() for t in out] for out, ev in src.batches()]
        assert (src.scans is None) == (resident == "disk")
    assert len(got["disk"]) == 2
    for resident in ("host", "device"):
        for x, y in zip(got["disk"], got[resident]):
            for k in range(9):
                assert torch.equal(x[k], y[k]), (resident, KEYS[k])


def _model(opt):
    from oracle import usip_oracle as orc
    from usip_b200.models.keypoint_detector import ModelDetector
    md = ModelDetector(opt)
    load_params(md.detector, orc.init_detector_params(S=opt.surface_normal_len, seed=1, C1=64, C2=256,   # indoor
                                                      randomize_bn=True))
    return md


def test_sources_feed_optimize(tmp_path):
    _m3_tree(tmp_path / "m3", rows=lambda i: 1500 if i == 0 else 12000)       # file 0 takes the tile path
    snl.write_synthetic_scenenn(str(tmp_path / "sn"), {"train": 3, "val": 2}, lambda s, i: 9000, seed=4)
    opt = _iopt(input_pc_num=2048, node_num=64, node_knn_k_1=16, batch_size=2)
    for src in (m3l.Match3DPairSource(str(tmp_path / "m3"), "train", opt, dev(), seed=1, resident="disk"),
                snl.SceneNNPairSource(str(tmp_path / "sn"), "train+val", opt, dev(), seed=1)):
        md = _model(opt)
        losses = []
        for _ in src.feed(md):
            md.optimize(epoch=0)
            losses.append(float(md.loss))
        assert len(losses) == len(src) == 2 and all(math.isfinite(v) for v in losses)
    assert src.augment_mask.tolist() == [True] * 3 + [False] * 2


def test_full_3dmatch_shape_step(tmp_path):
    """match3d/options_detector.py defaults: B = 2, N = 10240, M = 512, S = 4, node_knn_k_1 = 32, rot_3d."""
    _m3_tree(tmp_path, n_files=4, rows=lambda i: 250000 if i == 0 else 40000)
    opt = _iopt()
    src = m3l.Match3DPairSource(str(tmp_path), "train", opt, dev(), seed=2)
    md = _model(opt)
    n = 0
    for _ in src.feed(md):
        md.optimize(epoch=0)
        assert math.isfinite(float(md.loss))
        n += 1
    assert n == 2


def test_graph_and_eager_train_steps_agree_on_a_built_batch():
    scans, off, _ = _fragments([40000, 7000], seed=80)
    opt = _iopt(input_pc_num=2048, node_num=64, node_knn_k_1=16, batch_size=2)
    batch = m3l.IndoorPairBuilder(opt, "train", dev(), seed=5, divisor=snl.SCENENN_DIVISOR).build(
        scans, off, [0, 1], step=0, augment=[True, False])
    losses = {}
    for graph in (False, True):
        md = _model(opt)
        md.use_cuda_graph = graph
        ls = []
        for _ in range(2):
            md.set_input(*batch)
            md.optimize(epoch=0)
            ls.append(float(md.loss))
        losses[graph] = ls
    for x, y in zip(losses[False], losses[True]):
        assert abs(x - y) <= 5e-4 * abs(x), losses
