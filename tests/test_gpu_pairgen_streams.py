"""The pair builders' device-mode random streams (csrc/pairgen.cu) pinned to the Philox restatement in
tests/pairgen_ref.py, and the augmentation kernels' indexing at their edges.

Device mode against upload mode: every augment kernel runs once drawing its own jitter (or noise) and once with the
restated draws uploaded, on the same rows, nodes and params.  Upload mode's arithmetic is pinned to the reference
loaders by the parity tests, so this isolates the stream.  The device's double log and sincospi may differ from numpy's
in the last bits, so the rule is "bit-exact except inside a bracket": upload mode runs again with every restated normal
moved 8 double ulps down or up, per coordinate in all 8 sign combinations (the dst transform mixes coordinates, and each
output is monotone in each coordinate's jitter), and the device value must lie between the smallest and the largest of
those results.  8 ulps is not measured: it covers CUDA's documented bounds (log and sincospi 1 ulp each, sqrt and the
products correctly rounded) plus numpy's libm (under 1 ulp per call) with room to spare.  A bracket wider than 1 fp32
ulp fails, and the number of elements with a non-empty bracket is reported.  Clipped draws are exactly +-clip and must
match bit for bit.

Indexing: train mode off, outputs pre-filled with NaN, against the float64 restatement to within 1 fp32 ulp."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from tests import pairgen_ref as ref
from tests.test_gpu_pairgen import _ulps
from tests.util_gpu import dev, make_opt
from usip_b200 import _lib, ops
from usip_b200.ops import _p, _stream, check

pytestmark = pytest.mark.gpu
T, H, D3, PERT, TR, ENU, HS = (ops.PAIR_TRAIN, ops.PAIR_ROT_HORIZONTAL, ops.PAIR_ROT_3D, ops.PAIR_ROT_PERTURBATION,
                               ops.PAIR_TRANSLATION, ops.PAIR_ENU_TO_CAM, ops.PAIR_HEIGHT_SCALE)
CORNERS = [np.array([s[0], s[1], s[2], s[0]]) * 8 for s in itertools.product((-1, 1), repeat=3)]


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=dev())


# ------------------------------------------------------------------------------------------------------ cases
def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _case(kind, N, M, S, C, flags, n_pairs=2, seed=11, step=3, rows="random", zero=False):
    """Inputs of one augment call: kind "det" (usip_pair_augment), "desc" or "mn" (ModelNet, S = 3).  Pairs b and
    b + n_scans share a scan; rows="repeat" names one row at every position; zero=True makes every coordinate 0, so
    that without a shift an output is the scaled jitter itself, resolved to fp32's relative precision."""
    rng = np.random.RandomState(N * 7 + M + S + C + flags)
    n_scans = max(1, n_pairs - 1)
    L = max(N, 300) + 17
    scans = rng.uniform(-30, 30, (n_scans * L, C)).astype(np.float32)
    scans[:, 3:] = rng.normal(size=(n_scans * L, C - 3))
    if zero:
        scans[:] = 0
    off = (np.arange(n_scans + 1) * L).astype(np.int64)
    pair_scan = np.arange(n_pairs) % n_scans
    soc = (np.repeat(pair_scan, 2) if kind != "desc" else rng.randint(0, n_scans, 2 * n_pairs)).astype(np.int32)
    rws = rng.randint(0, L, (2 * n_pairs, N)).astype(np.int32) if rows == "random" else np.full((2 * n_pairs, N), 7,
                                                                                                  np.int32)
    nodes = rng.uniform(-30, 30, (2 * n_pairs, 3, M)).astype(np.float32)
    if zero:
        nodes[:] = 0
    nb = 2 * n_pairs if kind == "desc" else n_pairs
    params = np.zeros((nb, ops.DESC_PARAM_STRIDE if kind == "desc" else ops.PAIR_PARAM_STRIDE))
    for b in range(nb):
        for r in range(3):
            params[b, 9 * r:9 * r + 9] = _rotation(rng).ravel()
        params[b, 27] = rng.uniform(0.7, 1.3) if kind != "desc" or b % 2 == 0 else params[b - 1, 27]
        params[b, 28:31] = rng.uniform(-1, 1, 3)
        if kind != "desc":
            params[b, 31:40] = _rotation(rng).astype(np.float32).ravel()
            params[b, 40:43] = rng.uniform(-0.5, 0.5, 3).astype(np.float32)
            params[b, 43] = np.float32(rng.uniform(0.9, 1.1))
            params[b, 44] = rng.uniform(0.8, 1.2)
    return dict(kind=kind, scans=scans, off=off, soc=soc, rows=rws, nodes=nodes, params=params, S=S, flags=flags,
                seed=seed, step=step, B=n_pairs, N=N, M=M)


def _run(cs, jit=None, flags=None, seed=None, step=None):
    """One augment call with NaN-filled outputs -> the outputs as numpy arrays."""
    kind, B, N, M, S = cs["kind"], cs["B"], cs["N"], cs["M"], cs["S"]
    flags = cs["flags"] if flags is None else flags
    seed = cs["seed"] if seed is None else seed
    step = cs["step"] if step is None else step
    lib = _lib.load()
    ins = [_d(cs[k]) for k in ("scans", "off", "soc", "rows", "nodes", "params")]
    jt = [None if j is None else _d(j) for j in (jit or (None, None, None))]
    outs = [_nan(B, 3, N), _nan(B, S, N), _nan(B, 3, M), _nan(B, 3, N), _nan(B, S, N), _nan(B, 3, M)]
    if kind != "desc":
        outs += [_nan(B, 3, 3), _nan(B), _nan(B, 3, 1)]
    fn = {"det": lib.usip_pair_augment, "desc": lib.usip_desc_pair_augment, "mn": lib.usip_modelnet_pair_augment}[kind]
    rc = fn(_p(ins[0]), cs["scans"].shape[1], *[_p(t) for t in ins[1:]], *[_p(t) for t in jt],
            ctypes.c_uint64(seed & (2 ** 64 - 1)), ctypes.c_uint64(step & (2 ** 64 - 1)), int(flags), S, B, N, M,
            *[_p(t) for t in outs], _stream())
    check(rc, kind)
    return [o.cpu().numpy() for o in outs]


def _restated_jitter(cs, ulps=0, seed=None, step=None):
    seed = cs["seed"] if seed is None else seed
    step = cs["step"] if step is None else step
    if cs["kind"] == "mn":
        return ref.modelnet_jitter(seed, step, cs["B"], cs["N"], cs["M"], ulps)
    return ref.kitti_jitter(seed, step, 2 * cs["B"], cs["N"], cs["M"], cs["S"], ulps)


def _restatement(cs, jit=None, flags=None):
    fn = {"det": ref.pair_augment, "desc": ref.desc_pair_augment, "mn": ref.modelnet_pair_augment}[cs["kind"]]
    args = [cs[k] for k in ("scans", "off", "soc", "rows", "nodes", "params")]
    flags = cs["flags"] if flags is None else flags
    if cs["kind"] == "mn":
        return fn(*args, flags, *(jit or ()))
    return fn(*args, cs["S"], flags, *(jit or ()))


def _bracket(got, runs, what):
    """got lies between the smallest and the largest of runs, elementwise; no bracket wider than 1 fp32 ulp.
    -> (elements, non-empty brackets)."""
    lo, hi = np.minimum.reduce(runs), np.maximum.reduce(runs)
    assert not np.isnan(got).any(), (what, "unwritten (NaN) outputs", int(np.isnan(got).sum()))
    w = _ulps(lo, hi)
    assert w.max() <= 1, (what, "bracket wider than 1 fp32 ulp", int(w.max()))
    bad = ~((lo <= got) & (got <= hi))
    assert not bad.any(), (what, int(bad.sum()), "outside the bracket, first at", np.argwhere(bad)[0].tolist(),
                           float(got[bad][0]), float(lo[bad][0]), float(hi[bad][0]))
    return got.size, int((w > 0).sum())


def _device_equals_upload(cs, seed=None, step=None):
    """The device-mode outputs against the restated-jitter uploads (see the module docstring) -> (device outputs,
    clipped src pc and node draws, elements, non-empty brackets)."""
    got = _run(cs, seed=seed, step=step)
    nominal_jit = _restated_jitter(cs, 0, seed, step)
    nominal = _run(cs, nominal_jit)
    runs = [_run(cs, _restated_jitter(cs, u, seed, step)) for u in CORNERS]
    name = "%s flags=%d S=%d N=%d M=%d B=%d" % (cs["kind"], cs["flags"], cs["S"], cs["N"], cs["M"], cs["B"])
    n = nb = 0
    for k, g in enumerate(got):
        a, b = _bracket(g, [r[k] for r in runs] + [nominal[k]], "%s output %d" % (name, k))
        n += a; nb += b
    # clipped pc and node draws are exactly +-clip in both modes: src bit for bit there
    n_clipped = 0
    for k, law in ((0, ref.MN_PC_LAW if cs["kind"] == "mn" else ref.PC_LAW),
                   (2, ref.MN_NODE_LAW if cs["kind"] == "mn" else ref.NODE_LAW)):
        clipped = np.abs(nominal_jit[k]) == law[1]                             # (clouds or pairs, N or M, 3)
        src = clipped if cs["kind"] == "mn" else clipped[0::2]
        b, i, x = np.nonzero(src)
        np.testing.assert_array_equal(got[k][b, x, i], nominal[k][b, x, i], err_msg=name)
        n_clipped += len(b)
    # the float64 restatement with the same jitter, to within 1 fp32 ulp
    want = _restatement(cs, nominal_jit)
    for k, (g, w) in enumerate(zip(nominal, want)):
        assert _ulps(g, w.reshape(g.shape)).max() <= 1, (name, "upload vs restatement", k)
    return got, n_clipped, n, nb


DET_CASES = [  # (S, C, flags, N, M, extra)
    (1, 5, T, 1, 1, {}),
    (1, 9, T | H, 257, 300, {}),
    (2, 6, T | D3 | PERT | TR, 255, 64, {}),
    (3, 6, T | ENU | H, 257, 300, {}),
    (3, 7, T | ENU | HS | D3 | PERT | TR, 255, 64, {}),
    (4, 8, T | H, 16384, 512, {"seed": 2 ** 32 + 5}),
    (4, 8, T | D3, 16384, 512, {"zero": True}),
    (5, 8, T | D3 | PERT | TR, 257, 300, {"step": 2 ** 32}),
    (5, 9, T | ENU | HS | H, 255, 64, {"step": 2 ** 32 + 7}),
    (8, 11, T | H | TR, 257, 300, {"step": 0}),
    (8, 12, T | ENU | D3, 255, 64, {"n_pairs": 17, "seed": 2 ** 40 + 3}),
    (4, 8, T | H, 257, 64, {"n_pairs": 1, "rows": "repeat"}),
]
DESC_CASES = [
    (1, 5, T, 1, 1, {}),
    (2, 6, T | H | TR, 257, 300, {}),
    (4, 8, T | D3 | PERT | TR, 16384, 512, {"seed": 2 ** 33 + 1, "step": 2 ** 32}),
    (5, 8, T | ENU | H, 255, 64, {"n_pairs": 17}),
    (8, 11, T | ENU | D3 | PERT | TR, 257, 300, {"step": 2 ** 32 + 7, "rows": "repeat"}),
    (3, 6, T, 255, 64, {"zero": True}),
]
MN_CASES = [
    (3, 6, T, 1, 1, {}),
    (3, 6, T | D3, 257, 300, {"n_pairs": 17}),
    (3, 7, T | H | PERT | TR, 255, 64, {"step": 2 ** 32 + 7, "seed": 2 ** 32}),
    (3, 6, T | D3, 16384, 512, {"zero": True}),
    (3, 6, T | H, 300, 257, {"rows": "repeat", "n_pairs": 1}),
]
ALL = [("det",) + c for c in DET_CASES] + [("desc",) + c for c in DESC_CASES] + [("mn",) + c for c in MN_CASES]


def _ids(c):
    return "%s-S%d-C%d-f%d-N%d-M%d%s" % (c[0], c[1], c[2], c[3], c[4], c[5],
                                         "".join("-%s%s" % (k, v) for k, v in sorted(c[6].items())))


@pytest.mark.parametrize("c", ALL, ids=_ids)
def test_device_jitter_equals_restated_upload(c):
    kind, S, C, flags, N, M, extra = c
    cs = _case(kind, N, M, S, C, flags, **extra)
    got, n_clipped, n, nb = _device_equals_upload(cs)
    print("%s: %d of %d elements in a non-empty bracket, %d clipped src draws" % (_ids(c), nb, n, n_clipped))
    if N >= 16384:
        assert n_clipped > 0                                                     # clipped draws occur
    if extra.get("rows") == "repeat":                                           # one row, distinct jitter per position
        for b in range(cs["B"]):
            assert np.unique(got[0][b], axis=1).shape[1] == N and np.unique(got[3][b], axis=1).shape[1] == N


def test_step_high_word_and_seed_high_word_change_the_stream():
    cs = _case("det", 255, 64, 5, 8, T | H)
    a = _device_equals_upload(cs, step=0)[0]
    b = _device_equals_upload(cs, step=2 ** 32)[0]
    c = _device_equals_upload(cs, seed=cs["seed"] + 2 ** 32, step=0)[0]
    for k in range(6):                                   # the outputs keep the coordinates: most still move
        assert (a[k] == b[k]).mean() < 0.01 and (a[k] == c[k]).mean() < 0.01, k


@pytest.mark.parametrize("c", ALL, ids=_ids)
def test_indexing_without_augmentation(c):
    """Train mode off: every output slot written (NaN pre-fill), and equal to the restatement to within 1 fp32 ulp;
    R, scale and shift exactly the params' fp32 values."""
    kind, S, C, flags, N, M, extra = c
    cs = _case(kind, N, M, S, C, flags, **extra)
    got = _run(cs, flags=flags & ~T)
    want = _restatement(cs, flags=flags & ~T)
    for k, (g, w) in enumerate(zip(got, want)):
        assert not np.isnan(g).any(), (k, int(np.isnan(g).sum()))
        assert _ulps(g, w.reshape(g.shape)).max() <= 1, (k, int(_ulps(g, w.reshape(g.shape)).max()))
        if k >= 6:
            np.testing.assert_array_equal(g, w.reshape(g.shape), err_msg=str(k))
    if kind != "mn" and not flags & ENU:                                         # src is the rows themselves
        sn_col = C - 1 if kind == "det" and S == 1 else 3
        for c_ in range(0, 2 * cs["B"], 2):
            p = cs["scans"][cs["off"][cs["soc"][c_]] + cs["rows"][c_]]
            np.testing.assert_array_equal(got[0][c_ // 2], p[:, 0:3].T)
            np.testing.assert_array_equal(got[1][c_ // 2], p[:, sn_col:sn_col + S].T)
            np.testing.assert_array_equal(got[2][c_ // 2], cs["nodes"][c_])


# ------------------------------------------------------------------------------------------------- test clouds
def _cloud_case(N, M, S, C, flags, n_clouds=3, zero=False):
    cs = _case("desc", N, M, S, C, flags, n_pairs=(n_clouds + 1) // 2, zero=zero)
    cs["soc"], cs["rows"], cs["nodes"] = cs["soc"][:n_clouds], cs["rows"][:n_clouds], cs["nodes"][:n_clouds]
    cs["B"] = n_clouds
    return cs


def _run_cloud(cs, sigma, noise=None, seed=None, step=None):
    B, N, M, S = cs["B"], cs["N"], cs["M"], cs["S"]
    ins = [_d(cs[k]) for k in ("scans", "off", "soc", "rows", "nodes")]
    outs = [_nan(B, 3, N), _nan(B, S, N), _nan(B, 3, M)]
    rc = _lib.load().usip_test_cloud_gather(
        _p(ins[0]), cs["scans"].shape[1], *[_p(t) for t in ins[1:]], _p(None if noise is None else _d(noise)),
        float(sigma), ctypes.c_uint64((cs["seed"] if seed is None else seed) & (2 ** 64 - 1)),
        ctypes.c_uint64((cs["step"] if step is None else step) & (2 ** 64 - 1)), cs["flags"], S, B, N, M,
        *[_p(t) for t in outs], _stream())
    check(rc, "test_cloud_gather")
    return [o.cpu().numpy() for o in outs]


CLOUD_CASES = [(1, 1, 3, 6, 0, {}), (257, 300, 4, 8, ENU, {}), (255, 64, 8, 11, 0, {"n_clouds": 17}),
               (16384, 512, 4, 8, ENU, {"zero": True})]


@pytest.mark.parametrize("c", CLOUD_CASES, ids=lambda c: "N%d-M%d-S%d-f%d%s" % (c[0], c[1], c[2], c[4],
                                                                                  "".join(sorted(c[5]))))
def test_test_cloud_noise(c):
    N, M, S, C, flags, extra = c
    cs = _cloud_case(N, M, S, C, flags, **extra)
    args = [cs[k] for k in ("scans", "off", "soc", "rows", "nodes")]
    plain = _run_cloud(cs, 0.0)                                                  # sigma 0: a bit-exact copy
    for g, w in zip(plain, ref.cloud_gather(*args, S, flags)):
        np.testing.assert_array_equal(g, w)
    sigma = 1.0 if extra.get("zero") else 0.05
    noise = ref.noise_draws(cs["seed"], cs["step"], cs["B"], N)
    up = _run_cloud(cs, sigma, noise)                                            # uploaded noise: exact
    for g, w in zip(up, ref.cloud_gather(*args, S, flags, sigma, noise)):
        np.testing.assert_array_equal(g, w)
    got = _run_cloud(cs, sigma)                                                  # device noise: the bracket rule
    runs = [_run_cloud(cs, sigma, ref.noise_draws(cs["seed"], cs["step"], cs["B"], N, u)) for u in CORNERS]
    n, nb = _bracket(got[0], [r[0] for r in runs] + [up[0]], "test cloud pc")
    print("test clouds N=%d: %d of %d elements in a non-empty bracket" % (N, nb, n))
    np.testing.assert_array_equal(got[1], up[1])
    np.testing.assert_array_equal(got[2], up[2])
    assert not np.array_equal(got[0], _run_cloud(cs, sigma, step=cs["step"] + 2 ** 32)[0])


# --------------------------------------------------------------------------------- builders at the training shapes
def _e2e(builder, out, n_out):
    """A device-mode build against upload mode assembled from builder.last (rows, FPS nodes, params) and the restated
    jitter, under the bracket rule."""
    last = builder.last
    _, nodes = ops.fps(last["candidates"], last["start"], builder.M, want_nodes=True)
    cs = dict(kind={"DescriptorPairBuilder": "desc", "ModelNetPairBuilder": "mn"}.get(type(builder).__name__, "det"),
              rows=last["rows"].cpu().numpy(), nodes=nodes.cpu().numpy(), params=last["params"].cpu().numpy(),
              S=builder.S, flags=builder.flags, seed=builder.seed, step=builder.step - 1, N=builder.N, M=builder.M)
    cs["B"] = cs["rows"].shape[0] // 2
    return cs, [o.cpu().numpy() for o in out[:n_out]]


def _e2e_check(cs, got, scans, off, soc, name):
    cs.update(scans=scans, off=off, soc=soc)
    runs = [_run(cs, _restated_jitter(cs, u)) for u in [0] + CORNERS]
    n = nb = 0
    for k, g in enumerate(got):
        a, b = _bracket(g, [r[k] for r in runs], "%s output %d" % (name, k))
        n += a; nb += b
    print("%s: %d of %d elements in a non-empty bracket" % (name, nb, n))


def _stacked(arrs):
    off = np.concatenate([[0], np.cumsum([len(a) for a in arrs])]).astype(np.int64)
    return np.concatenate(arrs), off


def test_kitti_detector_build_at_the_training_shape():
    from usip_b200.data import kitti_detector_loader as kdl
    B, items = 8, [0, 1, 2, 3, 4, 5, 6, 2]
    scans, off = _stacked([kdl.synthetic_scan(300 + i, 20480) for i in range(7)])
    opt = make_opt(input_pc_num=16384, node_num=512, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                   rot_perturbation=False, translation_perturbation=True, radius_threshold=100.0, batch_size=B)
    b = kdl.DetectorPairBuilder(opt, "train", dev(), seed=2 ** 32 + 9, rng="device")
    out = b.build(_d(scans), off, items, step=2 ** 32 + 1)
    cs, got = _e2e(b, out, 9)
    _e2e_check(cs, got, scans, off, np.repeat(items, 2).astype(np.int32), "kitti detector B=8 N=16384")


def test_modelnet_build_at_the_training_shape():
    from usip_b200.data import modelnet_shrec_loader as mnl
    B = 24
    scans, off = _stacked([mnl.synthetic_object(500 + i, 10000) for i in range(6)])
    items = [i % 6 for i in range(B)]
    opt = make_opt(dataset="modelnet", classes=40, input_pc_num=5000, node_num=512, surface_normal_len=3,
                   rot_horizontal=False, rot_3d=True, rot_perturbation=True, translation_perturbation=True,
                   batch_size=B)
    b = mnl.ModelNetPairBuilder(opt, "train", dev(), seed=4, rng="device")
    out = b.build(_d(scans), off, items, step=6)
    cs, got = _e2e(b, out, 9)
    _e2e_check(cs, got, scans, off, np.repeat(items, 2).astype(np.int32), "modelnet B=24 N=5000")


def test_kitti_descriptor_build():
    from usip_b200.data import kitti_descriptor_loader as kdesc
    from usip_b200.data import kitti_detector_loader as kdl
    B = 4
    scans, off = _stacked([kdl.synthetic_scan(700 + i, 20480) for i in range(6)])
    anc, pos = [0, 2, 4, 1], [1, 3, 5, 1]
    opt = make_opt(input_pc_num=16384, node_num=512, surface_normal_len=4, rot_horizontal=True, rot_3d=True,
                   rot_perturbation=True, translation_perturbation=True, positive_radius_threshold=5.0,
                   negative_radius_threshold=50.0, batch_size=B)
    b = kdesc.DescriptorPairBuilder(opt, "train", dev(), seed=8, rng="device")
    out = b.build(_d(scans), off, anc, pos, step=2)
    cs, got = _e2e(b, out, 6)
    soc = np.stack([anc, pos], 1).ravel().astype(np.int32)
    _e2e_check(cs, got, scans, off, soc, "kitti descriptor B=4 N=16384")


def test_oxford_detector_build():
    from usip_b200.data import oxford_detector_loader as odet
    B = 4
    scans, off = _stacked([odet.synthetic_enu_scan(900 + i, 20000) for i in range(4)])
    items = [0, 1, 2, 3]
    opt = make_opt(input_pc_num=16384, node_num=512, surface_normal_len=4, rot_horizontal=True, rot_3d=False,
                   rot_perturbation=False, translation_perturbation=False, is_height_scaling=True, batch_size=B)
    b = odet.OxfordPairBuilder(opt, "train", dev(), seed=3, rng="device")
    assert b.flags & HS and b.flags & ENU
    out = b.build(_d(scans), off, items, step=2 ** 32 + 7)
    cs, got = _e2e(b, out, 9)
    _e2e_check(cs, got, scans, off, np.repeat(items, 2).astype(np.int32), "oxford detector B=4 N=16384")
