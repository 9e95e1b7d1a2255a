"""-m gpu: every element of every parameter gradient of the fused backward plans (engine.detector_backward,
ablation_backward, descriptor_backward) and of the two train steps (ModelDetector.optimize on its CUDA-graph and eager
paths, ModelDescriptor.optimize) against float64 autograd of tests/model_ref64.py, run on the GPU with every discrete
decision pinned to what the plan chose.

Network level: a keep=True forward, random float32 upstream gradients (g_kp, g_sig / g_desc: they reach every keypoint,
not only the ones the loss arg-mins pick), the plan's backward, and L = <g, outputs> differentiated in float64.
Pinning must not hide a wrong choice, so every pinned decision is checked first: min_idx and the kNN / ball indices equal
exact recomputations (oracle/), and every pinned pool choice lies within GAP of the float64 maximum of its group.

Metric per tensor: max|g - g64| / max|g64|.  A conv bias whose true gradient is 0 (its shift is removed by the next
train-mode BatchNorm) is checked as max|g| against max|g64| of its weight.

The ReLU active sets are pinned too.  An activation within float32 rounding of 0 is a decision like an arg-max: with the
active sets left to float64, the few that flip (3 to 41 of 5e6 to 3e7 per case) moved single gradient elements by 1e-2
to 2.7e-1 of max|g64|, on every path including fp32 SIMT.  Pinned -- and each pinned flip checked to lie within GAP of
0 -- the fp32 paths agree to 1e-5.

Measured on 1x H100 80GB HBM3 at a 700 W power limit (worst over use_tensor_cores False / True; the whole file, 27
cases, ran in 26 s):
  network level, max|g-g64|/max|g64|
    kitti 5.2e-6 / 1.1e-5   ragged 8.4e-6 / 1.0e-5   q1024 9.4e-6 / 1.5e-5   q1020 8.1e-6 / 1.2e-5
    kn8 6.1e-6 / 1.0e-5     kn32 6.1e-6 / 9.8e-6     s0 6.3e-6 / 1.3e-5      lite 4.5e-6 / 6.5e-6
    ablation knn 6.9e-6 / 1.1e-5   ablation ball 5.2e-6 / 9.0e-6   descriptor 1.4e-6 / 2.8e-6
    backward_precision="tf32": 1.1e-3
  train steps: ModelDetector.optimize graph 4.6e-5, eager 4.4e-5; ModelDescriptor.optimize 4.5e-6
  zero-gradient biases max|g| / max|gW64|: fp32 1.6e-6, tf32 1.5e-4
  worst pinned pool choice below its float64 max 2.6e-6, worst |z| of a flipped ReLU decision 3.5e-6 (x channel |max|)
The bounds below keep a factor of 2 or more over these.
"""
import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests import model_ref64 as ref64
from tests.util_gpu import dev, load_params, make_opt

pytestmark = pytest.mark.gpu

GAP = 1e-5                # a pinned pool choice may lie at most this far below its group's float64 max, and a pinned ReLU
                          # decision that disagrees with float64 this close to 0 (x the channel's |max|)
BOUND = dict(fp32=5e-5, tf32=2e-3)       # network level
STEP_BOUND = 1e-4                        # train steps: the loss backward kernels on top
ZERO_BIAS = dict(fp32=1e-5, tf32=1e-3)   # max|g| of a bias with true gradient 0, relative to max|g64| of its weight


def _flip_bn_signs(P, seed):
    """Negative BN scales in about a quarter of the channels of every BatchNorm: max_k relu(bn(y)) then sits at the
    arg-MIN of y there, which the pools and their backward must honour."""
    rng = np.random.default_rng(seed)
    for k in list(P):
        if k.endswith("norm.weight"):
            P[k] = (P[k] * np.where(rng.random(P[k].shape) < 0.25, -1, 1)).astype(np.float32)
    return P


def _sel(grp, st):
    """Row-in-group of max_k relu(bn(y_k)) as the plan's group_select takes it: arg-max where the BN scale >= 0, arg-min
    elsewhere.  -> [Q, C] int64."""
    return torch.where((st.scale >= 0)[None, :], grp["amax"], grp["amin"]).long()


def _bcm(t, B, M):
    return t.reshape(B, M, -1).permute(0, 2, 1).contiguous()


def _on(Y, st):
    """The plan's ReLU active set of a BN+ReLU layer, fmaf(y, scale, shift) > 0: the product of two floats is exact in
    float64, so the float64 sum has the sign of the fused multiply-add.  [rows, C] bool"""
    return Y.double() * st.scale.double()[None, :] + st.shift.double()[None, :] > 0


def _rows(t, B, L):
    """[B*L, C] rows in (cloud, group row) order -> (B, C, L)."""
    return t.reshape(B, L, -1).permute(0, 2, 1)


def _point_rows(t, perm):
    """[B*N, C] rows sorted by node (perm: sorted position -> original point) -> (B, C, N) in original point order."""
    B, N = perm.shape
    out = torch.empty((B, t.shape[1], N), dtype=t.dtype, device=t.device)
    return out.scatter_(2, perm.long().unsqueeze(1).expand(B, t.shape[1], N), _rows(t, B, N))


def _knn_relus(ctx, B, M):
    Kn = ctx["Kn"]
    pins = {}
    for side, name in (("before", "layers_before"), ("after", "layers_after")):
        for i, (Y, st) in enumerate(ctx[side]):
            pins["relu:knnlayer_1.%s.%d" % (name, i)] = _rows(_on(Y, st), B, M * Kn)
    pins["relu:mlp1"] = _rows(_on(ctx["Y10"], ctx["bn10"]), B, M)
    pins["relu:mlp2"] = _rows(_on(ctx["Y11"], ctx["bn11"]), B, M)
    return pins


def _group_relus(gctx, B, M, K, conv5=True):
    return {"relu:conv%d" % i: _rows(_on(gctx["Y%d" % i], gctx["bn%d" % i]), B, M * K) for i in range(1, 6 if conv5 else 5)}


def _check_pools(pins, record, tag, min_idx=None, M=None):
    gaps = ref64.pool_gaps(record)
    if min_idx is not None:
        gaps.update(ref64.seg_gaps(record, min_idx, M))
    relus = ref64.relu_gaps(record)
    worst = max(v[0] for v in gaps.values())
    print("  %s pools: worst gap %.1e, choices off the float64 arg-max: %s" % (
        tag, worst, ", ".join("%s %d/%d" % (k, v[1], v[2]) for k, v in sorted(gaps.items()))))
    print("  %s ReLUs: worst |z| of a flipped decision %.1e, flipped %d of %d" % (
        tag, max(v[0] for v in relus.values()), sum(v[1] for v in relus.values()), sum(v[2] for v in relus.values())))
    bad = {k: v for k, v in list(gaps.items()) + list(relus.items()) if v[0] > GAP}
    assert not bad, (tag, bad)


def _compare(named, grads64, tag, prec, bound=None):
    """named: [(name, gradient)] of the plan; grads64: name -> float64 gradient.  -> worst relative error."""
    bound = BOUND[prec] if bound is None else bound
    errs, zero, bad = {}, {}, []
    for name, g in named:
        g64 = grads64[name]
        s64 = float(g64.abs().max())
        if name.endswith("conv.bias"):
            sw = float(grads64[name.replace("conv.bias", "conv.weight")].abs().max())
            if s64 <= 1e-9 * sw:                            # true gradient 0
                zero[name] = float(g.abs().max()) / sw
                if not zero[name] <= ZERO_BIAS[prec]:
                    bad.append((name, "zero-gradient bias", zero[name]))
                continue
        errs[name] = float((g.double() - g64).abs().max()) / s64
        if not errs[name] <= bound:
            bad.append((name, errs[name]))
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print("  %s: worst max|g-g64|/max|g64| %.2e (%s); zero-gradient biases max|g| %.1e" % (
        tag, top[0][1], ", ".join("%s %.1e" % kv for kv in top), max(zero.values(), default=0.0)))
    assert not bad, (tag, bad)
    return top[0][1]


def _grads64(P64):
    return {k: v.grad for k, v in P64.items() if v.requires_grad}


def _c(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


# ----------------------------------------------------------------------------- detector pins from the plan's ctx
def _detector_pins(ctx, x, node, Kn):
    """Decisions of a keep=True detector_forward, as original point / row-in-group indices, each checked for validity."""
    Bp, N, M = ctx["Bp"], ctx["N"], ctx["M"]
    min_idx = ctx["min_idx"].long()
    assert np.array_equal(ctx["min_idx"].cpu().numpy(), orc.som_assign(x, node)), "SOM assignment differs from the oracle"
    knn_i = ctx["knn_i"].long()
    cm = ctx["cmean"].cpu().numpy()
    assert np.array_equal(ctx["knn_i"].cpu().numpy(), orc.knn(cm, cm, Kn)[0]), "node kNN differs from the oracle"
    perm = ctx["perm"].long().reshape(-1)

    def orig(arg):                                         # global sorted row -> original point index of its cloud
        return _bcm(perm[arg.long().clamp(min=0)], Bp, M)
    pins = ref64.Pins(min_idx=min_idx, knn_i=knn_i, arg1=orig(ctx["arg1"]), arg2=orig(ctx["arg2"]),
                      sel_b=_bcm(_sel(ctx["grp_b"], ctx["before"][-1][1]), Bp, M),
                      sel_a=_bcm(_sel(ctx["grp_a"], ctx["after"][-1][1]), Bp, M), record={}, **_knn_relus(ctx, Bp, M))
    for name, (Y, st) in (("first_pointnet.layers.0", ("Y0", "bn0")), ("first_pointnet.layers.1", ("Y1", "bn1")),
                          ("second_pointnet.layers.0", ("Y3", "bn3"))):
        pins["relu:" + name] = _point_rows(_on(ctx[Y], ctx[st]), ctx["perm"])
    return pins


def _detector_setup(B, N, M, S, Kn, use_tc, scene="outdoor", seed=0, far=False, prec="3xtf32"):
    from usip_b200.models import networks
    d = orc.synth_pair(B, N, M, S, kind="lidar", seed=seed)
    if far:
        d["src_node"][0, :, 7] = 500.0                   # an empty cluster
    C1, C2 = (64, 256) if scene == "indoor" else (128, 512)
    P = orc.init_detector_params(S=S, seed=seed + 1, C1=C1, C2=C2, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    _flip_bn_signs(P, seed + 2)
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, node_knn_k_1=Kn, scene=scene,
                   use_tensor_cores=use_tc, backward_precision=prec)
    return d, P, opt, (networks.RPN_DetectorLite if scene == "indoor" else networks.RPN_Detector)


DET_CASES = {
    # name: (B pairs, N, M, S, Kn, scene, far, backward_precision)
    "kitti": (2, 2048, 64, 4, 16, "outdoor", False, "3xtf32"),            # golden shape: C1=128, C2=512
    "ragged": (3, 3001, 50, 4, 16, "outdoor", True, "3xtf32"),            # B'=6, no tile multiple, one empty cluster
    "q1024": (2, 2048, 256, 4, 16, "outdoor", False, "3xtf32"),           # Q = B'M = 1024: node layers on tensor cores
    "q1020": (2, 2048, 255, 4, 16, "outdoor", False, "3xtf32"),           # Q = 1020: the same layers on SIMT
    "kn8": (2, 2048, 64, 4, 8, "outdoor", False, "3xtf32"),               # kNN groups of 8: SIMT group epilogue
    "kn32": (2, 2048, 64, 4, 32, "outdoor", False, "3xtf32"),
    "s0": (2, 2048, 64, 0, 16, "outdoor", False, "3xtf32"),               # no surface normals
    "lite": (2, 2048, 64, 4, 16, "indoor", False, "3xtf32"),              # RPN_DetectorLite: C1=64, C2=256
    "tf32": (2, 2048, 64, 4, 16, "outdoor", False, "tf32"),               # backward GEMMs as single-pass TF32
}


@pytest.mark.parametrize("use_tc", [False, True])
@pytest.mark.parametrize("case", list(DET_CASES))
def test_detector_backward_every_element_vs_float64(case, use_tc):
    from usip_b200 import engine
    B, N, M, S, Kn, scene, far, prec = DET_CASES[case]
    if prec == "tf32" and not use_tc:
        pytest.skip("backward_precision only selects the tensor-core GEMMs")
    d, P, opt, cls = _detector_setup(B, N, M, S, Kn, use_tc, scene, seed=100 + list(DET_CASES).index(case), far=far, prec=prec)
    net = cls(opt).to(dev())
    load_params(net, P)
    net.train()
    x = np.concatenate([d["src_pc"], d["dst_pc"]]); sn = np.concatenate([d["src_sn"], d["dst_sn"]])
    node = np.concatenate([d["src_node"], d["dst_node"]])
    with torch.no_grad():
        _, kp, sig, ctx, _ = engine.detector_forward(net, _c(x), _c(sn), _c(node), 0, use_tc=use_tc, keep=True)
        gen = torch.Generator().manual_seed(M + N)
        g_kp = torch.randn(tuple(kp.shape), generator=gen).to(dev())
        g_sig = torch.randn(tuple(sig.shape), generator=gen).to(dev())
        grads = engine.detector_backward(net, ctx, g_kp, g_sig)
    torch.cuda.synchronize()
    pins = _detector_pins(ctx, x, node, Kn)
    P64 = ref64.params64(net.state_dict(), dev())
    _, kp64, sig64 = ref64.detector_forward(P64, pins, _c(x).double(), _c(sn).double(), _c(node).double(),
                                            float(opt.loss_sigma_lower_bound))
    assert float((kp64.detach() - kp.double()).abs().max() / kp64.detach().abs().max()) < 1e-5
    ((kp64 * g_kp.double()).sum() + (sig64 * g_sig.double()).sum()).backward()
    tag = "%s use_tc=%s" % (case, use_tc)
    _check_pools(pins, pins.record, tag, pins["min_idx"], M)
    _compare([(k, g) for (k, _), g in zip(net.named_parameters(), grads)], _grads64(P64), tag,
             "tf32" if prec == "tf32" else "fp32")


# ----------------------------------------------------------------------------- ablation detectors
@pytest.mark.parametrize("use_tc", [False, True])
@pytest.mark.parametrize("mode", ["knn", "ball"])
def test_ablation_backward_every_element_vs_float64(mode, use_tc):
    from usip_b200 import engine, ops
    from usip_b200.models import networks
    B, N, M, S, Kn, seed = 2, 4096, 128, 4, 16, 1239
    d = orc.ablation_inputs(seed, B, N, M, S)
    P = orc.init_ablation_params(S=S, seed=seed, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    _flip_bn_signs(P, seed)
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, node_knn_k_1=Kn, use_tensor_cores=use_tc)
    net = (networks.RPN_Detector_KNN if mode == "knn" else networks.RPN_Detector_Ball)(opt).to(dev())
    load_params(net, P)
    net.train()
    x, sn, node = _c(d["pc"]), _c(d["sn"]), _c(d["node"])
    with torch.no_grad():
        _, kp, sig, ctx = engine.ablation_forward(net, x, sn, node, 0, use_tc=use_tc, keep=True, mode=mode)
        gen = torch.Generator().manual_seed(seed)
        g_kp = torch.randn(tuple(kp.shape), generator=gen).to(dev())
        g_sig = torch.randn(tuple(sig.shape), generator=gen).to(dev())
        grads = engine.ablation_backward(net, ctx, g_kp, g_sig)
        if mode == "knn":
            idx, _, rows = ops.knn_group(x, sn, node, 64, want_group=False, rows_ld=8)
        else:
            idx, _, rows = ops.ball_group(x, sn, node, engine.ABLATION_RADIUS, 64, want_group=False, rows_ld=8)
    torch.cuda.synchronize()
    gctx = ctx["group_net"]
    assert torch.equal(rows, gctx["rows"]), "the grouping call does not reproduce the plan's rows"
    gi = idx.cpu().numpy()
    if mode == "knn":
        ref_i, _ = orc.knn(d["node"], d["pc"], 64)
        assert np.array_equal(np.sort(gi, axis=2), np.sort(ref_i, axis=2)), "kNN groups differ from the oracle"
    else:
        assert np.array_equal(gi, orc.ball_query_xyz(d["pc"], d["node"], 2.0, 64)), "balls differ from the oracle"
    assert np.array_equal(ctx["knn_i"].cpu().numpy(), orc.knn(d["node"], d["node"], Kn)[0])
    pins = ref64.Pins(idx=idx.long(), knn_i=ctx["knn_i"].long(),
                      sel_b=_bcm(_sel(ctx["grp_b"], ctx["before"][-1][1]), B, M),
                      sel_a=_bcm(_sel(ctx["grp_a"], ctx["after"][-1][1]), B, M), record={},
                      sel3=_bcm(_sel(gctx["grp3"], gctx["bn3"]), B, M), sel5=_bcm(_sel(gctx["grp5"], gctx["bn5"]), B, M),
                      **_knn_relus(ctx, B, M), **_group_relus(gctx, B, M, 64))
    P64 = ref64.params64(net.state_dict(), dev())
    kp64, sig64 = ref64.ablation_forward(P64, pins, x.double(), sn.double(), node.double(), float(opt.loss_sigma_lower_bound))
    assert float((kp64.detach() - kp.double()).abs().max() / kp64.detach().abs().max()) < 1e-5
    ((kp64 * g_kp.double()).sum() + (sig64 * g_sig.double()).sum()).backward()
    tag = "ablation %s use_tc=%s" % (mode, use_tc)
    _check_pools(pins, pins.record, tag)
    _compare([(k, g) for (k, _), g in zip(net.named_parameters(), grads)], _grads64(P64), tag, "fp32")


# ----------------------------------------------------------------------------- descriptor
def _desc_setup(use_tc, seed=33, B=3, N=16384, M=40, S=4, K=64):
    from oracle import usip_oracle as o
    d = o.desc_train_inputs(B, N, M, S, seed)
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=1.0, ball_nsamples=K,
                   descriptor_len=128, use_tensor_cores=use_tc)
    return d, opt


def _desc_params(net, seed):
    """The module's own init with randomized BatchNorm affines (some scales negative) and non-zero conv biases."""
    rng = np.random.default_rng(seed)
    P = {k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}
    for k in P:
        if k.endswith("norm.weight"):
            P[k] = rng.uniform(0.5, 1.5, P[k].shape).astype(np.float32)
        elif k.endswith("norm.bias") or k.endswith("conv.bias"):
            P[k] = rng.normal(0, 0.1, P[k].shape).astype(np.float32)
    return _flip_bn_signs(P, seed + 1)


def _desc_pins(ctx, x, sn, kp, perm, K, feats):
    """Ball indices from the oracle on the permuted points -- the plan's x_features must be exactly their gather -- and
    the two pools of the plan."""
    B, M = ctx["Bp"], ctx["M"]
    xp = np.ascontiguousarray(x[:, :, perm])
    idx = orc.ball_query_xyz(xp, kp, 1.0, K)
    x_aug = np.concatenate([xp, sn[:, :, perm]], 1)
    want = np.take_along_axis(x_aug, np.broadcast_to(idx.astype(np.int64).reshape(B, 1, M * K), (B, x_aug.shape[1], M * K)),
                              2).reshape(B, -1, M, K)
    want[:, :3] -= kp[:, :, :, None]
    assert np.array_equal(feats.cpu().numpy(), want), "x_features are not the gather of the oracle's balls"
    hits = (np.linalg.norm(xp[:, :, None, :] - kp[:, :, :, None], axis=1) <= 1.0).sum(2)
    assert (hits < K).any() and (hits >= K).any(), "the inputs must hold both padded and full balls"
    return ref64.Pins(perm=torch.from_numpy(perm).to(dev()), idx=torch.from_numpy(idx.astype(np.int64)).to(dev()),
                      sel3=_bcm(_sel(ctx["grp3"], ctx["bn3"]), B, M), sel5=_bcm(ctx["grp5"]["amax"].long(), B, M),
                      record={}, **_group_relus(ctx, B, M, K, conv5=False))


@pytest.mark.parametrize("use_tc", [False, True])
def test_descriptor_backward_every_element_vs_float64(use_tc):
    from usip_b200 import engine
    from usip_b200.models import networks
    d, opt = _desc_setup(use_tc)
    torch.manual_seed(5)
    net = networks.DescriptorLiteOld(opt).to(dev())
    load_params(net, _desc_params(net, 5))
    net.train()
    x = np.concatenate([d["anc_pc"], d["pos_pc"]]); sn = np.concatenate([d["anc_sn"], d["pos_sn"]])
    kp = np.concatenate([d["anc_kp"], d["pos_kp"]])
    perm = np.random.RandomState(7).permutation(x.shape[2])
    with torch.no_grad():
        desc, feats, ctx = engine.descriptor_forward(net, _c(x), _c(sn), _c(kp), 0, _c(perm), use_tc=use_tc, keep=True)
        g_desc = torch.randn(tuple(desc.shape), generator=torch.Generator().manual_seed(11)).to(dev())
        grads = engine.descriptor_backward(net, ctx, g_desc)
    torch.cuda.synchronize()
    pins = _desc_pins(ctx, x, sn, kp, perm, opt.ball_nsamples, feats)
    P64 = ref64.params64(net.state_dict(), dev())
    desc64 = ref64.descriptor_forward(P64, pins, _c(x).double(), _c(sn).double(), _c(kp).double())
    assert float((desc64.detach() - desc.double()).abs().max()) < 1e-5
    (desc64 * g_desc.double()).sum().backward()
    tag = "descriptor use_tc=%s" % use_tc
    _check_pools(pins, pins.record, tag)
    _compare([(k, g) for (k, _), g in zip(net.named_parameters(), grads)], _grads64(P64), tag, "fp32")


# ----------------------------------------------------------------------------- train steps (loss level)
def _check_min_pins(pins, pairs):
    """Every pinned loss arg-min lies within 1e-6 (relative) of the float64 nearest distance."""
    for key, a, b in pairs:
        a = a.double(); b = b.double()
        d2 = ((a[:, :, :, None] - b[:, :, None, :]) ** 2).sum(1)
        got = torch.gather(d2, 2, pins[key].unsqueeze(2)).squeeze(2)
        best = d2.min(2).values
        assert bool(((got.sqrt() - best.sqrt()) <= 1e-6 * (1 + best.sqrt())).all()), key


@pytest.mark.parametrize("path", ["graph", "eager"])
def test_detector_train_step_grads_vs_float64(path):
    """ModelDetector.optimize(): the gradients it leaves in p.grad against float64 autograd of the restated forward and
    losses, the network decisions from a keep=True forward on the same inputs and parameters, the loss arg-mins from the
    same pairwise-min kernels on those keypoints."""
    from usip_b200 import engine, ops
    from usip_b200.models.keypoint_detector import ModelDetector
    B, N, M, S, Kn = 2, 2048, 64, 4, 16
    d, P, opt, _ = _detector_setup(B, N, M, S, Kn, True, seed=21)
    md = ModelDetector(opt)
    md.use_cuda_graph = path == "graph"
    load_params(md.detector, P)
    keys = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
    md.set_input(*[torch.from_numpy(d[k]) for k in keys])
    sd0 = {k: v.clone() for k, v in md.detector.state_dict().items()}
    x = np.concatenate([d["src_pc"], d["dst_pc"]]); sn = np.concatenate([d["src_sn"], d["dst_sn"]])
    node = np.concatenate([d["src_node"], d["dst_node"]])
    net = md.detector
    net.train()
    with torch.no_grad():
        _, kp, sig, ctx, _ = engine.detector_forward(net, _c(x), _c(sn), _c(node), 0, use_tc=True, keep=True)
        R, scale, shift = _c(d["R"]), _c(d["scale"]).reshape(-1), _c(d["shift"]).reshape(B, 3)
        kp_t = ops.transform_points(kp[:B].contiguous(), R, scale, shift)
        i_sd = ops.pairwise_min(kp_t, kp[B:].contiguous())[1]
        i_ds = ops.pairwise_min(kp[B:].contiguous(), kp_t)[1]
        i_pc = ops.pairwise_min(kp, _c(x))[1]
    pins = _detector_pins(ctx, x, node, Kn)
    pins.update(i_sd=i_sd.long(), i_ds=i_ds.long(), i_src=i_pc[:B].long(), i_dst=i_pc[B:].long())
    _check_min_pins(pins, [("i_sd", kp_t, kp[B:]), ("i_ds", kp[B:], kp_t), ("i_src", kp[:B], _c(d["src_pc"])),
                           ("i_dst", kp[B:], _c(d["dst_pc"]))])
    kp0 = kp.clone()
    del ctx
    md.detector.load_state_dict(sd0)                        # undo the running-statistic update of the decision forward
    md.optimize(epoch=0)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([md.src_keypoints, md.dst_keypoints]), kp0), "the step saw other keypoints"
    P64 = ref64.params64(sd0, dev())
    _, kp64, sig64 = ref64.detector_forward(P64, pins, _c(x).double(), _c(sn).double(), _c(node).double(),
                                            float(opt.loss_sigma_lower_bound))
    loss64, _ = ref64.detector_loss(pins, kp64, sig64, _c(d["src_pc"]).double(), _c(d["dst_pc"]).double(), R.double(),
                                    scale.double(), shift.double(), float(opt.keypoint_on_pc_alpha))
    assert abs(md.loss.item() - loss64.item()) <= 1e-5 * abs(loss64.item()), (md.loss.item(), loss64.item())
    loss64.backward()
    tag = "ModelDetector.optimize %s" % path
    _check_pools(pins, pins.record, tag, pins["min_idx"], M)
    _compare([(k, p.grad) for k, p in md.detector.named_parameters()], _grads64(P64), tag, "fp32", STEP_BOUND)


def test_descriptor_train_step_grads_vs_float64():
    """ModelDescriptor.optimize(): p.grad against float64 autograd of the restated descriptor and DescPairScanLoss, the
    triplet arg-mins from the same descriptor-space pairwise-min kernel on the plan's descriptors."""
    from usip_b200 import _lib, engine, ops
    from usip_b200.models.keypoint_descriptor import ModelDescriptor
    d, opt = _desc_setup(True, seed=35)
    B, M, K = opt.batch_size, opt.node_num, opt.ball_nsamples
    torch.manual_seed(6)
    md = ModelDescriptor(opt)
    load_params(md.descriptor, _desc_params(md.descriptor, 6))
    md.set_input(*[torch.from_numpy(d[k]) for k in ("anc_pc", "anc_sn", "anc_kp", "anc_sigma", "pos_pc", "pos_sn", "pos_kp",
                                                    "pos_sigma")], torch.from_numpy(d["neg_idx"]))
    sd0 = {k: v.clone() for k, v in md.descriptor.state_dict().items()}
    x = np.concatenate([d["anc_pc"], d["pos_pc"]]); sn = np.concatenate([d["anc_sn"], d["pos_sn"]])
    kp = np.concatenate([d["anc_kp"], d["pos_kp"]])
    perm = np.random.RandomState(35).permutation(x.shape[2])
    net = md.descriptor
    net.train()
    neg_idx = torch.from_numpy(d["neg_idx"]).to(dev())
    with torch.no_grad():
        desc, feats, ctx = engine.descriptor_forward(net, _c(x), _c(sn), _c(kp), 0, _c(perm), use_tc=True, keep=True)
        anc, pos = desc[:B].contiguous(), desc[B:].contiguous()
        neg = anc[neg_idx].contiguous()
        lib = _lib.load()
        am = {}
        for key, other in (("ipos", pos), ("ineg", neg)):
            dd = torch.empty((B, M), dtype=torch.float32, device=dev())
            ii = torch.empty((B, M), dtype=torch.int32, device=dev())
            _lib.check(lib.usip_desc_pairmin_f32(ops._p(anc), ops._p(other), ops._p(dd), ops._p(ii), B, anc.shape[1], M, M,
                                                 ops._stream()), "usip_desc_pairmin_f32")
            am[key] = ii.long()
    pins = _desc_pins(ctx, x, sn, kp, perm, K, feats)
    pins.update(am)
    _check_min_pins(pins, [("ipos", anc, pos), ("ineg", anc, neg)])
    desc0 = desc.clone()
    del ctx
    md.descriptor.load_state_dict(sd0)
    np.random.seed(35)                                      # the step's forward draws the same np.random.permutation(N)
    md.optimize(epoch=0)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([md.anc_descriptors, md.pos_descriptors]).detach(), desc0), "the step saw other descriptors"
    P64 = ref64.params64(sd0, dev())
    desc64 = ref64.descriptor_forward(P64, pins, _c(x).double(), _c(sn).double(), _c(kp).double())
    loss64, _ = ref64.descriptor_train_loss(pins, desc64, neg_idx, _c(d["anc_sigma"]).double(), opt.triple_loss_gamma,
                                            opt.sigma_max)
    assert abs(md.loss.item() - loss64.item()) <= 1e-5 * abs(loss64.item()), (md.loss.item(), loss64.item())
    loss64.backward()
    tag = "ModelDescriptor.optimize"
    _check_pools(pins, pins.record, tag)
    _compare([(k, p.grad) for k, p in md.descriptor.named_parameters()], _grads64(P64), tag, "fp32", STEP_BOUND)
