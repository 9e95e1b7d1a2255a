"""-m gpu: training the indoor descriptor -- usip_group_max_combine_arg, the DescCGFLoss kernels, the backward of
DescriptorLiteOldGlobal and ModelDescriptorIndoor.optimize() / test_model().

  * combine with args: values bit-identical to usip_group_max_combine, args the first index of the max / min (NaN never
    wins, an all -inf group gives row 0) over the whole group, with and without sub-group args;
  * usip_desc_cgf_f32 against the literal torch restatement of tests/cgf_ref.py on the same draws: picks and mask
    identical, loss and active within CGF_REL;
  * usip_desc_cgf_bwd against float64 autograd with the picks pinned, and bit-identical on a second run;
  * descriptor_global_backward: every element of every parameter gradient against a float64 autograd restatement
    (tests/model_ref64.py's grouped PointNet, a global pool over M, fc1..fc3, the L2 norm), pins checked first;
  * one optimize() against the reference run on the CPU (tests/golden/descriptor_indoor_train.npz, its draws substituted)
    and against float64 autograd; at SceneNN's training shape against the reference run on the GPU
    (tests/golden/reference_descriptor_indoor_train.npz, the seeded CUDA draws);
  * test_model(), a few training steps and update_learning_rate.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import cgf_ref
from tests import desc_indoor_ref as dref
from tests import model_ref64 as ref64
from oracle import usip_oracle as orc
from tests.test_gpu_model_grads import BOUND, STEP_BOUND, _bcm, _check_pools, _compare, _desc_params, _grads64, _group_relus, \
    _on, _rows, _sel
from tests.util_gpu import cu, dev, golden, load_params, make_opt, rel_err
from usip_b200 import _lib, ops

pytestmark = pytest.mark.gpu
CGF_REL = 1e-5           # loss of the kernel against the fp32 torch restatement, relative to its max
REL = 1e-4               # descriptors and loss against the reference (CPU / GPU)


# ----------------------------------------------------------------------------------------------- combine with args
def _first_arg(v, is_max):
    """numpy first-index arg-max (arg-min) over axis 1 of (Q, R, C), NaN never winning; all -inf (+inf) -> 0."""
    v = np.where(np.isnan(v), -np.inf if is_max else np.inf, v)
    return np.argmax(v, 1) if is_max else np.argmin(v, 1)


@pytest.mark.parametrize("ratio,sub", [(3, 64), (4, 64), (7, 64), (64, 0), (512, 0), (1000, 0)])
@pytest.mark.parametrize("C", [36, 128, 256])
def test_group_max_combine_arg(ratio, sub, C):
    g = torch.Generator(device="cuda").manual_seed(ratio * 7 + C)
    for Q in (1, 5, 97):
        gmax = torch.randn((Q * ratio, C), device="cuda", generator=g)
        gmin = torch.randn((Q * ratio, C), device="cuda", generator=g)
        gmax[1::ratio] = gmax[0::ratio]                     # exact ties across sub-groups: the first one wins
        gmin[2::ratio] = gmin[0::ratio] if ratio > 2 else gmin[2::ratio]
        gmax[:ratio, :4] = -float("inf")                    # a group that is -inf throughout
        gmin[:ratio, 4:8] = float("inf")
        gmax[ratio - 1::ratio, 8:10] = float("nan")         # NaN rows never win
        gmin[0::ratio, 10:12] = float("nan")
        amax = torch.randint(0, sub, gmax.shape, device="cuda", dtype=torch.int32, generator=g) if sub else None
        amin = torch.randint(0, sub, gmax.shape, device="cuda", dtype=torch.int32, generator=g) if sub else None
        om, on, am, an = ops.group_max_combine_arg(gmax, ratio, gmin, amax, amin, max(sub, 1))
        wm, wn = ops.group_max_combine(gmax, ratio, gmin)
        torch.cuda.synchronize()
        assert torch.equal(om, wm) and torch.equal(on, wn), (Q, ratio, C)
        for got, v, a, is_max in ((am, gmax, amax, True), (an, gmin, amin, False)):
            r = _first_arg(v.view(Q, ratio, C).cpu().numpy(), is_max)
            want = r if a is None else r * sub + np.take_along_axis(a.view(Q, ratio, C).cpu().numpy(), r[:, None], 1)[:, 0]
            assert np.array_equal(got.cpu().numpy(), want), (Q, ratio, C, is_max)
        # max only, the global-max form
        om2, on2, am2, an2 = ops.group_max_combine_arg(gmax, ratio, None, amax, None, max(sub, 1))
        assert on2 is None and an2 is None and torch.equal(om2, wm) and torch.equal(am2, am)


def test_group_max_combine_arg_refusals():
    lib = _lib.load()
    x = torch.zeros((64, 128), device="cuda")
    a = torch.zeros((64, 128), device="cuda", dtype=torch.int32)
    p, s = ops._p, ops._stream()
    call = lib.usip_group_max_combine_arg
    assert call(p(x), None, None, None, p(x), None, None, None, 4, 1, 16, 128, s) != 0           # no out_amax
    assert call(p(x), p(x), None, None, p(x), p(x), p(a), None, 4, 1, 16, 128, s) != 0           # gmin without out_amin
    assert call(p(x), None, None, p(a), p(x), None, p(a), None, 4, 64, 16, 128, s) != 0          # amin without amax
    assert call(p(x), p(x), p(a), None, p(x), p(x), p(a), p(a), 4, 64, 16, 128, s) != 0          # amax with gmin, no amin
    assert call(p(x), None, p(a), None, p(x), None, p(a), None, 4, 0, 16, 128, s) != 0           # sub 0 with args
    assert call(p(x), None, None, None, p(x), None, p(a), None, 0, 1, 16, 128, s) != 0
    assert call(p(x), None, None, None, p(x), None, p(a), None, 1, 1, 1, 128 * 65536, s) != 0
    assert "group_max_combine_arg" in lib.usip_last_error().decode()
    with pytest.raises(ValueError):
        ops.group_max_combine_arg(x, 5)
    with pytest.raises(ValueError):
        ops.group_max_combine_arg(x, 4, x, a, None, 64)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- DescCGFLoss kernels
def _cgf_case(B, M, D, seed, radius=0.075, sigma_max=0.5, special=()):
    """Keypoints where about half the anchors have a positive within radius, unit descriptors, sigmas, draws."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-1, 1, (B, 3, M))
    near = rng.random((B, M)) < 0.5
    src = rng.integers(0, M, (B, M))
    v = rng.normal(size=(B, 3, M))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    anc = np.where(near[:, None], np.take_along_axis(pos, src[:, None], 2) + v * rng.uniform(0, 0.8 * radius, (B, 1, M)),
                   rng.uniform(-1, 1, (B, 3, M)))
    desc = rng.normal(size=(2, B, D, M))
    desc /= np.linalg.norm(desc, axis=2, keepdims=True)
    sig = rng.uniform(0.05, 0.6, (B, M))
    u = [rng.random((B, M, M)), rng.random((B, M, M)), rng.random((B, M))]
    if "dup" in special:                                   # duplicated positive keypoints: `far` ties to the first index
        pos[:, :, M // 2:] = pos[:, :, :M - M // 2]
    if "all_in" in special:                                # anchor 1 has every positive inside: `out` falls back to 0
        pos[0] = anc[0, :, 1:2] + rng.uniform(-0.02, 0.02, (3, M))
    if "none" in special:                                  # anchor 2 has no positive
        anc[0, :, 2] = 50.0
    if "zero_draw" in special:                             # a masked-in draw of exactly 0 (and the only positive)
        anc[0, :, 3] = pos[0, :, 5]
        u[0][0, 3, :] = 0.0
    if "nan" in special:                                   # every sigma >= sigma_max in the last cloud: NaN, as the reference
        sig[-1] = sigma_max + rng.uniform(0, 0.1, M)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    return dict(anc_kp=f(anc), pos_kp=f(pos), anc=f(desc[0]), pos=f(desc[1]), sigma=f(sig), draws=tuple(f(x) for x in u),
                radius=radius, gamma=0.3, sigma_max=sigma_max)


def _kernel_fwd(c):
    return ops.desc_cgf(c["anc_kp"], c["pos_kp"], c["anc"], c["pos"], c["sigma"], c["draws"], c["radius"], c["gamma"],
                        c["sigma_max"])


CGF_CASES = {
    # name: (B, M, D, special)
    "m40": (2, 40, 64, ("none", "all_in")),
    "m64_d128": (3, 64, 128, ("dup", "zero_draw")),
    "m512": (2, 512, 128, ("dup", "none", "all_in", "zero_draw")),
    "max_m": (2, ops.CGF_MAX_M, 64, ()),
    "nan_cloud": (2, 64, 64, ("nan",)),
    "b1": (1, 64, 128, ("none",)),
}


@pytest.mark.parametrize("case", list(CGF_CASES))
def test_cgf_forward_vs_restatement(case):
    B, M, D, special = CGF_CASES[case]
    c = _cgf_case(B, M, D, 11 + len(case), special=special)
    loss, active, (sel, aux, cloud) = _kernel_fwd(c)
    near, far, out, mask = cgf_ref.selections(c["anc_kp"], c["pos_kp"], c["draws"][0], c["draws"][1], c["radius"])
    torch.cuda.synchronize()
    s = sel.long()
    assert torch.equal(s[..., 0], near) and torch.equal(s[..., 1], far) and torch.equal(s[..., 2], out), case
    assert torch.equal((s[..., 3] & 1).bool(), mask), case
    assert torch.equal((s[..., 3] & 2).bool(), c["draws"][2] < 0.5), case
    if "none" in special:
        assert not bool(mask[0, 2]) and int(near[0, 2]) == 0
    if "all_in" in special:
        assert int(out[0, 1]) == 0
    if "zero_draw" in special:
        assert int(near[0, 3]) == 0 or bool(mask[0, 3])
    want_l, want_a = cgf_ref.cgf_loss(c["anc"], c["pos"], c["sigma"], near, far, out, mask, c["draws"][2], c["gamma"],
                                      c["sigma_max"])
    if "nan" in special:
        assert bool(torch.isnan(loss[-1]).all()) and bool(torch.isnan(want_l[-1]).all())
        loss, want_l = loss[:-1], want_l[:-1]
    assert bool(torch.isfinite(loss).all())
    e = float((loss - want_l).abs().max() / want_l.abs().max().clamp(min=1e-30))
    print("[cgf %s] loss rel err %.2e, anchors with a positive %d/%d" % (case, e, int(mask.sum()), mask.numel()))
    assert e <= CGF_REL, (case, e)
    assert float((active - want_a).abs().max()) <= 1e-6, (case, active, want_a)


@pytest.mark.parametrize("case", ["m40", "m64_d128", "m512", "nan_cloud"])
def test_cgf_backward_vs_float64(case):
    B, M, D, special = CGF_CASES[case]
    c = _cgf_case(B, M, D, 23 + len(case), special=special)
    _, _, saved = _kernel_fwd(c)
    g = torch.randn((B, M), generator=torch.Generator().manual_seed(M)).cuda()
    ga, gp = ops.desc_cgf_bwd(c["anc"], c["pos"], c["sigma"], saved, g, c["sigma_max"])
    ga2, gp2 = ops.desc_cgf_bwd(c["anc"], c["pos"], c["sigma"], saved, g, c["sigma_max"])
    torch.cuda.synchronize()
    bits = lambda t: t.view(torch.int32)                 # NaN-safe bit comparison
    assert torch.equal(bits(ga), bits(ga2)) and torch.equal(bits(gp), bits(gp2)), "the backward must be bit-reproducible"
    s = saved[0].long()
    a64 = c["anc"].double().requires_grad_(True)
    p64 = c["pos"].double().requires_grad_(True)
    l64, _ = cgf_ref.cgf_loss(a64, p64, c["sigma"].double(), s[..., 0], s[..., 1], s[..., 2], (s[..., 3] & 1).bool(),
                              c["draws"][2], c["gamma"], c["sigma_max"])
    (l64 * g.double()).sum().backward()
    for name, got, want in (("anc", ga, a64.grad), ("pos", gp, p64.grad)):
        if "nan" in special:                              # NaN reaches every gradient of that cloud, as in the reference
            assert torch.equal(torch.isnan(got[-1]), torch.isnan(want[-1]))
            got, want = got[:-1], want[:-1]
        e = float((got.double() - want).abs().max() / want.abs().max())
        print("[cgf_bwd %s] g_%s max|g-g64|/max|g64| %.2e" % (case, name, e))
        assert e <= 1e-5, (case, name, e)


def test_cgf_refusals():
    c = _cgf_case(2, 64, 64, 3)
    lib = _lib.load()
    p, s = ops._p, ops._stream()
    B, M, D = 2, 64, 64
    loss = torch.empty((B, M), device="cuda"); act = torch.empty(B, device="cuda")
    sel = torch.empty((B, M, 4), device="cuda", dtype=torch.int32); aux = torch.empty((B, M, 4), device="cuda")
    cl = torch.empty((B, 2), device="cuda")
    args = [p(c["anc_kp"]), p(c["pos_kp"]), p(c["anc"]), p(c["pos"]), p(c["sigma"]), *[p(u) for u in c["draws"]]]
    F = ctypes.c_float

    def fwd(a=args, M_=M, D_=D, sel_=sel):
        return lib.usip_desc_cgf_f32(*a, F(0.075), F(0.3), F(0.5), p(loss), p(act), p(sel_), p(aux), p(cl), B, M_, D_, s)
    assert fwd() == 0
    assert fwd(M_=ops.CGF_MAX_M + 1) != 0
    assert fwd(D_=66) != 0 and fwd(D_=ops.CGF_MAX_D + 4) != 0
    assert fwd(a=[None] + args[1:]) != 0
    sel_off = torch.empty(B * M * 4 + 1, device="cuda", dtype=torch.int32)[1:]
    assert fwd(sel_=sel_off) != 0
    assert "desc_cgf" in lib.usip_last_error().decode()
    assert lib.usip_desc_cgf_bwd(p(c["anc"]), p(c["pos"]), p(c["sigma"]), p(sel), p(aux), p(cl), p(loss), F(0.5), p(loss),
                                 p(loss), B, M, 66, s) != 0
    with pytest.raises(ValueError, match="multiple of 4"):
        ops.desc_cgf(c["anc_kp"], c["pos_kp"], c["anc"][:, :62].contiguous(), c["pos"][:, :62].contiguous(), c["sigma"],
                     c["draws"], 0.075, 0.3, 0.5)
    with pytest.raises(ValueError, match="contiguous"):
        ops.desc_cgf(c["anc_kp"], c["pos_kp"], c["anc"].transpose(1, 2).contiguous().transpose(1, 2), c["pos"], c["sigma"],
                     c["draws"], 0.075, 0.3, 0.5)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- network backward
def global_forward64(P, pins, x, sn, kp):
    """DescriptorLiteOldGlobal.forward, train mode (networks.py:433-479) in float64 at pinned decisions: the grouped
    PointNet, the global max over the M keypoints (pins["selg"] (B,D,1)), fc1 on cat(local, global), fc2, fc3, L2 norm."""
    M = kp.shape[2]
    perm = pins["perm"]
    xp = x[:, :, perm]
    x_aug = torch.cat([xp, sn[:, :, perm]], 1)
    local = ref64.group_net(P, pins, ref64.gather_groups(x_aug, kp, pins["idx"]), bn5=False)         # (B,D,M)
    glob = ref64.group_pool(pins, "selg", local, local, None, M)                                     # (B,D,1)
    h = ref64.layer(torch.cat([local, glob.expand(-1, -1, M)], 1), P, "fc1", pins)
    h = ref64.layer(h, P, "fc2", pins)
    out = ref64.layer(h, P, "fc3", pins, bn=False, act=False)
    return out / (torch.sqrt((out * out).sum(1, keepdim=True)) + 1e-5)


def _global_pins(ctx, x, sn, kp, perm, K, feats, radius):
    """Ball indices from the oracle on the permuted points (the plan's x_features must be exactly their gather), the plan's
    pools -- conv3 and conv5 over the whole ball, the global max over the keypoints -- and its ReLU active sets."""
    B, M = ctx["Bp"], ctx["M"]
    xp = np.ascontiguousarray(x[:, :, perm])
    idx = orc.ball_query_xyz(xp, kp, radius, K)
    x_aug = np.concatenate([xp, sn[:, :, perm]], 1)
    want = np.take_along_axis(x_aug, np.broadcast_to(idx.astype(np.int64).reshape(B, 1, M * K), (B, x_aug.shape[1], M * K)),
                              2).reshape(B, -1, M, K)
    want[:, :3] -= kp[:, :, :, None]
    assert np.array_equal(feats.cpu().numpy(), want), "x_features are not the gather of the oracle's balls"
    pins = ref64.Pins(perm=torch.from_numpy(perm).to(dev()), idx=torch.from_numpy(idx.astype(np.int64)).to(dev()),
                      sel3=_bcm(_sel(ctx["grp3"], ctx["bn3"]), B, M), sel5=_bcm(ctx["grp5"]["amax"].long(), B, M),
                      selg=ctx["glob_arg"].long().reshape(B, -1, 1), record={}, **_group_relus(ctx, B, M, K, conv5=False))
    pins["relu:fc1"] = _rows(_on(ctx["Y1f"], ctx["bn1f"]), B, M)
    pins["relu:fc2"] = _rows(_on(ctx["Y2f"], ctx["bn2f"]), B, M)
    return pins


def _global_net(opt, seed):
    from usip_b200.models import networks
    torch.manual_seed(seed)
    net = networks.DescriptorLiteOldGlobal(opt).to(dev())
    load_params(net, _desc_params(net, seed))
    net.train()
    return net


@pytest.mark.parametrize("use_tc", [False, True])
@pytest.mark.parametrize("K", [64, 192, 448])
def test_global_backward_every_element_vs_float64(K, use_tc):
    from usip_b200 import engine
    B, N, M, S, D, seed = 2, 2048, 64, 4, 128, 50 + K
    pc, sn, kp = dref.make_inputs(B, N, M, S, seed, half=1.0)
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=1.0, ball_nsamples=K,
                   descriptor_len=D, use_tensor_cores=use_tc)
    net = _global_net(opt, seed)
    perm = np.random.RandomState(seed).permutation(N)
    with torch.no_grad():
        desc, feats, ctx = engine.descriptor_global_forward(net, cu(pc), cu(sn), cu(kp), 0, cu(perm), use_tc=use_tc, keep=True)
        g_desc = torch.randn(tuple(desc.shape), generator=torch.Generator().manual_seed(K)).to(dev())
        grads = engine.descriptor_global_backward(net, ctx, g_desc)
    torch.cuda.synchronize()
    pins = _global_pins(ctx, pc, sn, kp, perm, K, feats, 1.0)
    P64 = ref64.params64(net.state_dict(), dev())
    desc64 = global_forward64(P64, pins, cu(pc).double(), cu(sn).double(), cu(kp).double())
    assert float((desc64.detach() - desc.double()).abs().max()) < 1e-5
    (desc64 * g_desc.double()).sum().backward()
    tag = "indoor descriptor K=%d use_tc=%s" % (K, use_tc)
    _check_pools(pins, pins.record, tag)
    _compare([(k, g) for (k, _), g in zip(net.named_parameters(), grads)], _grads64(P64), tag, "fp32", BOUND["fp32"])


# ----------------------------------------------------------------------------------------------- the train step
def _model(g, use_tc=True, **over):
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    B, N, M, S, K, D, seed = [int(v) for v in g["cfg"]]
    radius, cgf_radius, gamma, smax = [float(v) for v in g["radii"]]
    kw = dict(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=radius, ball_nsamples=K,
              descriptor_len=D, CGF_radius=cgf_radius, triple_loss_gamma=gamma, sigma_max=smax,
              random_pc_dropout_lower_limit=1.0, use_tensor_cores=use_tc)
    kw.update(over)
    opt = make_opt(**kw)
    md = ModelDescriptorIndoor(opt)
    load_params(md.descriptor, {k[len("param/"):]: g[k] for k in g.files if k.startswith("param/")})
    d = cgf_ref.train_inputs(B, N, M, S, seed, radius=cgf_radius)
    md.set_input(*[torch.from_numpy(d[k]) for k in cgf_ref.SET_INPUT_KEYS])
    return md, d, seed


def _stored_draws(md, g, tag):
    md.triplet_criteria.draws = lambda B, M, device: tuple(cu(g["%s/%s" % (tag, k)]) for k in ("u_near", "u_out", "u_sel"))


def _check_picks(md, g, tag):
    s = md.triplet_criteria.last_picks.long().cpu().numpy()
    for i, k in enumerate(("near", "far", "out")):
        assert np.array_equal(s[..., i], g["%s/%s" % (tag, k)]), (tag, k)


@pytest.mark.parametrize("use_tc", [False, True])
def test_optimize_vs_reference_cpu_golden(use_tc):
    """One ModelDescriptorIndoor.optimize() against the reference's own (CPU): picks, loss, active, descriptors,
    gradients and post-Adam parameters, in the format and bounds of test_gpu_detector's descriptor train step."""
    g = golden("descriptor_indoor_train.npz")
    md, _, seed = _model(g, use_tc)
    _stored_draws(md, g, "train")
    np.random.seed(seed)
    md.optimize(epoch=0)
    torch.cuda.synchronize()
    _check_picks(md, g, "train")
    assert abs(md.loss.item() - float(g["loss"])) <= REL * abs(float(g["loss"])), (md.loss.item(), float(g["loss"]))
    assert abs(md.active_percentage.item() - float(g["active"])) < 1e-6
    assert rel_err(md.anc_descriptors.detach().cpu().numpy(), g["anc_desc"]) < REL
    assert rel_err(md.pos_descriptors.detach().cpu().numpy(), g["pos_desc"]) < REL
    worst = 0.0
    for k, p in md.descriptor.named_parameters():
        ref = g["grad/" + k]
        gr = p.grad.detach().cpu().numpy().reshape(-1).astype(np.float64)
        absmax, norm = float(ref[2]), float(ref[3])
        wnorm = float(g["grad/" + k.replace("bias", "weight")][3]) if k.endswith("conv.bias") else norm
        if k.endswith("conv.bias") and norm < 1e-3 * max(wnorm, 1e-12):
            assert np.linalg.norm(gr) < 1e-3 * max(wnorm, 1e-12), k
            continue
        e_norm = abs(np.linalg.norm(gr) - norm) / max(norm, 1e-12)
        e_el = np.abs(gr[:24] - ref[4:4 + min(24, gr.size)]).max() / max(absmax, 1e-12)
        worst = max(worst, e_norm, e_el)
        assert e_norm < 2e-3 and e_el < 5e-3, (k, e_norm, e_el)
    for k, v in md.descriptor.state_dict().items():
        if k.endswith("num_batches_tracked"):
            continue
        ref = g["after/" + k]
        flat = v.cpu().numpy().reshape(-1)
        n = min(24, flat.size)
        diff = np.abs(flat[:n] - ref[3:3 + n])
        if "running" in k:
            assert diff.max() <= 1e-5 * max(np.abs(ref[3:3 + n]).max(), 1.0), (k, diff.max())
            continue
        assert diff.max() <= 2.2e-3, (k, diff.max())
        if k.endswith("conv.bias") and float(g["grad/" + k][3]) < 1e-3 * max(float(g["grad/" + k.replace("bias", "weight")][3]), 1e-12):
            continue
        gref = g["grad/" + k][4:]
        solid = np.abs(gref[:n]) > max(1e-5, 1e-2 * float(g["grad/" + k][2]))
        assert np.all(diff[solid] <= 2e-5 + 2e-4 * np.abs(ref[3:3 + n][solid])), (k, diff, gref[:n])
    print("[indoor optimize use_tc=%s vs reference (CPU)] loss %.6f, worst gradient rel err %.2e" % (use_tc, md.loss.item(),
                                                                                                    worst))


def test_optimize_grads_vs_float64():
    """p.grad of optimize() against float64 autograd of the restated network and DescCGFLoss, the network decisions from
    a keep=True forward on the same inputs and parameters, the loss picks from the step itself (checked against the
    restatement's selections on the step's draws)."""
    from usip_b200 import engine
    g = golden("descriptor_indoor_train.npz")
    md, d, seed = _model(g)
    B, M, K = md.opt.batch_size, md.opt.node_num, md.opt.ball_nsamples
    sd0 = {k: v.clone() for k, v in md.descriptor.state_dict().items()}
    x = np.concatenate([d["anc_pc"], d["pos_pc"]]); sn = np.concatenate([d["anc_sn"], d["pos_sn"]])
    kp = np.concatenate([d["anc_kp"], d["pos_kp"]])
    perm = np.random.RandomState(seed).permutation(x.shape[2])
    net = md.descriptor
    net.train()
    with torch.no_grad():
        desc, feats, ctx = engine.descriptor_global_forward(net, cu(x), cu(sn), cu(kp), 0, cu(perm), use_tc=True, keep=True)
    pins = _global_pins(ctx, x, sn, kp, perm, K, feats, md.opt.ball_radius)
    desc0 = desc.clone()
    del ctx
    md.descriptor.load_state_dict(sd0)
    _stored_draws(md, g, "train")
    np.random.seed(seed)
    md.optimize(epoch=0)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([md.anc_descriptors, md.pos_descriptors]).detach(), desc0), "the step saw other descriptors"
    s = md.triplet_criteria.last_picks.long()
    u = [cu(g["train/" + k]) for k in ("u_near", "u_out", "u_sel")]
    near, far, out, mask = cgf_ref.selections(md.anc_keypoints_transformed, md.pos_keypoints, u[0], u[1], md.opt.CGF_radius)
    assert torch.equal(s[..., 0], near) and torch.equal(s[..., 1], far) and torch.equal(s[..., 2], out)
    P64 = ref64.params64(sd0, dev())
    desc64 = global_forward64(P64, pins, cu(x).double(), cu(sn).double(), cu(kp).double())
    l64, _ = cgf_ref.cgf_loss(desc64[:B], desc64[B:], md.anc_sigmas.double(), near, far, out, mask, u[2],
                              md.opt.triple_loss_gamma, md.opt.sigma_max)
    loss64 = l64.mean()
    assert abs(md.loss.item() - loss64.item()) <= 1e-5 * abs(loss64.item()), (md.loss.item(), loss64.item())
    loss64.backward()
    tag = "ModelDescriptorIndoor.optimize"
    _check_pools(pins, pins.record, tag)
    _compare([(k, p.grad) for k, p in md.descriptor.named_parameters()], _grads64(P64), tag, "fp32", STEP_BOUND)


def test_test_model_eval_bn_and_no_update():
    g = golden("descriptor_indoor_train.npz")
    md, _, seed = _model(g)
    sd0 = {k: v.clone() for k, v in md.descriptor.state_dict().items()}
    _stored_draws(md, g, "test")
    np.random.seed(seed + 1)
    md.test_model()
    torch.cuda.synchronize()
    assert not md.descriptor.training
    for k, v in md.descriptor.state_dict().items():
        assert torch.equal(v, sd0[k]), k
    # the golden's test_model ran after its optimize() step: only its picks are comparable from the initial parameters
    _check_picks(md, g, "test")
    # from the golden's post-step parameters is not stored whole; the loss is checked on a model that took the same step
    md2, _, _ = _model(g)
    _stored_draws(md2, g, "train")
    np.random.seed(seed)
    md2.optimize(epoch=0)
    _stored_draws(md2, g, "test")
    np.random.seed(seed + 1)
    md2.test_model()
    torch.cuda.synchronize()
    assert abs(md2.loss.item() - float(g["test_loss"])) <= REL * abs(float(g["test_loss"])), (md2.loss.item(), float(g["test_loss"]))
    assert abs(md2.active_percentage.item() - float(g["test_active"])) < 1e-6


def test_training_runs_and_learning_rate():
    g = golden("descriptor_indoor_train.npz")
    md, d, seed = _model(g, random_pc_dropout_lower_limit=0.8)
    p0 = [p.detach().clone() for p in md.descriptor.parameters()]
    torch.cuda.manual_seed(seed)
    for step in range(4):
        if step:                                          # point dropout thinned the staged batch: stage it again
            with pytest.raises(ValueError, match="set_input"):
                md.optimize(epoch=step)
            md.set_input(*[torch.from_numpy(d[k]) for k in cgf_ref.SET_INPUT_KEYS])
        md.optimize(epoch=step)
        torch.cuda.synchronize()
        assert math.isfinite(md.loss.item()) and 0.0 <= md.active_percentage.item() <= 1.0
        assert all(bool(torch.isfinite(p.grad).all()) for p in md.descriptor.parameters())
    moved = sum(int(not torch.equal(a, b.detach())) for a, b in zip(p0, md.descriptor.parameters()))
    assert moved >= len(p0) - 6, moved                   # the zero-gradient conv biases in front of BatchNorm stay
    errs = md.get_current_errors()
    assert set(errs) == {"O_loss", "O_triplet", "O_active_perc", "E_loss", "E_triplet", "E_active_perc"}
    lr = md.old_lr_descriptor
    md.update_learning_rate(0.5)
    assert md.old_lr_descriptor == lr * 0.5 and md.optimizer_descriptor.param_groups[0]["lr"] == lr * 0.5
    with pytest.raises(NotImplementedError):
        md.get_current_visuals()


# ----------------------------------------------------------------------------------------------- SceneNN's training shape
FULL = dict(B=2, N=5000, M=512, S=4, K=448, D=128, seed=7, radius=0.75, cgf_radius=0.075, gamma=0.3, sigma_max=0.5)
NGRAD = 4096


def full_setup():
    """The SceneNN training shape: inputs (tests/cgf_ref.train_inputs) and parameters (this repo's module, seeded, with
    randomized BatchNorm affines); tools/make_gpu_golden.py gives the reference the same state."""
    from usip_b200.models import networks
    c = FULL
    d = cgf_ref.train_inputs(c["B"], c["N"], c["M"], c["S"], c["seed"], radius=c["cgf_radius"])
    opt = make_opt(batch_size=c["B"], input_pc_num=c["N"], node_num=c["M"], surface_normal_len=c["S"], ball_radius=c["radius"],
                   ball_nsamples=c["K"], descriptor_len=c["D"], CGF_radius=c["cgf_radius"], triple_loss_gamma=c["gamma"],
                   sigma_max=c["sigma_max"], random_pc_dropout_lower_limit=1.0)
    torch.manual_seed(c["seed"])
    state = dref.randomized_params(networks.DescriptorLiteOldGlobal(opt), c["seed"])
    return opt, d, state


def grad_sample(name, n):
    from tests.util_gpu import sample_idx
    return sample_idx(n, NGRAD, sum(map(ord, name)) % 1000)


def test_optimize_full_size_vs_reference_gpu():
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    g = golden("reference_descriptor_indoor_train.npz")
    opt, d, state = full_setup()
    md = ModelDescriptorIndoor(opt)
    md.descriptor.load_state_dict(state)
    md.set_input(*[torch.from_numpy(d[k]) for k in cgf_ref.SET_INPUT_KEYS])
    torch.cuda.manual_seed(FULL["seed"])
    np.random.seed(FULL["seed"])
    md.optimize(epoch=0)
    torch.cuda.synchronize()
    s = md.triplet_criteria.last_picks.long().cpu().numpy()
    for i, k in enumerate(("near", "far", "out")):
        assert np.array_equal(s[..., i], g[k]), k
    e_loss = abs(md.loss.item() - float(g["loss32"])) / abs(float(g["loss64"]))
    e_ref = abs(float(g["loss32"]) - float(g["loss64"])) / abs(float(g["loss64"]))
    print("[indoor optimize, SceneNN shape] loss %.6f (reference %.6f), rel err %.2e (reference fp32 vs fp64 %.2e)" % (
        md.loss.item(), float(g["loss32"]), e_loss, e_ref))
    assert e_loss <= max(REL, 10 * e_ref)
    assert abs(md.active_percentage.item() - float(g["active"])) < 1e-6
    worst = 0.0
    for k, p in md.descriptor.named_parameters():
        gr = p.grad.detach().cpu().numpy().reshape(-1).astype(np.float64)
        g64 = g["g64__" + k]
        scale = float(g["gscale__" + k])
        if scale == 0.0:                                   # a conv bias in front of BatchNorm: true gradient 0
            continue
        e = np.abs(gr[grad_sample(k, gr.size)] - g64).max() / scale
        band = max(5e-4, 10 * float(g["eref__" + k]))     # DESIGN section 2: within ten times the reference's own error
        worst = max(worst, e)
        assert e <= band, (k, e, band)
    print("   worst sampled gradient error %.2e of max|g64|" % worst)
