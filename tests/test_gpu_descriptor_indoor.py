"""-m gpu: the indoor descriptor DescriptorLiteOldGlobal (448-sample balls, PPFNet global context) and its new kernel.

  * usip_group_max_combine against torch's amax / amin over a reshaped view, bit for bit, and its refusals;
  * the network against the reference run on the CPU (tests/golden/descriptor_indoor.npz) and on the GPU at the indoor
    evaluation shape (tests/golden/reference_descriptor_indoor.npz, tools/make_gpu_golden.py): x_features bit-exact,
    descriptors 1e-4 relative, running statistics after a train-mode forward 1e-5;
  * K = 64 (direct group max), 192 and 448 (64-row sub-groups combined) against a float64 restatement;
  * IndoorRegistration.describe with a ModelDescriptorIndoor loaded from checkpoints.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import desc_indoor_ref as dref
from tests.util_gpu import cu, golden, make_opt, rel_err, sample_idx
from usip_b200 import _lib, ops

pytestmark = pytest.mark.gpu
REL, REL_RUN = 1e-4, 1e-5
NDESC = 16384


@pytest.mark.parametrize("ratio", [1, 7, 37, 512])
@pytest.mark.parametrize("C", [128, 256, 36])
@pytest.mark.parametrize("with_min", [True, False])
def test_group_max_combine_bit_exact(ratio, C, with_min):
    g = torch.Generator(device="cuda").manual_seed(ratio * 1000 + C)
    for Q in (1, 5, 333):
        gmax = torch.randn((Q * ratio, C), device="cuda", generator=g)
        gmin = torch.randn((Q * ratio, C), device="cuda", generator=g) if with_min else None
        if ratio > 1:
            gmax[1::ratio] = gmax[0::ratio]                 # exact ties inside every group
            gmax[:ratio, :4] = -float("inf")                # a group that is -inf throughout
        omax, omin = ops.group_max_combine(gmax, ratio, gmin)
        torch.cuda.synchronize()
        assert torch.equal(omax, gmax.view(Q, ratio, C).amax(1)), (Q, ratio, C)
        if with_min:
            assert torch.equal(omin, gmin.view(Q, ratio, C).amin(1))
        else:
            assert omin is None


def test_group_max_combine_refusals():
    lib = _lib.load()
    x = torch.zeros((64, 128), device="cuda")
    p = ops._p
    s = ops._stream()
    assert lib.usip_group_max_combine(p(x), None, p(x), None, 0, 4, 128, s) != 0
    assert lib.usip_group_max_combine(p(x), None, p(x), None, 4, 0, 128, s) != 0
    assert lib.usip_group_max_combine(p(x), None, p(x), None, 4, 4, 0, s) != 0
    assert lib.usip_group_max_combine(p(x), p(x), p(x), None, 4, 4, 128, s) != 0          # gmin without out_min
    assert lib.usip_group_max_combine(None, None, p(x), None, 4, 4, 128, s) != 0
    assert lib.usip_group_max_combine(p(x), None, p(x), None, 1, 1, 128 * 65536, s) != 0   # too many column slabs
    assert "group_max_combine" in lib.usip_last_error().decode()
    with pytest.raises(ValueError):
        ops.group_max_combine(x, 5)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- the network
def _net(B, N, M, S, K, D, radius=0.75, state=None, seed=0):
    from usip_b200.models.networks import DescriptorLiteOldGlobal
    opt = make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=radius, ball_nsamples=K,
                   descriptor_len=D)
    if state is None:
        torch.manual_seed(seed)
        state = dref.randomized_params(DescriptorLiteOldGlobal(opt), seed)
    net = DescriptorLiteOldGlobal(opt).cuda()
    net.load_state_dict(state)
    for p in net.parameters():
        p.requires_grad_(False)
    return net


def _run(net, x, s, k, seed):
    """(descriptor, x_features, running statistics) of an eval then a train forward, each after np.random.seed(seed)."""
    out = {}
    for mode in ("eval", "train"):
        net.train(mode == "train")
        np.random.seed(seed)
        desc, feats = net(x, s, k, mode == "train", None)
        out[mode + "_desc"], out[mode + "_feats"] = desc, feats
    out["run"] = {k: v.detach().clone() for k, v in net.state_dict().items() if "running" in k}
    return out


def test_descriptor_vs_reference_cpu_golden():
    g = golden("descriptor_indoor.npz")
    B, N, M, S, K, seed = [int(v) for v in g["cfg"]]
    state = {k[len("param/"):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param/")}
    net = _net(B, N, M, S, K, int(g["D"]), float(g["radius"]), state=state)
    o = _run(net, cu(g["pc"]), cu(g["sn"]), cu(g["kp"]), seed)
    want = dref.reconstruct_features(g["pc"], g["sn"], g["kp"], g["idx"].astype(np.int64), g["perm"])
    for mode in ("eval", "train"):
        f = o[mode + "_feats"].cpu().numpy()
        assert np.array_equal(f, want), "x_features must be the reference's ball groups bit for bit"
        assert np.array_equal(f.ravel()[dref.feats_sample(f.size)], g["feats"])
        e = rel_err(o[mode + "_desc"].cpu().numpy(), g[mode + "_desc"])
        print("[indoor descriptor %s-BN vs reference (CPU)] rel err %.2e" % (mode, e))
        assert e < REL, (mode, e)
    for k, v in o["run"].items():
        e = rel_err(v.cpu().numpy(), g["after/" + k])
        assert e < REL_RUN, (k, e)


FULL = dict(B=4, N=10240, M=512, S=4, K=448, D=128, seed=5)


def full_setup():
    """The indoor evaluation shape (N=10240, M=512, K=448, radius 0.75): inputs and the parameters of this repo's module,
    seeded (tools/make_gpu_golden.py builds the reference network from the same state)."""
    c = FULL
    pc, sn, kp = dref.make_inputs(c["B"], c["N"], c["M"], c["S"], c["seed"], half=1.5)
    from usip_b200.models.networks import DescriptorLiteOldGlobal
    opt = make_opt(batch_size=c["B"], input_pc_num=c["N"], node_num=c["M"], surface_normal_len=c["S"], ball_radius=0.75,
                   ball_nsamples=c["K"], descriptor_len=c["D"])
    torch.manual_seed(c["seed"])
    state = dref.randomized_params(DescriptorLiteOldGlobal(opt), c["seed"])
    return opt, (pc, sn, kp), state


def sampled(desc, feats):
    desc, feats = np.asarray(desc).ravel(), np.asarray(feats).ravel()
    return desc[sample_idx(desc.size, NDESC, 7)], feats[dref.feats_sample(feats.size)]


def test_descriptor_full_size_vs_reference_gpu():
    c = FULL
    _, (pc, sn, kp), state = full_setup()
    g = golden("reference_descriptor_indoor.npz")
    net = _net(c["B"], c["N"], c["M"], c["S"], c["K"], c["D"], state=state)
    o = _run(net, cu(pc), cu(sn), cu(kp), c["seed"])
    for mode in ("eval", "train"):
        d, f = sampled(o[mode + "_desc"].cpu().numpy(), o[mode + "_feats"].cpu().numpy())
        assert np.array_equal(f, g["feats_" + mode]), "x_features must be bit-identical"
        e = rel_err(d, g["desc_" + mode])
        print("[indoor descriptor %s-BN, full size, vs reference (GPU)] rel err %.2e" % (mode, e))
        assert e < REL, (mode, e)
    for k, v in o["run"].items():
        e = rel_err(v.cpu().numpy(), g["run__" + k])
        print("   %-32s rel err %.2e" % (k, e))
        assert e < REL_RUN, (k, e)


@pytest.mark.parametrize("K", [64, 192, 448])
def test_descriptor_vs_float64_restatement(K):
    B, N, M, S, D, seed = 2, 2048, 64, 4, 128, 17 + K
    pc, sn, kp = dref.make_inputs(B, N, M, S, seed, half=1.0)
    net = _net(B, N, M, S, K, D, seed=seed)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    o = _run(net, cu(pc), cu(sn), cu(kp), seed)
    for mode in ("eval", "train"):
        ref, run = dref.forward64(sd, o[mode + "_feats"], mode == "train")
        e = rel_err(o[mode + "_desc"].cpu().numpy(), ref.cpu().numpy())
        print("[K=%d %s-BN vs float64] rel err %.2e" % (K, mode, e))
        assert e < REL, (K, mode, e)
    for k, v in run.items():
        e = rel_err(o["run"][k].cpu().numpy(), v.cpu().numpy())
        assert e < REL_RUN, (K, k, e)


def test_grouped_pointnet_sub_groups_forward_only():
    """K above 128 has no arg outputs across the combine: the train step of DescriptorLiteOld keeps refusing it."""
    from usip_b200.models.networks import DescriptorLiteOld
    with pytest.raises(NotImplementedError):
        DescriptorLiteOld(make_opt(ball_nsamples=448))


# ----------------------------------------------------------------------------------------------- evaluation
def test_indoor_registration_describe_from_checkpoints(tmp_path):
    from tests.test_gpu_indoor_registration import SCENE, _room_tree
    from usip_b200.evaluation import indoor_registration as idr
    from usip_b200.evaluation import registration as reg
    from usip_b200.evaluation.repeatability import load_detector_checkpoint
    from usip_b200.models.keypoint_descriptor import ModelDescriptorIndoor
    from usip_b200.models.keypoint_detector import ModelDetector
    npy, gt, _, _, _ = _room_tree(str(tmp_path))
    opt = reg.descriptor_opt("redwood", input_pc_num=1024, node_num=128, batch_size=4)
    torch.manual_seed(0)
    det_path, des_path = str(tmp_path / "det.pth"), str(tmp_path / "des.pth")
    torch.save({"module." + k: v for k, v in ModelDetector(opt).detector.state_dict().items()}, det_path)
    torch.save(dref.randomized_params(ModelDescriptorIndoor(opt).descriptor, 9), des_path)

    def describe():
        det, des = ModelDetector(opt), ModelDescriptorIndoor(opt)
        load_detector_checkpoint(det, det_path)
        reg.load_descriptor_checkpoint(des, des_path)
        ev = idr.IndoorRegistration.redwood(npy, gt, opt, scenes=[(SCENE, 6)], seed=4)
        ev.describe(det, des, L=128)
        return ev, des

    ev, des = describe()
    res = ev.score([64, 128], [1000], pairs="all", seed=3)
    assert len(res.per_scene[SCENE]["pairs"]) == 15
    ev2, _ = describe()
    r = ev.ev
    assert torch.equal(r.descriptors, ev2.ev.descriptors), "same seed, same descriptors"
    assert torch.isfinite(r.descriptors).all()
    # the descriptors are a direct run_model on the clouds the detector saw, at all M keypoints
    direct = torch.empty_like(r.descriptors)
    seeded = reg._SeededNumpy(des, r.source.seed)
    for items, (pc, sn, _) in r.source.batches(0.0):
        direct[items[0]:items[-1] + 1] = seeded.run_model(pc, sn, r.keypoints[items[0]:items[-1] + 1])
    assert torch.equal(direct, r.descriptors)
    np.testing.assert_array_equal(ev.desc.cpu().numpy()[0, :3],
                                  r.descriptors[0, :, r.order[0, :3].long()].t().cpu().numpy())
