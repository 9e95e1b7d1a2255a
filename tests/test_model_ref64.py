"""Anchors tests/model_ref64.py -- the float64 autograd restatement the GPU gradient tests compare against -- to the
reference: at the golden shapes, with the decisions derived on the CPU (oracle.som_assign / oracle.knn, float64 arg-max
and arg-min elsewhere), it must reproduce the oracle's train-mode forward and every gradient summary the reference wrote
(tools/make_golden.py: loss, norm, absmax and the first 24 elements of each parameter gradient).  CPU only."""
import numpy as np
import pytest
import torch

from oracle import usip_oracle as orc
from tests import model_ref64 as ref64
from tests.util_gpu import golden

FWD_REL = 1e-4            # keypoints / sigmas / descriptors / loss vs the oracle and the golden loss

# Gradient tolerances per fixture: (norm, absmax, first 24 elements), each relative to the reference's |g|max except the
# norm.  The reference ran in float32, so it differs from float64 wherever its float32 forward flips a near-tied arg-max;
# the fixtures with more such pools per channel show more of it.  Measured worst (norm, absmax, elements):
#   kitti 2.0e-4 6.5e-4 5.5e-4 | modelnet 5.5e-4 2.2e-3 3.1e-3 | lite 2.1e-6 4.7e-6 1.0e-5
#   ablation knn 1.5e-3 7.4e-3 7.7e-3 | ablation ball 2.4e-4 1.3e-3 8.1e-3 | descriptor 4.8e-7 2.1e-6 1.7e-6
# The golden train-step tests allow 2e-3 (norm) and 5e-3 (elements), 3e-3 and 3e-2 for the ablation networks.
TOL = {"detector_kitti_small.npz": (5e-4, 1.5e-3, 1.5e-3), "detector_modelnet_small.npz": (1e-3, 4e-3, 5e-3),
       "detector_lite_small.npz": (1e-4, 1e-4, 1e-4), "knn": (3e-3, 1.5e-2, 1.5e-2), "ball": (1e-3, 3e-3, 1.5e-2),
       "descriptor": (1e-5, 1e-5, 1e-5)}


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.float64)


def _check_grads(P64, ref_of, fails, tag):
    """Compare every parameter's autograd gradient with the golden summary [mean, std, absmax, norm, first 24]."""
    worst = 0.0
    for k, v in P64.items():
        if not v.requires_grad:
            continue
        ref = ref_of(k)
        gr = v.grad.numpy().reshape(-1)
        absmax, norm = float(ref[2]), float(ref[3])
        wkey = k.replace("conv.bias", "conv.weight")
        if k.endswith("conv.bias") and norm < 1e-3 * float(ref_of(wkey)[3]):
            # a bias whose constant shift the next BatchNorm removes: gradient 0 (the reference holds rounding noise)
            assert np.linalg.norm(gr) < 1e-9 * float(ref_of(wkey)[3]) + 1e-12, (tag, k, np.linalg.norm(gr))
            continue
        e_norm = abs(np.linalg.norm(gr) - norm) / norm
        e_abs = abs(np.abs(gr).max() - absmax) / absmax
        e_el = np.abs(gr[:24] - ref[4:4 + min(24, gr.size)]).max() / absmax
        worst = max(worst, e_norm, e_abs, e_el)
        t_norm, t_abs, t_el = TOL[tag]
        if not (e_norm < t_norm and e_abs < t_abs and e_el < t_el):
            fails.append((tag, k, e_norm, e_abs, e_el))
    return worst


def _rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("fname", ["detector_kitti_small.npz", "detector_modelnet_small.npz", "detector_lite_small.npz"])
def test_detector_restatement_reproduces_reference_train_step(fname):
    g = golden(fname)
    B, N, M, S, Kn, seed = [int(v) for v in g["cfg"]]
    kind, scene = str(g["kind"]), str(g["scene"])
    lb, alpha = float(g["lb"]), float(g["alpha"])
    d = orc.synth_pair(B, N, M, S, kind=kind, seed=seed)
    C1, C2 = (64, 256) if scene == "indoor" else (128, 512)
    P = orc.init_detector_params(S=S, seed=seed, C1=C1, C2=C2, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    x = np.concatenate([d["src_pc"], d["dst_pc"]]); sn = np.concatenate([d["src_sn"], d["dst_sn"]])
    node = np.concatenate([d["src_node"], d["dst_node"]])
    pins = ref64.cpu_detector_pins(x, node, Kn)
    P64 = ref64.params64(P)
    _, kp, sig = ref64.detector_forward(P64, pins, _t(x), _t(sn), _t(node), lb)
    loss, _ = ref64.detector_loss(pins, kp, sig, _t(d["src_pc"]), _t(d["dst_pc"]), _t(d["R"]), _t(d["scale"]),
                                  _t(d["shift"]), alpha)
    loss.backward()
    r = orc.detector_fwd_loss(P, d["src_pc"], d["src_sn"], d["src_node"], d["dst_pc"], d["dst_sn"], d["dst_node"],
                              d["R"], d["scale"], d["shift"], node_knn_k=Kn, sigma_lower_bound=lb, alpha=alpha, training=True)
    e_kp = _rel(kp.detach().numpy(), np.concatenate([r["src_keypoints"], r["dst_keypoints"]]))
    e_sig = _rel(sig.detach().numpy(), np.concatenate([r["src_sigmas"], r["dst_sigmas"]]))
    assert e_kp < FWD_REL and e_sig < FWD_REL, (e_kp, e_sig)
    assert abs(loss.item() - float(r["loss"])) <= FWD_REL * abs(float(r["loss"])), (loss.item(), float(r["loss"]))
    assert abs(loss.item() - float(g["train_loss"][0])) <= FWD_REL * abs(float(g["train_loss"][0]))
    fails = []
    worst = _check_grads(P64, lambda k: g["grad/" + k], fails, fname)
    print("%s: worst gradient summary error %.2e" % (fname, worst))
    assert not fails, fails


@pytest.mark.parametrize("mode", ["knn", "ball"])
def test_ablation_restatement_reproduces_reference_gradients(mode):
    g = golden("detector_ablation.npz")
    B, N, M, S, Kn, seed = [int(v) for v in g["cfg"]]
    d = orc.ablation_inputs(seed, B, N, M, S)
    P = orc.init_ablation_params(S=S, seed=seed, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    if mode == "knn":
        idx, _ = orc.knn(d["node"], d["pc"], 64)
    else:
        idx = orc.ball_query_xyz(d["pc"], d["node"], 2.0, 64)
    knn_i, _ = orc.knn(d["node"], d["node"], Kn)
    pins = ref64.Pins(idx=torch.from_numpy(idx.astype(np.int64)), knn_i=torch.from_numpy(knn_i.astype(np.int64)),
                      strict=False)
    P64 = ref64.params64(P)
    kp, sig = ref64.ablation_forward(P64, pins, _t(d["pc"]), _t(d["sn"]), _t(d["node"]), 1e-3)
    loss = (kp * _t(d["w_kp"])).sum() + (sig * _t(d["w_sig"])).sum()
    loss.backward()
    r = orc.ablation_forward(P, d["pc"], d["sn"], d["node"], mode=mode, node_knn_k=Kn, training=True)
    assert _rel(kp.detach().numpy(), r["keypoints"]) < FWD_REL and _rel(sig.detach().numpy(), r["sigmas"]) < FWD_REL
    assert _rel(kp.detach().numpy(), g[mode + "/train_kp"]) < FWD_REL
    assert abs(loss.item() - float(g[mode + "/loss"])) <= 2e-4 * abs(float(g[mode + "/loss"]))
    fails = []
    worst = _check_grads(P64, lambda k: g[mode + "/grad/" + k], fails, mode)
    print("ablation %s: worst gradient summary error %.2e" % (mode, worst))
    assert not fails, fails


def test_descriptor_restatement_reproduces_reference_train_step():
    g = golden("descriptor_train.npz")
    B, N, M, S, K, seed = [int(v) for v in g["cfg"]]
    d = orc.desc_train_inputs(B, N, M, S, seed)
    P = {k[len("param/"):]: g[k] for k in g.files if k.startswith("param/")}
    perm = np.random.RandomState(seed).permutation(N)          # the one np.random.permutation(N) of the siamese forward
    x = np.concatenate([d["anc_pc"], d["pos_pc"]]); sn = np.concatenate([d["anc_sn"], d["pos_sn"]])
    kp = np.concatenate([d["anc_kp"], d["pos_kp"]])
    idx = orc.ball_query_xyz(np.ascontiguousarray(x[:, :, perm]), kp, 1.0, K)
    pins = ref64.Pins(perm=torch.from_numpy(perm), idx=torch.from_numpy(idx.astype(np.int64)), strict=False)
    P64 = ref64.params64(P)
    desc = ref64.descriptor_forward(P64, pins, _t(x), _t(sn), _t(kp))
    loss, active = ref64.descriptor_train_loss(pins, desc, torch.from_numpy(d["neg_idx"]), _t(d["anc_sigma"]))
    loss.backward()
    r = orc.descriptor_forward(P, x, sn, kp, radius=1.0, nsamples=K, training=True, permute_idx=perm)
    assert _rel(desc.detach().numpy(), r["descriptor"]) < FWD_REL
    assert _rel(desc.detach().numpy()[:B], g["anc_desc"]) < FWD_REL and _rel(desc.detach().numpy()[B:], g["pos_desc"]) < FWD_REL
    assert abs(loss.item() - float(g["loss"])) <= FWD_REL * abs(float(g["loss"])), (loss.item(), float(g["loss"]))
    assert abs(active.item() - float(g["active"])) < 1e-6
    fails = []
    worst = _check_grads(P64, lambda k: g["grad/" + k], fails, "descriptor")
    print("descriptor: worst gradient summary error %.2e" % worst)
    assert not fails, fails


def test_point_on_surface_restatement_vs_reference_gradient():
    """point_to_plane keypoint-on-cloud loss: value and the reference's gradient of 0.37 * mean(loss) (losses.npz)."""
    g = golden("losses.npz")
    B, M = g["kp"].shape[0], g["kp"].shape[2]
    kp = _t(g["kp"]).requires_grad_(True)
    pins = ref64.Pins(strict=False)
    ls = ref64.point_on_surface(pins, "i", kp, _t(g["pc"]), _t(g["sn4"]))
    (0.37 * ls.mean()).backward()
    assert _rel(ls.detach().numpy(), g["on_surface"].reshape(B, M)) < 1e-5
    assert _rel(kp.grad.numpy(), g["g_kp_surface"]) < 1e-5


def test_pins_are_arguments():
    """A strict Pins refuses to derive: the GPU comparison can only run on decisions it was given."""
    pins = ref64.Pins(knn_i=torch.zeros((1, 4, 2), dtype=torch.long))
    with pytest.raises(KeyError):
        ref64.detector_forward({}, pins, torch.zeros((1, 3, 8), dtype=torch.float64), None,
                               torch.zeros((1, 3, 4), dtype=torch.float64), 1e-3)
