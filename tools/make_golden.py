"""Generate tests/golden/*.npz by RUNNING THE REFERENCE (lijx10/USIP at /root/reference, unmodified) on CPU
through oracle/ref_shim.py.  Only runs in the build container (the reference is not shipped); the outputs are
small, committed, and are what pins oracle/ (tests/test_oracle_vs_golden.py) and the CUDA path
(tests/test_gpu_*.py) to the reference.

Inputs are regenerated from seeds by oracle.usip_oracle.{synth_pair,init_detector_params}, so the fixtures only
hold outputs (+ tiny inputs where no generator exists).

    python tools/make_golden.py
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, usip_oracle as orc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def load_params(module, P):
    sd = module.state_dict()
    for k in sd:
        assert k in P, k
        sd[k] = torch.from_numpy(np.asarray(P[k])).reshape(sd[k].shape).to(sd[k].dtype)
    module.load_state_dict(sd)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def golden_index_max(ref):
    import index_max as im  # the shimmed module -> reference C++ forward_cpu
    rng = np.random.default_rng(7)
    cases = {}
    # (a) generic, (b) duplicates/ties, (c) empty clusters + values <= -1000, (d) B*K beyond the reference smem cap
    specs = dict(a=(2, 8, 1000, 16), b=(2, 4, 512, 8), c=(2, 4, 300, 32), d=(30, 2, 700, 512))
    for name, (B, C, N, K) in specs.items():
        data = rng.normal(size=(B, C, N)).astype(np.float32)
        index = rng.integers(0, K, size=(B, N)).astype(np.int32)
        if name == "b":
            data = np.round(data * 2) / 2          # many exact ties
        if name == "c":
            index = rng.integers(0, K // 2, size=(B, N)).astype(np.int32)   # upper half empty
            data[:, 0, :] = -2000.0                                        # never above the -1000 floor
            data[:, 1, ::3] = -1000.0
        out = im.forward_cpu(t(data), t(index), K).numpy()
        cases["data_" + name] = data; cases["index_" + name] = index; cases["out_" + name] = out
        cases["K_" + name] = np.int32(K)
    np.savez_compressed(os.path.join(OUT, "index_max.npz"), **cases)


def golden_query_topk(ref):
    out = {}
    for name, (B, N, M, kind, seed) in dict(lidar=(2, 2048, 64, "lidar", 11), obj=(3, 1500, 32, "object", 12)).items():
        d = orc.synth_pair(B, N, M, 4 if kind == "lidar" else 3, kind=kind, seed=seed)
        node = d["src_node"].copy()
        if name == "obj":
            node[:, :, 5] = node[:, :, 4]          # duplicated node -> exact distance ties
            node[:, :, 9] = 100.0                  # far away node -> empty cluster
        mask, row_max, min_idx = ref.som.query_topk(t(node), t(d["src_pc"]), M, 1)
        out["node_" + name] = node; out["seed_" + name] = np.int32(seed)
        out["min_idx_" + name] = min_idx.numpy().astype(np.int32)
        out["row_max_" + name] = row_max.numpy().astype(np.int32)
    np.savez_compressed(os.path.join(OUT, "query_topk.npz"), **out)


def golden_losses(ref):
    torch.manual_seed(1234 + 0)
    B, M = 2, 256                                   # BASELINE.json configs[0]
    src = torch.randn(B, 3, M); dst = torch.randn(B, 3, M)
    ss = torch.rand(B, M) + 0.01; sd = torch.rand(B, M) + 0.01
    opt = ref_shim.make_opt()
    crit = ref.losses.ChamferLoss_Brute(opt)
    a = src.clone().requires_grad_(True); b = dst.clone().requires_grad_(True)
    sa = ss.clone().requires_grad_(True); sb = sd.clone().requires_grad_(True)
    loss, pure, weighted = crit(a, b, sa, sb)
    loss.backward()
    out = dict(src=src.numpy(), dst=dst.numpy(), sig_src=ss.numpy(), sig_dst=sd.numpy(),
               loss=loss.detach().numpy(), pure=pure.numpy(), weighted=weighted.numpy(),
               g_src=a.grad.numpy(), g_dst=b.grad.numpy(), g_sig_src=sa.grad.numpy(), g_sig_dst=sb.grad.numpy())
    # single side
    kp = torch.randn(B, 3, 64); pc = torch.randn(B, 3, 700)
    kpg = kp.clone().requires_grad_(True)
    ssc = ref.losses.SingleSideChamferLoss_Brute(opt)(kpg, pc)
    ssc.mean().backward()
    out.update(kp=kp.numpy(), pc=pc.numpy(), single=ssc.detach().numpy(), g_kp=kpg.grad.numpy())
    # point_to_plane (PointOnSurfaceLoss through KeypointOnPCLoss): value + gradient w.r.t. the keypoints
    sn = torch.nn.functional.normalize(torch.randn(B, 3, 700), dim=1)
    sn4 = torch.cat([sn, torch.rand(B, 1, 700)], 1)              # S=4: only the first three channels are the normal
    kpp = kp.clone().requires_grad_(True)
    pos = ref.losses.KeypointOnPCLoss(opt)(kpp, pc, sn4)
    (pos.mean() * 0.37).backward()
    out.update(sn4=sn4.numpy(), on_surface=pos.detach().numpy(), g_kp_surface=kpp.grad.numpy())
    # no-sigma branch
    l2, p2, w2 = crit(src, dst)
    out.update(nosigma=l2.numpy())
    np.savez_compressed(os.path.join(OUT, "losses.npz"), **out)


def detector_case(ref, name, B, N, M, S, Kn, kind, seed, scene="outdoor", lb=1e-3, alpha=0.01):
    d = orc.synth_pair(B, N, M, S, kind=kind, seed=seed)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, node_knn_k_1=Kn,
                            scene=scene, loss_sigma_lower_bound=lb, keypoint_on_pc_alpha=alpha)
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    md = ref.keypoint_detector.ModelDetector(opt)
    C1, C2 = (64, 256) if scene == "indoor" else (128, 512)
    P = orc.init_detector_params(S=S, seed=seed, C1=C1, C2=C2, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)   # make keypoint offsets non-trivial
    load_params(md.detector, P)
    out = dict(cfg=np.array([B, N, M, S, Kn, seed], np.int64), kind=kind, scene=scene,
               lb=np.float32(lb), alpha=np.float32(alpha))
    args = [t(d[k]) for k in ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")]
    md.set_input(*args)
    # --- eval forward + loss
    md.test_model()
    out.update(eval_kp=torch.cat([md.src_keypoints, md.dst_keypoints]).detach().numpy(),
               eval_sig=torch.cat([md.src_sigmas, md.dst_sigmas]).detach().numpy(),
               eval_node=torch.cat([md.src_node_recomputed, md.dst_node_recomputed]).detach().numpy(),
               eval_loss=np.array([md.loss.item(), md.loss_chamfer.item(), md.chamfer_pure.item(),
                                   md.chamfer_weighted.item(), md.loss_keypoint_on_pc_src.item(),
                                   md.loss_keypoint_on_pc_dst.item()], np.float32))
    # --- one training step (train-mode BN forward, backward, Adam)
    md.optimize(epoch=0)
    out.update(train_kp=torch.cat([md.src_keypoints, md.dst_keypoints]).detach().numpy(),
               train_sig=torch.cat([md.src_sigmas, md.dst_sigmas]).detach().numpy(),
               train_loss=np.array([md.loss.item(), md.loss_chamfer.item(), md.chamfer_pure.item(),
                                    md.chamfer_weighted.item(), md.loss_keypoint_on_pc_src.item(),
                                    md.loss_keypoint_on_pc_dst.item()], np.float32))
    sd = md.detector.state_dict()
    for k, v in sd.items():
        v = v.detach().numpy()
        if k.endswith("num_batches_tracked"):
            out["nbt/" + k] = v
            continue
        flat = v.reshape(-1).astype(np.float64)
        out["after/" + k] = np.concatenate([[flat.mean(), flat.std(), np.abs(flat).max()], flat[:24]]).astype(np.float32)
    grads = {}
    for k, p in md.detector.named_parameters():
        g = p.grad.detach().numpy().reshape(-1).astype(np.float64)
        grads["grad/" + k] = np.concatenate([[g.mean(), g.std(), np.abs(g).max(), np.linalg.norm(g)], g[:24]]).astype(np.float32)
    out.update(grads)
    np.savez_compressed(os.path.join(OUT, "detector_%s.npz" % name), **out)
    print("detector", name, "eval loss", out["eval_loss"], "train loss", out["train_loss"])


def golden_descriptor(ref):
    B, N, M, S, K = 2, 2048, 48, 4, 32
    seed = 21
    rng = np.random.default_rng(seed)
    d = orc.synth_pair(B, N, 16, S, kind="lidar", seed=seed)
    pc = d["src_pc"] * np.array([0.2, 1.0, 0.2], np.float32).reshape(1, 3, 1)      # denser cloud: balls get 0..>K hits
    sel = rng.choice(N, M, replace=False)
    kp = (pc[:, :, sel] + rng.normal(0, 0.1, (B, 3, M))).astype(np.float32)
    kp[:, :, 0] = 500.0                                                             # a keypoint with zero hits
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=1.0,
                            ball_nsamples=K, descriptor_len=128)
    torch.manual_seed(seed)
    net = ref.networks.DescriptorLiteOld(opt)
    out = dict(cfg=np.array([B, N, M, S, K, seed], np.int64), pc=pc, sn=d["src_sn"], kp=kp)
    sdn = {k: v.detach().numpy().copy() for k, v in net.state_dict().items()}
    for k, v in sdn.items():
        out["param/" + k] = v
    for mode in ("eval", "train"):
        net.train(mode == "train")
        np.random.seed(seed)                               # the forward consumes np.random.permutation(N)
        perm = np.random.RandomState(seed).permutation(N)  # same stream, recorded for the consumers
        np.random.seed(seed)
        with torch.no_grad():
            desc, feats = net(t(pc), t(d["src_sn"]), t(kp), mode == "train", None)
        out[mode + "_desc"] = desc.numpy(); out[mode + "_feats"] = feats.numpy()
        out["perm"] = perm.astype(np.int64)
    np.savez_compressed(os.path.join(OUT, "descriptor.npz"), **out)


def golden_descriptor_indoor(ref):
    """DescriptorLiteOldGlobal (models/networks.py:388-479) on the CPU, with tests/desc_indoor_ref.py supplying the
    operations.ball_query_wrapper the reference ships commented out: eval and train BatchNorm, the running statistics
    after the train forward, the ball indices and a fixed sample of x_features."""
    from tests import desc_indoor_ref as dref
    B, N, M, S, K, seed, D, radius = 2, 2048, 64, 4, 448, 81, 64, 0.75
    pc, sn, kp = dref.make_inputs(B, N, M, S, seed, half=1.0)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=radius,
                            ball_nsamples=K, descriptor_len=D)
    torch.manual_seed(seed)
    params = dref.randomized_params(ref.networks.DescriptorLiteOldGlobal(opt), seed)
    case = dict(cfg=np.array([B, N, M, S, K, seed], np.int64), radius=np.float32(radius), D=np.int64(D), pc=pc, sn=sn,
                kp=kp, **{"param/" + k: v.numpy() for k, v in params.items()})
    out = dref.reference_outputs(ref, _NpzLike(case))
    assert np.array_equal(out["eval_feats"], out["train_feats"])
    perm = np.random.RandomState(seed).permutation(N)
    dist = np.linalg.norm(kp[:, :, :, None] - pc[:, :, perm][:, :, None, :], axis=1)
    idx = orc.ball_query_dist(np.ascontiguousarray(dist, dtype=np.float32), radius, K)
    assert np.array_equal(dref.reconstruct_features(pc, sn, kp, idx, perm), out["eval_feats"])
    hits = (dist <= np.float32(radius)).sum(2)
    print("descriptor_indoor: ball hits min %d median %d max %d (K=%d)" % (hits.min(), np.median(hits), hits.max(), K))
    case.update(perm=perm.astype(np.int64), idx=idx.astype(np.int16),
                feats=out["eval_feats"].ravel()[dref.feats_sample(out["eval_feats"].size)], eval_desc=out["eval_desc"], train_desc=out["train_desc"],
                **{k: v for k, v in out.items() if k.startswith("after/")})
    np.savez_compressed(os.path.join(OUT, "descriptor_indoor.npz"), **case)


class _NpzLike(dict):
    @property
    def files(self):
        return list(self.keys())


def golden_descriptor_train(ref):
    """One ModelDescriptor.optimize() of the reference (keypoint_descriptor.py:126-157) on CPU: loss, gradient
    summaries, post-Adam parameter summaries.  Inputs are regenerated from the seed by the consumers."""
    B, N, M, S, K = 3, 2048, 40, 4, 32
    seed = 33
    d = desc_train_inputs(B, N, M, S, seed)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=1.0,
                            ball_nsamples=K, descriptor_len=128, random_pc_dropout_lower_limit=1.0)
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    md = ref.keypoint_descriptor.ModelDescriptor(opt)
    out = dict(cfg=np.array([B, N, M, S, K, seed], np.int64))
    for k, v in md.descriptor.state_dict().items():
        out["param/" + k] = v.detach().numpy().copy()
    md.set_input(*[t(d[k]) for k in ("anc_pc", "anc_sn", "anc_kp", "anc_sigma", "pos_pc", "pos_sn", "pos_kp", "pos_sigma")],
                 torch.from_numpy(d["neg_idx"]))
    np.random.seed(seed)                                   # the forward consumes np.random.permutation(N)
    md.optimize(epoch=0)
    out["loss"] = np.float32(md.loss.item()); out["active"] = np.float32(md.active_percentage.item())
    out["anc_desc"] = md.anc_descriptors.detach().numpy(); out["pos_desc"] = md.pos_descriptors.detach().numpy()
    for k, p in md.descriptor.named_parameters():
        g = p.grad.detach().numpy().reshape(-1).astype(np.float64)
        out["grad/" + k] = np.concatenate([[g.mean(), g.std(), np.abs(g).max(), np.linalg.norm(g)], g[:24]]).astype(np.float32)
    for k, v in md.descriptor.state_dict().items():
        v = v.detach().numpy()
        if k.endswith("num_batches_tracked"):
            continue
        flat = v.reshape(-1).astype(np.float64)
        out["after/" + k] = np.concatenate([[flat.mean(), flat.std(), np.abs(flat).max()], flat[:24]]).astype(np.float32)
    np.savez_compressed(os.path.join(OUT, "descriptor_train.npz"), **out)
    print("descriptor train loss", out["loss"], "active", out["active"])


INDOOR_TRAIN = dict(B=2, N=2048, M=64, S=4, K=448, D=128, seed=91, radius=0.75, cgf_radius=0.075, gamma=0.3, sigma_max=0.5)


def golden_descriptor_indoor_train(ref):
    """One ModelDescriptorIndoor.optimize() and one test_model() of the reference (keypoint_descriptor.py:451-519) on the
    CPU, with tests/desc_indoor_ref.py supplying ball_query_wrapper: the three torch.rand draws of each DescCGFLoss call,
    the picks (the index arguments of its three torch.gather calls), per-anchor loss and active share, the descriptors,
    gradient and post-Adam parameter summaries (descriptor_train.npz's format).  Inputs: tests/cgf_ref.train_inputs."""
    from tests import cgf_ref
    from tests import desc_indoor_ref as dref
    c = INDOOR_TRAIN
    B, N, M, S, K, D, seed = (c[k] for k in ("B", "N", "M", "S", "K", "D", "seed"))
    d = cgf_ref.train_inputs(B, N, M, S, seed, radius=c["cgf_radius"])
    dref.install(ref)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, ball_radius=c["radius"],
                            ball_nsamples=K, descriptor_len=D, random_pc_dropout_lower_limit=1.0,
                            CGF_radius=c["cgf_radius"], triple_loss_gamma=c["gamma"], sigma_max=c["sigma_max"])
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    md = ref.keypoint_descriptor.ModelDescriptorIndoor(opt)
    out = dict(cfg=np.array([B, N, M, S, K, D, seed], np.int64),
               radii=np.array([c["radius"], c["cgf_radius"], c["gamma"], c["sigma_max"]], np.float64))
    for k, v in md.descriptor.state_dict().items():
        out["param/" + k] = v.detach().numpy().copy()
    md.set_input(*[t(d[k]) for k in cgf_ref.SET_INPUT_KEYS])
    crit = md.triplet_criteria.forward

    def recording(tag):
        def forward(*a, **k):
            draws, picks = [], []
            rand, gather = torch.rand, torch.gather

            def rec_rand(*ra, **rk):
                draws.append(rand(*ra, **rk)); return draws[-1]

            def rec_gather(x, dim, index, *ga, **gk):
                picks.append(index.squeeze(2)); return gather(x, dim, index, *ga, **gk)
            torch.rand, torch.gather = rec_rand, rec_gather
            try:
                loss, active = crit(*a, **k)
            finally:
                torch.rand, torch.gather = rand, gather
            assert len(draws) == 3 and len(picks) == 3
            for name, v in zip(("u_near", "u_out", "u_sel"), draws):
                out["%s/%s" % (tag, name)] = v.numpy()
            for name, v in zip(("near", "far", "out"), picks):
                out["%s/%s" % (tag, name)] = v.numpy().astype(np.int16)
            out[tag + "/anc_kp_t"] = a[0].detach().numpy()
            out[tag + "/loss_vec"] = loss.detach().numpy(); out[tag + "/active_vec"] = active.detach().numpy()
            return loss, active
        return forward
    md.triplet_criteria.forward = recording("train")
    np.random.seed(seed)                                   # the forward consumes np.random.permutation(N)
    md.optimize(epoch=0)
    out["loss"] = np.float32(md.loss.item()); out["active"] = np.float32(md.active_percentage.item())
    out["anc_desc"] = md.anc_descriptors.detach().numpy(); out["pos_desc"] = md.pos_descriptors.detach().numpy()
    for k, p in md.descriptor.named_parameters():
        g = p.grad.detach().numpy().reshape(-1).astype(np.float64)
        out["grad/" + k] = np.concatenate([[g.mean(), g.std(), np.abs(g).max(), np.linalg.norm(g)], g[:24]]).astype(np.float32)
    for k, v in md.descriptor.state_dict().items():
        v = v.detach().numpy()
        if k.endswith("num_batches_tracked"):
            continue
        flat = v.reshape(-1).astype(np.float64)
        out["after/" + k] = np.concatenate([[flat.mean(), flat.std(), np.abs(flat).max()], flat[:24]]).astype(np.float32)
    md.triplet_criteria.forward = recording("test")
    np.random.seed(seed + 1)
    md.test_model()
    out["test_loss"] = np.float32(md.loss.item()); out["test_active"] = np.float32(md.active_percentage.item())
    print("descriptor_indoor_train: loss %.6f active %.4f, test loss %.6f, anchors with a positive %d of %d" % (
        out["loss"], out["active"], out["test_loss"], int(cgf_ref.selections(
            t(out["train/anc_kp_t"]), t(d["pos_kp"]), t(out["train/u_near"]), t(out["train/u_out"]),
            c["cgf_radius"])[3].sum()), B * M))
    np.savez_compressed(os.path.join(OUT, "descriptor_indoor_train.npz"), **out)


def desc_train_inputs(B, N, M, S, seed):
    """Synthetic (anchor, positive) scan pair with keypoints + sigmas for the descriptor train step (shared with the
    tests through oracle.usip_oracle.desc_train_inputs)."""
    return orc.desc_train_inputs(B, N, M, S, seed)


def golden_desc_loss(ref):
    torch.manual_seed(5)
    B, C, M = 3, 128, 40
    anc = torch.nn.functional.normalize(torch.randn(B, C, M), dim=1)
    pos = torch.nn.functional.normalize(anc + 0.3 * torch.randn(B, C, M), dim=1)
    neg_idx = torch.tensor([1, 2, 0])
    sig = torch.rand(B, M) * 4
    opt = ref_shim.make_opt()
    loss, act = ref.losses.DescPairScanLoss(opt)(anc, pos, anc[neg_idx], sig)
    np.savez_compressed(os.path.join(OUT, "desc_loss.npz"), anc=anc.numpy(), pos=pos.numpy(), neg_idx=neg_idx.numpy(),
                        sig=sig.numpy(), loss=loss.numpy(), active=act.numpy(),
                        gamma=np.float32(opt.triple_loss_gamma), sigma_max=np.float32(opt.sigma_max))


def golden_fps(ref):
    """FarthestSampler of the reference's KITTI loader (float64 distances, np.argmax) on three small clouds: lidar-like,
    a cloud with duplicated points (exact ties) and k larger than the number of distinct points."""
    import importlib
    loader = importlib.import_module("data.kitti_detector_loader")
    fs = loader.FarthestSampler()
    out = {}
    rng = np.random.default_rng(31)
    clouds = dict(lidar=(rng.uniform(-40, 40, (700, 3)) * np.array([1, 0.05, 1])).astype(np.float32),
                  dup=np.repeat(rng.normal(size=(60, 3)).astype(np.float32), 5, axis=0),
                  few=np.repeat(rng.normal(size=(5, 3)).astype(np.float32), 4, axis=0))
    for name, pts in clouds.items():
        k = dict(lidar=64, dup=48, few=12)[name]
        np.random.seed(77)
        nodes = fs.sample(pts, k)                       # consumes np.random.randint(len(pts)) for the first node
        np.random.seed(77)
        start = np.random.randint(len(pts))
        out["pts_" + name] = pts; out["k_" + name] = np.int32(k); out["start_" + name] = np.int32(start)
        out["nodes_" + name] = nodes
    np.savez_compressed(os.path.join(OUT, "fps.npz"), **out)


def golden_ablation(ref):
    """RPN_Detector_KNN / RPN_Detector_Ball (models/networks.py:482-738): eval and train forward, and the gradients of
    L = sum(w_kp * keypoints) + sum(w_sig * sigmas) (ModelDetector cannot select these networks -- the lines are commented
    out at keypoint_detector.py:23-24 -- so the fixture drives the networks directly)."""
    B, N, M, S, Kn, seed = 2, 4096, 128, 4, 16, 1239          # 256 groups per channel: one flipped arg-max moves a sum by < 1 %
    d = orc.ablation_inputs(seed, B, N, M, S)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S, node_knn_k_1=Kn)
    P = orc.init_ablation_params(S=S, seed=seed, randomize_bn=True)
    P["mlp3.conv.weight"] = (P["mlp3.conv.weight"] * 1000).astype(np.float32)
    out = dict(cfg=np.array([B, N, M, S, Kn, seed], np.int64))
    for mode, cls in (("knn", ref.networks.RPN_Detector_KNN), ("ball", ref.networks.RPN_Detector_Ball)):
        torch.manual_seed(seed)
        net = cls(opt)
        load_params(net, P)
        net.eval()
        with torch.no_grad():
            node_o, kp, sig, _ = net(t(d["pc"]), t(d["sn"]), t(d["node"]), False, None)
        assert torch.equal(node_o, t(d["node"]))
        out[mode + "/eval_kp"] = kp.numpy(); out[mode + "/eval_sig"] = sig.numpy()
        net.train()
        _, kp, sig, _ = net(t(d["pc"]), t(d["sn"]), t(d["node"]), True, 0)
        loss = (kp * t(d["w_kp"])).sum() + (sig * t(d["w_sig"])).sum()
        net.zero_grad()
        loss.backward()
        out[mode + "/train_kp"] = kp.detach().numpy(); out[mode + "/train_sig"] = sig.detach().numpy()
        out[mode + "/loss"] = np.float32(loss.item())
        for k, p_ in net.named_parameters():
            g = p_.grad.detach().numpy().reshape(-1).astype(np.float64)
            out[mode + "/grad/" + k] = np.concatenate([[g.mean(), g.std(), np.abs(g).max(), np.linalg.norm(g)], g[:24]]).astype(np.float32)
        for k, v in net.state_dict().items():
            if k.endswith("running_mean") or k.endswith("running_var"):
                out[mode + "/after/" + k] = v.detach().numpy().reshape(-1)[:24].copy()
        print("ablation", mode, "loss", out[mode + "/loss"])
    np.savez_compressed(os.path.join(OUT, "detector_ablation.npz"), **out)


def _reference_function(relpath, name):
    """The reference's own, unmodified source of one top-level function, executed here (its module cannot be imported:
    evaluation/save_keypoints.py is a script with hard-coded dataset paths and GUI / visdom imports)."""
    import ast
    src = open(os.path.join(ref_shim.build_ref_root(), relpath)).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == name)
    ns = {"np": np}
    exec(compile(ast.Module(body=[node], type_ignores=[]), relpath, "exec"), ns)
    return ns[name]


def golden_nms(ref):
    """evaluation/save_keypoints.py:180-216 nms() + the sigma-sorted top-k that follows it (:346-351)."""
    nms = _reference_function("evaluation/save_keypoints.py", "nms")
    rng = np.random.default_rng(41)
    out = {}
    cases = dict(lidar=(rng.uniform(-40, 40, (512, 3)) * np.array([1, 0.05, 1]), 2.0),
                 dense=(rng.normal(size=(300, 3)) * 1.5, 1.0),
                 ties=(np.round(rng.normal(size=(200, 3)) * 2) / 2, 0.5),       # duplicated positions, exact distance ties
                 off=(rng.normal(size=(64, 3)), 0.0))                            # radius < 0.01: pass-through
    for name, (kp, r) in cases.items():
        kp = kp.astype(np.float32)
        sg = (rng.uniform(0.01, 2.0, kp.shape[0])).astype(np.float32)
        if name == "ties":
            sg = np.round(sg * 4) / 4                                            # equal sigmas too
            sg = sg.astype(np.float32)
        vk, vs = nms(kp.copy(), sg.copy(), r)
        out["kp_" + name] = kp; out["sigma_" + name] = sg; out["radius_" + name] = np.float32(r)
        out["valid_kp_" + name] = vk; out["valid_sigma_" + name] = vs
    np.savez_compressed(os.path.join(OUT, "nms.npz"), **out)


# data/kitti_detector_loader.py KittiLoader.__getitem__ on a synthetic KITTI tree (usip_b200.data.kitti_detector_loader.
# write_synthetic_kitti): train sequences 0..8, test sequences 9..10, every scan (PAIRS_NS, 8) float32.
PAIRS_COUNTS = [2, 1, 1, 1, 1, 1, 1, 1, 2, 1, 2]
PAIRS_NS, PAIRS_TREE_SEED = 1300, 7100
PAIRS_CASES = {     # name: (mode, index, np seed, S, rot_horizontal, rot_3d, rot_perturbation, translation, radius)
    "kitti": ("train", 3, 11, 4, 1, 0, 0, 0, 100.0),
    "s1": ("train", 0, 12, 1, 1, 0, 0, 0, 100.0),
    "s5": ("train", 10, 13, 5, 1, 0, 0, 0, 100.0),
    "rot3d": ("train", 5, 14, 3, 0, 1, 1, 1, 100.0),
    "radius": ("train", 1, 15, 4, 1, 0, 0, 0, 20.0),
    "test": ("test", 2, 16, 4, 1, 0, 0, 0, 100.0),
}


def golden_pairs(ref):
    import importlib
    import tempfile
    from usip_b200.data.kitti_detector_loader import write_synthetic_kitti
    kl = importlib.import_module("data.kitti_detector_loader")
    out = {"tree/counts": np.array(PAIRS_COUNTS), "tree/Ns": np.int64(PAIRS_NS), "tree/seed": np.int64(PAIRS_TREE_SEED),
           "N": np.int64(1024), "M": np.int64(64)}
    keys = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
    with tempfile.TemporaryDirectory() as root:
        write_synthetic_kitti(root, PAIRS_COUNTS, PAIRS_NS, seed=PAIRS_TREE_SEED)
        for name, (mode, index, seed, S, rh, r3, rp, tp, radius) in PAIRS_CASES.items():
            opt = ref_shim.make_opt(input_pc_num=1024, node_num=64, surface_normal_len=S, rot_horizontal=bool(rh),
                                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp),
                                    radius_threshold=radius)
            loader = kl.KittiLoader(root, mode, opt)
            np.random.seed(seed)
            res = loader[index]
            out[name + "/case"] = np.array([index, seed, S, rh, r3, rp, tp], dtype=np.int64)
            out[name + "/mode"] = np.array(mode)
            out[name + "/radius"] = np.float64(radius)
            for k, v in zip(keys, res):
                out[name + "/" + k] = np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32)
            print("pairs", name, {k: out[name + "/" + k].shape for k in keys})
    np.savez_compressed(os.path.join(OUT, "detector_pairs.npz"), **out)


# data/kitti_descriptor_loader.py KittiDescriptorLoader.__getitem__ + mine_negative_sample on a synthetic KITTI tree with
# a pose trajectory: sequence 0 is 40 scans 1.5 m apart along a gently turning path (positives within 5 m, scans more
# than 50 m apart), the other sequences a few scans each.  Every scan is (DESC_NS, 8) float32.
DESC_COUNTS = [40, 3, 2, 2, 2, 2, 2, 2, 3, 3, 3]
DESC_NS, DESC_TREE_SEED, DESC_N, DESC_M = 700, 7200, 512, 32
DESC_CASES = {     # name: (mode, anchors, np/random seed, S, rot_horizontal, rot_3d, rot_perturbation, translation)
    "kitti": ("train", [3, 41, 17, 44], 21, 4, 1, 0, 0, 0),
    "s1": ("train", [40, 7, 52, 30], 22, 1, 1, 0, 0, 0),
    "s5": ("train", [22, 5, 20, 39], 23, 5, 1, 0, 0, 0),       # anchors 0 and 2 have no negative in this batch
    "rot3d": ("train", [12, 45, 48, 0], 24, 3, 0, 1, 1, 1),
    "test": ("test", [0, 4, 2, 5], 25, 4, 1, 0, 0, 0),
}


def desc_trajectory(counts):
    """poses[seq][i] (4, 4) float64: sequence s runs along a heading that turns 1 degree per scan, 1.5 m per scan,
    from an offset of 1000 m * s."""
    poses = []
    for s, n in enumerate(counts):
        ps, pos, yaw = [], np.array([1000.0 * s, 0.0, 0.0]), 0.3 * s
        for i in range(n):
            c, si = np.cos(yaw), np.sin(yaw)
            P = np.eye(4)
            P[:3, :3] = [[c, 0, si], [0, 1, 0], [-si, 0, c]]
            P[:3, 3] = pos
            ps.append(P)
            pos = pos + 1.5 * np.array([si, 0.0, c])
            yaw += np.pi / 180
        poses.append(ps)
    return poses


def golden_descpairs(ref):
    import importlib
    import tempfile
    from torch.utils.data.dataloader import default_collate
    from usip_b200.data.kitti_detector_loader import write_synthetic_kitti
    kl = importlib.import_module("data.kitti_descriptor_loader")
    poses = desc_trajectory(DESC_COUNTS)
    out = {"tree/counts": np.array(DESC_COUNTS), "tree/Ns": np.int64(DESC_NS), "tree/seed": np.int64(DESC_TREE_SEED),
           "tree/poses": np.concatenate([np.stack(p) for p in poses if p]), "N": np.int64(DESC_N), "M": np.int64(DESC_M)}
    keys = ("anc_pc", "anc_sn", "anc_node", "anc_seq", "anc_pose", "pos_pc", "pos_sn", "pos_node", "pos_seq", "pos_pose")
    with tempfile.TemporaryDirectory() as root:
        write_synthetic_kitti(root, DESC_COUNTS, DESC_NS, seed=DESC_TREE_SEED, poses=poses)
        for name, (mode, anchors, seed, S, rh, r3, rp, tp) in DESC_CASES.items():
            opt = ref_shim.make_opt(input_pc_num=DESC_N, node_num=DESC_M, surface_normal_len=S, rot_horizontal=bool(rh),
                                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp),
                                    positive_radius_threshold=5.0, negative_radius_threshold=50.0)
            loader = kl.KittiDescriptorLoader(root, mode, opt)
            np.random.seed(seed)
            random.seed(seed)
            batch = default_collate([loader[i] for i in anchors])
            neg_idx = loader.mine_negative_sample(batch[3], batch[4], opt.negative_radius_threshold)
            out[name + "/case"] = np.array([seed, S, rh, r3, rp, tp], dtype=np.int64)
            out[name + "/anchors"] = np.array(anchors, dtype=np.int64)
            out[name + "/mode"] = np.array(mode)
            for k, v in zip(keys, batch):
                out[name + "/" + k] = v.numpy()
            out[name + "/neg_idx"] = neg_idx.numpy()
            print("descpairs", name, "pos_seq", out[name + "/pos_seq"], "neg_idx", out[name + "/neg_idx"])
    np.savez_compressed(os.path.join(OUT, "descriptor_pairs.npz"), **out)
    print("descriptor_pairs.npz", os.path.getsize(os.path.join(OUT, "descriptor_pairs.npz")) // 1024, "KB")


# data/modelnet_shrec_loader.py ModelNet_Shrec_Loader.__getitem__ (dataset 'modelnet') on a synthetic ModelNet tree
# (usip_b200.data.modelnet_shrec_loader.write_synthetic_modelnet): every object (MN_ROWS, 6) float32.  One case builds two
# items in a row from one seed, so a batch of two pairs with its per-pair jitter is pinned too.
MN_SHAPES, MN_TRAIN, MN_TEST, MN_ROWS, MN_TREE_SEED, MN_N, MN_M = ("airplane", "night_stand", "cup"), 2, 1, 2000, 7300, 1000, 64
MN_CASES = {        # name: (mode, items, np seed, rot_horizontal, rot_3d, rot_perturbation, translation)
    "rot3d": ("train", [4, 1], 31, 0, 1, 0, 0),                 # modelnet/options_detector.py defaults
    "horizontal": ("train", [2], 32, 1, 0, 0, 1),
    "allrot": ("train", [5], 33, 1, 1, 1, 1),                   # the transform drops the perturbation
    "norot": ("train", [0], 34, 0, 0, 0, 1),                    # pc and sn stay float32
    "test": ("test", [2], 35, 0, 1, 0, 0),
}


def golden_modelnet_pairs(ref):
    import importlib
    import tempfile
    from usip_b200.data.modelnet_shrec_loader import write_synthetic_modelnet
    ml = importlib.import_module("data.modelnet_shrec_loader")
    out = {"tree/shapes": np.array(MN_SHAPES), "tree/counts": np.array([MN_TRAIN, MN_TEST]),
           "tree/rows": np.int64(MN_ROWS), "tree/seed": np.int64(MN_TREE_SEED), "N": np.int64(MN_N), "M": np.int64(MN_M)}
    keys = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
    with tempfile.TemporaryDirectory() as root:
        write_synthetic_modelnet(root, MN_SHAPES, MN_TRAIN, MN_TEST, MN_ROWS, seed=MN_TREE_SEED)
        for name, (mode, items, seed, rh, r3, rp, tp) in MN_CASES.items():
            opt = ref_shim.make_opt(dataset="modelnet", classes=40, input_pc_num=MN_N, node_num=MN_M,
                                    surface_normal_len=3, rot_horizontal=bool(rh), rot_3d=bool(r3),
                                    rot_perturbation=bool(rp), translation_perturbation=bool(tp))
            loader = ml.ModelNet_Shrec_Loader(root, mode, opt)
            np.random.seed(seed)
            res = [loader[i] for i in items]
            out[name + "/case"] = np.array([seed, rh, r3, rp, tp], dtype=np.int64)
            out[name + "/items"] = np.array(items, dtype=np.int64)
            out[name + "/mode"] = np.array(mode)
            for k, vals in zip(keys, zip(*res)):
                out[name + "/" + k] = np.stack([np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32)
                                                for v in vals])
            print("modelnet_pairs", name, {k: out[name + "/" + k].shape for k in keys})
    np.savez_compressed(os.path.join(OUT, "modelnet_pairs.npz"), **out)
    print("modelnet_pairs.npz", os.path.getsize(os.path.join(OUT, "modelnet_pairs.npz")) // 1024, "KB")


# data/match3d_detector_loader.py Match3DDetectorLoader.__getitem__ and data/scenenn_detector_loader.py
# SceneNNDetectorLoader.__getitem__ on synthetic trees (usip_b200.data.match3d_detector_loader.write_synthetic_3dmatch_train,
# scenenn_detector_loader.write_synthetic_scenenn), every fragment a (rows, 7) synthetic_fragment.  The 3DMatch
# loader lists folders with os.listdir, so every item is recorded by its path relative to the tree's root.  One
# SceneNN case runs a train item and then a val item from one seed: the mixed batch of scenenn/train_detector.py.
IN_N, IN_M, IN_SEED = 1024, 64, 7500
IN_M3_LAYOUT = {"train": {"kitchen": {"seq-01": 3, "seq-02": 2}, "office": {"seq-01": 2}},
                "test": {"lab": {"seq-01": 2}}}
IN_M3_ROWS = [1500, 1500, 700, 1500, 1500, 1500, 1500, 1500, 1500]      # file i in listing order; file 2 < N
IN_M3_CASES = {     # name: (mode, relative paths, np seed, S, rot_horizontal, rot_3d, rot_perturbation, translation)
    "m3_default": ("train", ["kitchen/seq-01/2.npy", "office/seq-01/0.npy"], 61, 4, 0, 1, 0, 0),   # options defaults
    "m3_horizontal": ("train", ["kitchen/seq-02/1.npy"], 62, 4, 1, 0, 1, 1),
    "m3_s3": ("train", ["kitchen/seq-01/0.npy"], 63, 3, 0, 1, 0, 0),
    "m3_test": ("test", ["lab/seq-01/1.npy"], 64, 4, 0, 1, 0, 0),
}
IN_SN_COUNTS = {"train": 3, "val": 2, "test": 2}
IN_SN_CASES = {     # name: ([(split, item)], np seed); scenenn/options_detector.py defaults (S 4, rot_3d)
    "sn_train": ([("train", 1)], 71),                  # train item 1 has fewer than N rows
    "sn_val": ([("val", 0)], 72),
    "sn_test": ([("test", 1)], 73),
    "sn_mixed": ([("train", 2), ("val", 1)], 74),
}


def indoor_scenenn_rows(split, i):
    return 600 if (split, i) == ("train", 1) else 1300


def golden_indoor_pairs(ref):
    import importlib
    import tempfile
    from usip_b200.data.match3d_detector_loader import write_synthetic_3dmatch_train
    from usip_b200.data.scenenn_detector_loader import write_synthetic_scenenn
    m3 = importlib.import_module("data.match3d_detector_loader")
    sn = importlib.import_module("data.scenenn_detector_loader")
    keys = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
    out = {"N": np.int64(IN_N), "M": np.int64(IN_M), "tree/seed": np.int64(IN_SEED),
           "m3/layout": np.array(["%s/%s/%s/%d" % (split, scene, sub, n) for split, scenes in IN_M3_LAYOUT.items()
                                  for scene, subs in scenes.items() for sub, n in subs.items()]),
           "m3/rows": np.array(IN_M3_ROWS, dtype=np.int64),
           "sn/counts": np.array([IN_SN_COUNTS[k] for k in ("train", "val", "test")], dtype=np.int64)}

    def store(name, res):
        for k, vals in zip(keys, zip(*res)):
            out[name + "/" + k] = np.stack([np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32)
                                            for v in vals])
        print("indoor_pairs", name, {k: out[name + "/" + k].shape for k in keys})

    with tempfile.TemporaryDirectory() as root:
        write_synthetic_3dmatch_train(root, IN_M3_LAYOUT, lambda i: IN_M3_ROWS[i], seed=IN_SEED)
        for name, (mode, rel, seed, S, rh, r3, rp, tp) in IN_M3_CASES.items():
            opt = ref_shim.make_opt(input_pc_num=IN_N, node_num=IN_M, surface_normal_len=S, rot_horizontal=bool(rh),
                                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp))
            loader = m3.Match3DDetectorLoader(root, mode, opt)
            listed = [os.path.relpath(p, root) for p in loader.dataset]
            np.random.seed(seed)
            store(name, [loader[listed.index(r)] for r in rel])
            out[name + "/case"] = np.array([seed, S, rh, r3, rp, tp], dtype=np.int64)
            out[name + "/paths"] = np.array(rel)
            out[name + "/mode"] = np.array(mode)
    with tempfile.TemporaryDirectory() as root:
        write_synthetic_scenenn(root, IN_SN_COUNTS, indoor_scenenn_rows, seed=IN_SEED)
        opt = ref_shim.make_opt(input_pc_num=IN_N, node_num=IN_M, surface_normal_len=4, rot_horizontal=False,
                                rot_3d=True, rot_perturbation=False, translation_perturbation=False)
        loaders = {split: sn.SceneNNDetectorLoader(root, split, opt) for split in IN_SN_COUNTS}
        for name, (items, seed) in IN_SN_CASES.items():
            np.random.seed(seed)
            store(name, [loaders[split][i] for split, i in items])
            out[name + "/case"] = np.array([seed, 4, 0, 1, 0, 0], dtype=np.int64)
            out[name + "/paths"] = np.array(["frames_%s/%d.npy" % (split, i) for split, i in items])
            out[name + "/mode"] = np.array([split for split, _ in items])
    np.savez_compressed(os.path.join(OUT, "indoor_pairs.npz"), **out)
    print("indoor_pairs.npz", os.path.getsize(os.path.join(OUT, "indoor_pairs.npz")) // 1024, "KB")


# data/scenenn_descriptor_loader.py SceneNNDescriptorLoader.__getitem__ on a synthetic SceneNN tree
# (usip_b200.data.scenenn_detector_loader.write_synthetic_scenenn with pairs): every positive frame the rigid image of its
# anchor, icp_np the aligning transform.  Train frame 4 (and so its positive, frame 5) has fewer than SD_N rows.
SD_N, SD_M, SD_SEED = 1024, 64, 8100
SD_COUNTS = {"train": 8, "val": 4, "test": 14}
SD_PAIRS = {"train": [(0, 1), (2, 3), (4, 5), (6, 7)], "val": [(0, 1), (2, 3)],
            "test": [(2 * k, 2 * k + 1) for k in range(7)]}          # the test loader keeps pairs 0, 3, 6
SD_CASES = {        # name: ([(split, item)], np seed, S, rot_horizontal, rot_3d, rot_perturbation, translation)
    "train": ([("train", 0)], 81, 4, 1, 0, 1, 0),                     # scenenn/options_descriptor.py defaults
    "rot3d": ([("train", 1)], 82, 4, 0, 1, 1, 1),
    "s3": ([("train", 3)], 83, 3, 1, 0, 1, 0),
    "short": ([("train", 2)], 84, 4, 1, 0, 1, 0),
    "val": ([("val", 1)], 85, 4, 1, 0, 1, 0),
    "test": ([("test", 1)], 86, 4, 1, 0, 1, 0),
    "seq": ([("train", 0), ("val", 0)], 87, 4, 1, 0, 1, 1),
    "wdiv": ([("train", 3)], 88, 4, 1, 0, 1, 0),                      # icp_np[3] replaced by SD_WDIV_ICP
}
SD_WDIV_ICP = np.array([[0.0, -1.0, 0.0, 0.5], [1.0, 0.0, 0.0, -0.25], [0.0, 0.0, 1.0, 0.125],
                        [0.01, -0.02, 0.015, 1.1]])                    # last row not [0 0 0 1]: pins the w division


def scenenn_desc_rows(split, i):
    return 600 if (split, i) in (("train", 4), ("train", 5)) else 1300


def golden_scenenn_descpairs(ref):
    import importlib
    import tempfile
    from usip_b200.data.scenenn_detector_loader import write_synthetic_scenenn
    sd = importlib.import_module("data.scenenn_descriptor_loader")
    keys = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node", "R", "scale", "shift")
    out = {"N": np.int64(SD_N), "M": np.int64(SD_M), "tree/seed": np.int64(SD_SEED),
           "tree/counts": np.array([SD_COUNTS[k] for k in ("train", "val", "test")], dtype=np.int64),
           "wdiv_icp": SD_WDIV_ICP}
    for split, p in SD_PAIRS.items():
        out["tree/pairs_" + split] = np.array(p, dtype=np.int64)
    with tempfile.TemporaryDirectory() as root:
        write_synthetic_scenenn(root, SD_COUNTS, scenenn_desc_rows, seed=SD_SEED, pairs=SD_PAIRS)
        for name, (items, seed, S, rh, r3, rp, tp) in SD_CASES.items():
            opt = ref_shim.make_opt(input_pc_num=SD_N, node_num=SD_M, surface_normal_len=S, rot_horizontal=bool(rh),
                                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp))
            loaders = {split: sd.SceneNNDescriptorLoader(root, split, opt) for split in SD_COUNTS}
            if name == "wdiv":
                loaders["train"].icp_np = loaders["train"].icp_np.copy()
                loaders["train"].icp_np[3] = SD_WDIV_ICP
            np.random.seed(seed)
            res = [loaders[split][i] for split, i in items]
            for k, vals in zip(keys, zip(*res)):
                out[name + "/" + k] = np.stack([np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32)
                                                for v in vals])
            out[name + "/case"] = np.array([seed, S, rh, r3, rp, tp], dtype=np.int64)
            out[name + "/split"] = np.array([split for split, _ in items])
            out[name + "/item"] = np.array([i for _, i in items], dtype=np.int64)
            out[name + "/frames"] = np.stack([loaders[split].pairs_np[i] for split, i in items]).astype(np.int64)
            out[name + "/icp"] = np.stack([loaders[split].icp_np[i] for split, i in items]).astype(np.float64)
            print("scenenn_descpairs", name, {k: out[name + "/" + k].shape for k in keys})
    np.savez_compressed(os.path.join(OUT, "scenenn_descpairs.npz"), **out)
    print("scenenn_descpairs.npz", os.path.getsize(os.path.join(OUT, "scenenn_descpairs.npz")) // 1024, "KB")


# data/oxford_detector_loader.py OxfordLoader.__getitem__ and data/oxford_descriptor_loader.py OxfordDescriptorLoader
# (items + default_collate + mine_negative_sample) on a synthetic Oxford tree (usip_b200.data.oxford_detector_loader.
# write_synthetic_oxford): OX_TRAIN ENU scans along a line (positives within 2, non-negatives within 4), an invalid line
# in train_relative.txt, OX_TEST test scans numbered 100 + 3 i; every scan (OX_ROWS, 8) float32.
OX_TRAIN, OX_TEST, OX_ROWS, OX_TREE_SEED, OX_N, OX_M = 16, 6, 1300, 7400, 1024, 64
OX_DESC_N = 512                                   # the descriptor's batches: 4 pairs
OX_CASES = {        # name: (mode, item, np seed, S, rot_horizontal, rot_3d, rot_perturbation, translation, height scaling)
    "default": ("train", 9, 41, 4, 1, 0, 0, 0, 1),              # oxford/options_detector.py defaults
    "s3": ("train", 2, 42, 3, 1, 0, 0, 0, 1),
    "s5": ("train", 14, 43, 5, 1, 0, 0, 0, 1),
    "rot3d": ("train", 5, 44, 4, 0, 1, 1, 1, 1),
    "noheight": ("train", 11, 45, 4, 1, 0, 0, 0, 0),
    "test": ("test", 3, 46, 4, 1, 0, 0, 0, 1),
}
OX_DESC_CASES = {   # name: (mode, items, np / random seed, S, rot_horizontal, rot_3d, rot_perturbation, translation)
    "train": ("train", [3, 12, 7, 0], 51, 4, 1, 0, 0, 0),
    "noneg": ("train", [5, 6, 9, 12], 52, 5, 0, 1, 1, 1),     # anchor 2 (line 9) has no negative in this batch
    "test": ("test", [0, 3, 1, 5], 53, 4, 1, 0, 0, 0),        # the mining runs B times
}


def _oxford_tree(root):
    from usip_b200.data.oxford_detector_loader import write_synthetic_oxford
    write_synthetic_oxford(root, OX_TRAIN, OX_ROWS, n_test=OX_TEST, seed=OX_TREE_SEED)
    return {"tree/counts": np.array([OX_TRAIN, OX_TEST]), "tree/rows": np.int64(OX_ROWS),
            "tree/seed": np.int64(OX_TREE_SEED), "N": np.int64(OX_N), "M": np.int64(OX_M)}


def golden_oxford_pairs(ref):
    import importlib
    import tempfile
    ol = importlib.import_module("data.oxford_detector_loader")
    keys = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "R", "scale", "shift")
    with tempfile.TemporaryDirectory() as root:
        out = _oxford_tree(root)
        for name, (mode, index, seed, S, rh, r3, rp, tp, hsc) in OX_CASES.items():
            opt = ref_shim.make_opt(input_pc_num=OX_N, node_num=OX_M, surface_normal_len=S, rot_horizontal=bool(rh),
                                    rot_3d=bool(r3), rot_perturbation=bool(rp), translation_perturbation=bool(tp),
                                    is_height_scaling=bool(hsc))
            loader = ol.OxfordLoader(root, mode, opt)
            np.random.seed(seed)
            res = loader[index]
            out[name + "/case"] = np.array([index, seed, S, rh, r3, rp, tp, hsc], dtype=np.int64)
            out[name + "/mode"] = np.array(mode)
            for k, v in zip(keys, res):
                out[name + "/" + k] = np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float32)
            print("oxford_pairs", name, {k: out[name + "/" + k].shape for k in keys})
    np.savez_compressed(os.path.join(OUT, "oxford_pairs.npz"), **out)
    print("oxford_pairs.npz", os.path.getsize(os.path.join(OUT, "oxford_pairs.npz")) // 1024, "KB")


def golden_oxford_descpairs(ref):
    import importlib
    import tempfile
    import types
    from torch.utils.data.dataloader import default_collate
    if "torch._six" not in sys.modules:                    # removed from torch; the loader only imports these names
        sys.modules["torch._six"] = types.ModuleType("torch._six")
        sys.modules["torch._six"].__dict__.update(string_classes=str, int_classes=int,
                                                 FileNotFoundError=FileNotFoundError)
    dl = importlib.import_module("data.oxford_descriptor_loader")
    keys = ("anc_pc", "anc_sn", "anc_node", "pos_pc", "pos_sn", "pos_node", "index")
    loaded = []
    np_load = np.load

    def logging_load(path, *a, **k):                       # which scan each item and positive reads
        loaded.append(os.path.basename(str(path)))
        return np_load(path, *a, **k)
    with tempfile.TemporaryDirectory() as root:
        out = _oxford_tree(root)
        out["N"] = np.int64(OX_DESC_N)
        np.load = logging_load
        try:
            for name, (mode, items, seed, S, rh, r3, rp, tp) in OX_DESC_CASES.items():
                opt = ref_shim.make_opt(input_pc_num=OX_DESC_N, node_num=OX_M, surface_normal_len=S,
                                        rot_horizontal=bool(rh), rot_3d=bool(r3), rot_perturbation=bool(rp),
                                        translation_perturbation=bool(tp))
                loader = dl.OxfordDescriptorLoader(root, mode, opt)
                np.random.seed(seed)
                random.seed(seed)
                del loaded[:]
                batch = default_collate([loader[i] for i in items])
                neg_idx = loader.mine_negative_sample(batch[6])
                out[name + "/case"] = np.array([seed, S, rh, r3, rp, tp], dtype=np.int64)
                out[name + "/items"] = np.array(items, dtype=np.int64)
                out[name + "/mode"] = np.array(mode)
                for k, v in zip(keys, batch):
                    out[name + "/" + k] = v.numpy()
                out[name + "/pos_file"] = np.array([int(f.split(".")[0]) for f in loaded[1::2]], dtype=np.int64)
                out[name + "/neg_idx"] = neg_idx.numpy()
                print("oxford_descpairs", name, "pos_file", out[name + "/pos_file"], "neg_idx", out[name + "/neg_idx"])
        finally:
            np.load = np_load
    np.savez_compressed(os.path.join(OUT, "oxford_descpairs.npz"), **out)
    print("oxford_descpairs.npz", os.path.getsize(os.path.join(OUT, "oxford_descpairs.npz")) // 1024, "KB")


# evaluation/kitti_test_loader.py KittiTestLoader and evaluation/oxford_test_loader.py OxfordTestLoader, batched by
# default_collate as save_keypoints.py's DataLoader does, plus save_keypoints.py:275's noise per batch, on synthetic
# test trees (usip_b200.evaluation.*.write_synthetic_*_test).  The index draws (rows, FPS candidates, FPS start) are
# logged from np.random as the loaders make them.  Five scans in batches of two: the last batch is odd.
TEST_COUNTS, TEST_PAIRS = [3, 2], [[(0, 1), (2, 1), (0, 2)], [(1, 0)]]
TEST_OX_NUMBERS, TEST_OX_PAIRS = [0, 1, 2, 3, 4], [(0, 1), (3, 2), (4, 4)]
TEST_ROWS, TEST_SEED, TEST_N, TEST_M, TEST_B = 1300, 7500, 512, 32, 2
TEST_CASES = {"plain": (61, 0.0), "noise": (62, 0.05)}      # name: (np / torch seed, noise sigma)


def _golden_test_clouds(ref, module, make_loader, write_tree, out_name, sn_len=4, N=TEST_N, M=TEST_M, B=TEST_B,
                        items=None, extra=None):
    """module: the reference loader's module under evaluation/ or a dotted path; items: the loader indices, in order
    (default all).  A rows draw of varying length (Redwood's remainder) is stored flat with its lengths."""
    import importlib
    import tempfile
    from torch.utils.data.dataloader import default_collate
    if ref_shim.build_ref_root() not in sys.path:
        sys.path.insert(0, ref_shim.build_ref_root())
    try:
        import PIL.Image  # noqa: F401               util/vis_tools.py imports it; only its plots use it
    except ImportError:
        import types
        sys.modules["PIL"] = types.ModuleType("PIL")
        sys.modules["PIL"].__dict__.update(Image=None, ImageMath=None)
    tl = importlib.import_module(module if "." in module else "evaluation." + module)
    out = {"tree/rows": np.int64(TEST_ROWS), "tree/seed": np.int64(TEST_SEED), "N": np.int64(N),
           "M": np.int64(M), "batch_size": np.int64(B)}
    draws = []
    np_choice, np_randint = np.random.choice, np.random.randint

    def choice(a, size=None, replace=True, p=None):
        r = np_choice(a, size, replace, p)
        draws.append(np.asarray(r))
        return r

    def randint(low, high=None, size=None, dtype=int):
        r = np_randint(low, high, size, dtype)
        draws.append(np.asarray(r))
        return r
    with tempfile.TemporaryDirectory() as root:
        write_tree(root)
        opt = ref_shim.make_opt(input_pc_num=N, node_num=M, surface_normal_len=sn_len)
        loader = make_loader(tl, root, opt)
        out.update(extra or {})                          # after make_loader, which may fill it
        order = list(range(len(loader))) if items is None else list(items)
        np.random.choice, np.random.randint = choice, randint
        try:
            for name, (seed, sigma) in TEST_CASES.items():
                np.random.seed(seed)
                torch.manual_seed(seed)
                del draws[:]
                res = {"pc": [], "sn": [], "node": []}
                for b0 in range(0, len(order), B):
                    batch = default_collate([loader[i] for i in order[b0:b0 + B]])
                    pc = batch[0]
                    if sigma:
                        pc = pc + torch.randn(pc.size()) * sigma
                    for k, v in zip(("pc", "sn", "node"), (pc, batch[1], batch[2])):
                        res[k].append(v.numpy())
                out[name + "/case"] = np.array([seed], dtype=np.int64)
                out[name + "/noise_sigma"] = np.float64(sigma)
                for k, v in res.items():
                    out[name + "/" + k] = np.concatenate(v)
                if len({len(r) for r in draws[0::3]}) == 1:
                    out[name + "/rows"] = np.stack(draws[0::3]).astype(np.int32)
                else:
                    out[name + "/rows_flat"] = np.concatenate(draws[0::3]).astype(np.int32)
                    out[name + "/rows_len"] = np.array([len(r) for r in draws[0::3]], dtype=np.int32)
                out[name + "/cand"] = np.stack(draws[1::3]).astype(np.int32)
                out[name + "/start"] = np.array(draws[2::3], dtype=np.int32)
                print(out_name, name, {k: out[name + "/" + k].shape for k in ("pc", "sn", "node", "cand")})
        finally:
            np.random.choice, np.random.randint = np_choice, np_randint
    np.savez_compressed(os.path.join(OUT, out_name), **out)
    print(out_name, os.path.getsize(os.path.join(OUT, out_name)) // 1024, "KB")


def golden_kitti_test(ref):
    from usip_b200.evaluation.kitti_test_loader import write_synthetic_kitti_test
    _golden_test_clouds(
        ref, "kitti_test_loader",
        lambda tl, root, opt: tl.KittiTestLoader(os.path.join(root, "txt"), os.path.join(root, "numpy"), opt),
        lambda root: write_synthetic_kitti_test(os.path.join(root, "txt"), os.path.join(root, "numpy"),
                                                os.path.join(root, "calib"), TEST_COUNTS, TEST_ROWS, TEST_PAIRS,
                                                seed=TEST_SEED),
        "kitti_test_clouds.npz")


def golden_oxford_test(ref):
    from usip_b200.evaluation.oxford_test_loader import write_synthetic_oxford_test
    def make_loader(tl, root, opt):
        loader = tl.OxfordTestLoader(root, opt)
        loader.dataset = list(TEST_OX_NUMBERS)           # the synthetic tree has 5 of the 828 test scans
        return loader
    _golden_test_clouds(
        ref, "oxford_test_loader", make_loader,
        lambda root: write_synthetic_oxford_test(root, TEST_OX_NUMBERS, TEST_ROWS, TEST_OX_PAIRS,
                                                 os.path.join(root, "groundtruths.txt"), seed=TEST_SEED),
        "oxford_test_clouds.npz")


# The rotated ModelNet40, Redwood and 3DMatch test loaders on synthetic trees, as above.  ModelNet: the reference
# hard-codes 2468 objects, so the tree has MN_TEST_K of them and items 0..k-1 and 2468..2468+k-1 are drawn.  Redwood:
# the reference's 207 frames, small, some shorter than N (taken whole, then a remainder).  3DMatch: every scene with
# frame numbers out of order on disk; the reference's os.listdir order is recorded as `listing/<scene>`.
MN_TEST_K, MN_TEST_N, MN_TEST_M, MN_TEST_B = 4, 512, 32, 4
RW_TEST_N, RW_TEST_M, RW_TEST_B = 32, 8, 4
M3_TEST_FRAMES, M3_TEST_N, M3_TEST_M, M3_TEST_B = (0, 10, 3), 256, 16, 4


def redwood_test_rows(s, f):
    """Rows of Redwood frame f of scene s in the synthetic tree: 5..80, so some frames are shorter than 32."""
    return 5 + (37 * f + 11 * s) % 76


def golden_modelnet_test(ref):
    from usip_b200.evaluation import modelnet_test_loader as mtl
    def write_tree(root):
        names = ["obj_%04d" % i for i in range(MN_TEST_K)]
        os.makedirs(os.path.join(root, "normal"))
        mtl.write_synthetic_modelnet40_normal(os.path.join(root, "normal"), names, TEST_ROWS, seed=TEST_SEED)
        mtl.write_rotated_modelnet(os.path.join(root, "normal"), os.path.join(root, "rotated_tree"), seed=TEST_SEED)
    _golden_test_clouds(
        ref, "data.modelnet_rotated_loader",
        lambda tl, root, opt: tl.ModelNet_Rotated_Loader(os.path.join(root, "rotated_tree"), opt), write_tree,
        "modelnet_test_clouds.npz", sn_len=3, N=MN_TEST_N, M=MN_TEST_M, B=MN_TEST_B,
        items=list(range(MN_TEST_K)) + list(range(2468, 2468 + MN_TEST_K)), extra={"objects": np.int64(MN_TEST_K)})


def golden_redwood_test(ref):
    from usip_b200.evaluation import indoor_test_loader as itl
    _golden_test_clouds(
        ref, "redwood_loader", lambda tl, root, opt: tl.RedwoodLoader(os.path.join(root, "npy"), opt),
        lambda root: itl.write_synthetic_redwood(os.path.join(root, "npy"), os.path.join(root, "gt"),
                                                 redwood_test_rows, {}, seed=TEST_SEED),
        "redwood_test_clouds.npz", N=RW_TEST_N, M=RW_TEST_M, B=RW_TEST_B)


def golden_3dmatch_test(ref):
    from usip_b200.evaluation import indoor_test_loader as itl
    listing = {}
    def make_loader(tl, root, opt):
        loader = tl.Match3DEvalLoader(os.path.join(root, "npy"), opt)
        for s in itl.MATCH3D_SCENES:
            listing["listing/" + s] = np.array([os.path.basename(d[0]) for d in loader.dataset
                                                if os.path.basename(os.path.dirname(d[0])) == s])
        return loader
    _golden_test_clouds(
        ref, "data.match3d_eval_loader", make_loader,
        lambda root: itl.write_synthetic_3dmatch(os.path.join(root, "npy"),
                                                 {s: M3_TEST_FRAMES for s in itl.MATCH3D_SCENES}, TEST_ROWS, {},
                                                 seed=TEST_SEED),
        "3dmatch_test_clouds.npz", N=M3_TEST_N, M=M3_TEST_M, B=M3_TEST_B, extra=listing)


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    ref = ref_shim.modules()
    if len(sys.argv) > 1:                                  # regenerate selected fixtures only, e.g. `make_golden.py ablation`
        for name in sys.argv[1:]:
            globals()["golden_" + name](ref)
        return
    golden_index_max(ref)
    golden_query_topk(ref)
    golden_losses(ref)
    detector_case(ref, "kitti_small", B=2, N=2048, M=64, S=4, Kn=16, kind="lidar", seed=1237)
    detector_case(ref, "modelnet_small", B=3, N=1000, M=32, S=3, Kn=32, kind="object", seed=1236, lb=1e-4, alpha=1.0)
    detector_case(ref, "lite_small", B=2, N=1024, M=32, S=4, Kn=16, kind="lidar", seed=1238, scene="indoor")
    golden_descriptor(ref)
    golden_desc_loss(ref)
    golden_descriptor_train(ref)
    golden_descriptor_indoor(ref)
    golden_descriptor_indoor_train(ref)
    golden_fps(ref)
    golden_nms(ref)
    golden_ablation(ref)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KB")


if __name__ == "__main__":
    main()
