"""Freezes what the original USIP implementation computes ON THE GPU into tests/golden/reference_*.npz, for the tests that
compare against it (tests/test_gpu_ops.py, tests/test_gpu_vs_reference.py).  Needs the original code's two CUDA extensions
and its Python tree under oracle/_ref (oracle/build_ref.py) and a CUDA device:

    python tools/make_gpu_golden.py OUT_DIR        # then copy OUT_DIR/reference_*.npz to tests/golden/

The inputs are built by the tests' own helpers, so a test and this script see the same tensors.  Large outputs are stored
as fixed, seeded samples (tests/util_gpu.sample_idx) to keep every file under 1 MB."""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import build_ref, ref_shim, usip_oracle as orc  # noqa: E402
from tests import test_gpu_ops as O, test_gpu_vs_reference as T  # noqa: E402
from tests.util_gpu import cu, sample_idx  # noqa: E402


def ops_golden(out):
    im, bq = build_ref.load_reference_index_max(), build_ref.load_reference_ball_query()
    data, index = O.index_max_full_inputs()
    g = {"index_max": im.forward_cuda(cu(data), cu(index), 512)[:, ::16].cpu().numpy().astype(np.int16)}
    _, _, dist = O.ball_query_inputs()
    g["ball_query"] = bq.forward_cuda_shared_mem(cu(dist), 1.0, 64).cpu().numpy().astype(np.int16)
    for dense in (False, True):
        pc, _, kp = (cu(a) for a in O.ball_group_inputs(dense))
        dist = torch.norm(kp.unsqueeze(3) - pc.unsqueeze(2), dim=1).contiguous()
        idx = bq.forward_cuda_shared_mem(dist, 1.0, 64).cpu().numpy()
        g["ball_group_dense" if dense else "ball_group"] = idx[:, ::(1 if dense else 8)].astype(np.int16)
        del dist
        torch.cuda.empty_cache()
    np.savez_compressed(os.path.join(out, "reference_ops.npz"), **g)


def ref_run(ref, cfg, ins, double=False):
    """The unmodified reference on cuda: test_model() (eval BN) then optimize(epoch=0).  double=True runs the same modules
    in float64 -- the arbiter for the gradient comparison (only index_max, a float32-only extension, gets a float32 copy of
    its input; it returns indices)."""
    import index_max as ref_im
    big = 2 * cfg["B"] * cfg["M"] > 12288
    saved_fn = ref_im.forward_cuda_shared_mem
    # index_max_cuda.cu:92-96: the shared-memory variant needs B*K*4 <= 48 KB and silently returns zeros beyond it (no
    # cudaFuncSetAttribute); the reference's global-memory entry point is the same algorithm
    base_fn = ref_im.forward_cuda if big else saved_fn
    ref_im.forward_cuda_shared_mem = (lambda d, i, k: base_fn(d.float().contiguous(), i, k)) if double else base_fn
    try:
        rmd = T._mk(ref.keypoint_detector.ModelDetector, cfg)
        if double:
            rmd.detector.double()
            rmd.optimizer_detector = torch.optim.Adam(rmd.detector.parameters(), lr=rmd.opt.lr, betas=(0.9, 0.999), weight_decay=0)
            names = ("src_pc", "src_sn", "src_node", "dst_pc", "dst_sn", "dst_node", "src_R_dst", "src_scale_dst", "src_shift_dst")
            for k, v in zip(names, ins):                         # set_input() casts to float32 (keypoint_detector.py:125-133)
                setattr(rmd, k, v.double().to(rmd.opt.device))
        else:
            rmd.set_input(*ins)
        with torch.no_grad():
            rmd.test_model()
        r_eval = T._outs(rmd)
        random.seed(0); np.random.seed(0)
        rmd.optimize(epoch=0)
        torch.cuda.synchronize()
        r_train = T._outs(rmd)
        r_grad = {k: p.grad.detach().cpu().numpy().astype(np.float64) for k, p in rmd.detector.named_parameters()}
        r_sd = {k: v.detach().cpu().numpy() for k, v in rmd.detector.state_dict().items()}
    finally:
        ref_im.forward_cuda_shared_mem = saved_fn
    del rmd
    torch.cuda.empty_cache()
    return r_eval, r_train, r_grad, r_sd


def detector_golden(ref, name, out):
    cfg = T.CONFIGS[name]
    d = orc.synth_pair(cfg["B"], cfg["N"], cfg["M"], cfg["S"], kind=cfg["kind"], seed=cfg["seed"])
    ins = [torch.from_numpy(d[k]) for k in T.KEYS]
    r_eval, r_train, r_grad, r_sd = ref_run(ref, cfg, ins)
    _, r64_train, r64_grad, _ = ref_run(ref, cfg, ins, double=True)
    g = {}
    for tag, o in (("eval", r_eval), ("train", r_train), ("train64", r64_train)):
        for k, v in T.sampled_outs(o).items():
            g["%s__%s" % (tag, k)] = v.astype(np.float64 if k == "loss" else np.float32)
    for k in r_grad:
        g32, g64 = r_grad[k], r64_grad[k]
        wk = k.replace("bias", "weight")
        scale = np.abs(g64).max()
        if k.endswith("conv.bias"):
            scale = max(scale, np.abs(r64_grad[wk]).max())
        n64 = np.linalg.norm(g64)
        l2_scale = max(n64, np.linalg.norm(r64_grad[wk]) * 1e-3 if k.endswith("conv.bias") else n64, 1e-300)
        analytic_zero = bool(n64 < 1e-6 * np.linalg.norm(r64_grad[wk])) if k.endswith("conv.bias") else False
        st = dict(scale=scale, l2_scale=l2_scale, n64=n64, analytic_zero=float(analytic_zero),
                  e_ref=T._grad_err(g32, g64, scale), l2_ref=np.linalg.norm(g32 - g64) / l2_scale, gmax32=np.abs(g32).max())
        g["gstat__" + k] = np.array([st[s] for s in T.GSTAT], np.float64)
        g["g64__" + k] = g64.ravel()[sample_idx(g64.size, T.NGRAD, T.name_seed(k))]
    for k, v in r_sd.items():
        idx = sample_idx(v.size, T.NGRAD, T.name_seed(k))
        g["sd__" + k] = v.ravel()[idx]
        if k in r_grad:
            g["g32sd__" + k] = r_grad[k].ravel()[idx].astype(np.float32)
    np.savez_compressed(os.path.join(out, "reference_detector_%s.npz" % name), **g)


def descriptor_golden(ref, out):
    from usip_b200.models import networks as our_networks
    opt, (x, s, k) = T.descriptor_setup()
    torch.manual_seed(3)                                         # as the test: the parameters come from this repo's module
    ours = our_networks.DescriptorLiteOld(opt)
    net = ref.networks.DescriptorLiteOld(opt).cuda()
    net.load_state_dict(T._randomized_state(ours, seed=3))
    np.savez_compressed(os.path.join(out, "reference_descriptor.npz"), **T.descriptor_run(net, x, s, k))


def descriptor_indoor_golden(ref, out):
    """DescriptorLiteOldGlobal at the indoor evaluation shape, with tests/desc_indoor_ref.py's ball_query_wrapper on the
    reference's ball_query extension: fixed samples of descriptors and x_features, the running statistics whole."""
    from tests import desc_indoor_ref as dref
    from tests import test_gpu_descriptor_indoor as DI
    c = DI.FULL
    _, (pc, sn, kp), state = DI.full_setup()
    case = dict(cfg=np.array([c["B"], c["N"], c["M"], c["S"], c["K"], c["seed"]], np.int64), radius=np.float32(0.75),
                D=np.int64(c["D"]), pc=pc, sn=sn, kp=kp, **{"param/" + k: v.numpy() for k, v in state.items()})

    class Case(dict):
        files = property(lambda self: list(self.keys()))
    r = dref.reference_outputs(ref, Case(case))
    g = {}
    for mode in ("eval", "train"):
        g["desc_" + mode], g["feats_" + mode] = DI.sampled(r[mode + "_desc"], r[mode + "_feats"])
    for k, v in r.items():
        if k.startswith("after/") and "running" in k:
            g["run__" + k[len("after/"):]] = v
    np.savez_compressed(os.path.join(out, "reference_descriptor_indoor.npz"), **g)


def descriptor_indoor_train_golden(ref, out):
    """One ModelDescriptorIndoor.optimize() of the reference at SceneNN's training shape (B=2 pairs, N=5000, M=512, K=448,
    D=128, radius 0.75, CGF_radius 0.075, gamma 0.3, sigma_max 0.5) after torch.cuda.manual_seed, in float32 and in
    float64 (the same modules and draws): the picks (its three torch.gather indices), loss, active share, sampled float64
    gradients, their scales and the float32 run's own error against them (DESIGN section 2)."""
    from tests import cgf_ref
    from tests import desc_indoor_ref as dref
    from tests import test_gpu_descriptor_indoor_train as TI
    c = TI.FULL
    opt, d, state = TI.full_setup()
    dref.install(ref)
    ref_opt = ref_shim.make_opt(**{k: getattr(opt, k) for k in vars(opt) if k != "use_tensor_cores"})
    runs = {}
    for dtype in (torch.float32, torch.float64):
        md = ref.keypoint_descriptor.ModelDescriptorIndoor(ref_opt)
        md.descriptor.load_state_dict(state)
        if dtype == torch.float64:
            md.descriptor.double()
            md.optimizer_descriptor = torch.optim.Adam(md.descriptor.parameters(), lr=ref_opt.lr, betas=(0.9, 0.999),
                                                       weight_decay=0)
        ins = [torch.from_numpy(d[k]) for k in cgf_ref.SET_INPUT_KEYS]
        md.set_input(*ins)
        if dtype == torch.float64:                           # set_input keeps float32 placeholders: cast the batch
            for k in ("anc_pc", "anc_sn", "anc_keypoints", "anc_sigmas", "pos_pc", "pos_sn", "pos_keypoints", "pos_sigmas",
                      "anc_R_pos", "anc_scale_pos", "anc_shift_pos"):
                setattr(md, k, getattr(md, k).double())
        picks = []
        gather = torch.gather

        def rec_gather(x, dim, index, *a, **k):
            if index.dim() == 3 and index.shape[2] == 1 and x.shape[1] == x.shape[2]:
                picks.append(index.squeeze(2).cpu().numpy())
            return gather(x, dim, index, *a, **k)
        bq = sys.modules["ball_query"].forward_cuda_shared_mem
        sys.modules["ball_query"].forward_cuda_shared_mem = lambda dist, r, n: bq(dist.float().contiguous(), r, n)
        torch.gather = rec_gather
        try:
            torch.cuda.manual_seed(c["seed"])
            np.random.seed(c["seed"])
            md.optimize(epoch=0)
            torch.cuda.synchronize()
        finally:
            torch.gather = gather
            sys.modules["ball_query"].forward_cuda_shared_mem = bq
        assert len(picks) == 3, len(picks)
        runs[dtype] = dict(picks=picks, loss=md.loss.item(), active=md.active_percentage.item(),
                           grad={k: p.grad.detach().cpu().numpy().astype(np.float64)
                                 for k, p in md.descriptor.named_parameters()})
        del md
        torch.cuda.empty_cache()
    r32, r64 = runs[torch.float32], runs[torch.float64]
    for a, b in zip(r32["picks"], r64["picks"]):
        assert np.array_equal(a, b), "float32 and float64 runs picked differently"
    g = dict(near=r32["picks"][0], far=r32["picks"][1], out=r32["picks"][2], loss32=np.float64(r32["loss"]),
             loss64=np.float64(r64["loss"]), active=np.float32(r32["active"]))
    for k, g64 in r64["grad"].items():
        g32 = r32["grad"][k]
        idx = TI.grad_sample(k, g64.size)
        scale = np.abs(g64).max()
        if k.endswith("conv.bias") and np.linalg.norm(g64) < 1e-6 * np.linalg.norm(r64["grad"][k.replace("bias", "weight")]):
            scale = 0.0                                       # in front of a train-mode BatchNorm: true gradient 0
        g["g64__" + k] = g64.ravel()[idx]
        g["gscale__" + k] = np.float64(scale)
        g["gnorm__" + k] = np.float64(np.linalg.norm(g64))
        g["eref__" + k] = np.float64(np.abs(g32 - g64).max() / scale if scale else 0.0)
    print("descriptor_indoor_train: loss fp32 %.7f fp64 %.7f, worst fp32 gradient error %.2e" % (
        r32["loss"], r64["loss"], max(float(v) for k, v in g.items() if k.startswith("eref__"))))
    np.savez_compressed(os.path.join(out, "reference_descriptor_indoor_train.npz"), **g)


def main():
    out = sys.argv[1]
    only = sys.argv[2:]                        # e.g. `descriptor_indoor`: regenerate that file only
    os.makedirs(out, exist_ok=True)
    if not (ref_shim.reference_available() and build_ref.have("index_max") and build_ref.have("ball_query")):
        raise SystemExit("oracle/_ref (the original code's extensions and Python tree) is not built")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    if only:
        ref = ref_shim.modules(mode="cuda")
        for name in only:
            globals()[name + "_golden"](ref, out)
        return
    ops_golden(out)
    ref = ref_shim.modules(mode="cuda")
    for name in T.CONFIGS:
        detector_golden(ref, name, out)
    descriptor_golden(ref, out)
    descriptor_indoor_golden(ref, out)
    descriptor_indoor_train_golden(ref, out)
    for f in sorted(os.listdir(out)):
        print(f, os.path.getsize(os.path.join(out, f)))


if __name__ == "__main__":
    main()
