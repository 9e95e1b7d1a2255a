"""References for the indoor descriptor DescriptorLiteOldGlobal (models/networks.py:388-479).

* ball_query_wrapper: the reference network calls models.operations.ball_query_wrapper, which the reference ships
  commented out (operations.py:436-469).  This is that function restated: the (B,M,N) distance matrix by torch.norm, then
  the ball query of the `ball_query` module oracle/ref_shim.py installed -- the CPU restatement of ball_query_cuda.cu in
  cpu mode, the reference's own extension in cuda mode.  install() gives it to the reference's operations module, so the
  unmodified reference network runs.
* numba_ball_query: the commented-out numba kernel (operations.py:397-432) in numpy, loop for loop.  An empty ball reads
  `i % 0`, which is 0 under numba's CUDA error model, from a zero-initialised buffer: index 0.
* forward64: the network's forward in float64 from its x_features, eval or train BatchNorm.
* reference_outputs: one eval and one train forward of the reference network on a stored case (the golden's recipe).
"""
import os
import sys

import numpy as np
import torch

EPS = 1e-5


def ball_query_wrapper(pc, node, radius, nsamples):
    """operations.py:436-469: pc (B,3,N), node (B,3,M) -> (B,M,nsamples) int64."""
    dist = torch.norm(node.unsqueeze(3) - pc.unsqueeze(2), p=2, dim=1, keepdim=False).detach()
    return sys.modules["ball_query"].forward_cuda_shared_mem(dist.contiguous(), radius, int(nsamples)).long()


def install(ref):
    ref.networks.operations.ball_query_wrapper = ball_query_wrapper


def numba_ball_query(dist, radius, nsamples):
    dist = np.asarray(dist, np.float32)
    B, M, N = dist.shape
    out = np.zeros((B, M, nsamples), np.int64)
    r = np.float32(radius)
    for b in range(B):
        for m in range(M):
            hits = np.flatnonzero(dist[b, m] <= r)[:nsamples]
            u = hits.size
            out[b, m, :u] = hits
            for i in range(nsamples - u):
                out[b, m, u + i] = out[b, m, i % u] if u else 0
    return out


def _bn(y, sd, name, train, momentum, axes):
    w, b = sd[name + ".norm.weight"].double(), sd[name + ".norm.bias"].double()
    shape = [1, -1] + [1] * (y.dim() - 2)
    if train:
        n = 1
        for a in axes:
            n *= y.shape[a]
        mean = y.mean(dim=axes)
        var = ((y - mean.view(shape)) ** 2).mean(dim=axes)
        run = (sd[name + ".norm.running_mean"].double() * (1 - momentum) + momentum * mean,
               sd[name + ".norm.running_var"].double() * (1 - momentum) + momentum * var * n / (n - 1))
    else:
        mean, var = sd[name + ".norm.running_mean"].double(), sd[name + ".norm.running_var"].double()
        run = None
    out = torch.relu((y - mean.view(shape)) / torch.sqrt(var.view(shape) + EPS) * w.view(shape) + b.view(shape))
    return out, run


def forward64(sd, feats, train, momentum=0.1):
    """x_features (B,3+S,M,K) -> (descriptor (B,D,M) float64, {running stat name: float64 tensor} after a train forward)."""
    sd = {k: v.to(feats.device) for k, v in sd.items()}
    run = {}

    def conv(x, name, bn):
        W = sd[name + ".conv.weight"].double().reshape(sd[name + ".conv.weight"].shape[0], -1)
        y = torch.einsum("oc,bc...->bo...", W, x) + sd[name + ".conv.bias"].double().view([1, -1] + [1] * (x.dim() - 2))
        if not bn:
            return y
        y, r = _bn(y, sd, name, train, momentum, [0] + list(range(2, x.dim())))
        if r is not None:
            run[name + ".norm.running_mean"], run[name + ".norm.running_var"] = r
        return y

    x = feats.double()
    y3 = conv(conv(conv(x, "conv1", True), "conv2", True), "conv3", True)
    y3max = y3.max(dim=3, keepdim=True)[0].expand_as(y3)
    desc = conv(conv(torch.cat((y3, y3max), 1), "conv4", True), "conv5", False).max(dim=3)[0]        # (B,D,M)
    glob = desc.max(dim=2, keepdim=True)[0].expand_as(desc)
    out = conv(conv(conv(torch.cat((desc, glob), 1), "fc1", True), "fc2", True), "fc3", False)
    return out / (torch.norm(out, dim=1, keepdim=True) + EPS), run


def make_inputs(B, N, M, S, seed, half):
    """Clouds uniform in a cube of half-size `half` (float32 pc (B,3,N), sn (B,S,N)) and M keypoints near points, so that
    balls of radius 0.75 range from partly filled (cube faces) to over-full (interior) at 448 samples; keypoint 0 of
    every cloud lies far outside, an empty ball."""
    rng = np.random.default_rng(seed)
    pc = rng.uniform(-half, half, (B, 3, N)).astype(np.float32)
    sn = rng.normal(0, 1, (B, S, N)).astype(np.float32)
    pick = rng.integers(0, N, (B, M))
    kp = (np.take_along_axis(pc, pick[:, None, :], axis=2) + rng.normal(0, 0.05, (B, 3, M))).astype(np.float32)
    kp[:, :, 0] = 50.0
    return pc, sn, kp


def randomized_params(net, seed):
    """state_dict of a freshly built network (torch seeded by the caller) with non-trivial BatchNorm affines, running
    statistics and conv biases."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in net.state_dict().items():
        v = v.detach().cpu().clone()
        if k.endswith("norm.weight") or k.endswith("running_var"):
            v = torch.rand(v.shape, generator=g) + 0.5
        elif k.endswith("norm.bias") or k.endswith("running_mean"):
            v = torch.randn(v.shape, generator=g) * 0.1
        elif k.endswith("conv.bias"):
            v = torch.randn(v.shape, generator=g) * 0.05
        sd[k] = v
    return sd


def reference_outputs(ref, case):
    """The reference network with the case's weights: eval then train forward, each after np.random.seed(seed) (the
    forward draws its point permutation from numpy, networks.py:443).  -> dict of numpy arrays."""
    B, N, M, S, K, seed = [int(v) for v in case["cfg"]]
    from oracle import ref_shim
    install(ref)
    opt = ref_shim.make_opt(batch_size=B, input_pc_num=N, node_num=M, surface_normal_len=S,
                            ball_radius=float(case["radius"]), ball_nsamples=K, descriptor_len=int(case["D"]))
    net = ref.networks.DescriptorLiteOldGlobal(opt)
    net.load_state_dict({k[len("param/"):]: torch.from_numpy(np.asarray(case[k])) for k in case.files
                         if k.startswith("param/")})
    dev = "cuda" if ref_shim._installed == "cuda" else "cpu"
    net = net.to(dev)
    pc, sn, kp = (torch.from_numpy(np.asarray(case[k])).to(dev) for k in ("pc", "sn", "kp"))
    out = {}
    for mode in ("eval", "train"):
        net.train(mode == "train")
        np.random.seed(seed)
        with torch.no_grad():
            desc, feats = net(pc, sn, kp, mode == "train", None)
        out[mode + "_desc"] = desc.cpu().numpy()
        out[mode + "_feats"] = feats.cpu().numpy()
    for k, v in net.state_dict().items():
        if "running" in k or "num_batches" in k:
            out["after/" + k] = v.cpu().numpy()
    return out


def feats_sample(n):
    """The fixed sample of x_features the golden files store."""
    from tests.util_gpu import sample_idx
    return sample_idx(n, 16384, 5)


def reconstruct_features(pc, sn, kp, idx, perm):
    """x_features from the ball indices into the permuted cloud (networks.py:443-463), in float32 as the reference."""
    x_aug = np.concatenate([pc, sn], 1)[:, :, perm]
    B, C = x_aug.shape[:2]
    _, M, K = idx.shape
    f = np.take_along_axis(x_aug, idx.reshape(B, 1, M * K).astype(np.int64), axis=2).reshape(B, C, M, K)
    f[:, :3] = f[:, :3] - kp[:, :, :, None]
    return f


def main_check(golden_path):
    """Run the reference on the CPU through the shim (a process of its own: the cpu-mode shim patches torch.cuda) and
    print the largest differences from the golden file."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from oracle import ref_shim
    torch.set_num_threads(4)
    ref = ref_shim.modules()
    case = np.load(golden_path)
    out = reference_outputs(ref, case)
    for mode in ("eval", "train"):
        d, g = out[mode + "_desc"].astype(np.float64), case[mode + "_desc"].astype(np.float64)
        print("desc_%s %.3e" % (mode, np.abs(d - g).max() / np.abs(g).max()))
        f = out[mode + "_feats"].ravel()[feats_sample(out[mode + "_feats"].size)]
        print("feats_%s %d" % (mode, int(not np.array_equal(f, case["feats"]))))
    for k in case.files:
        if k.startswith("after/"):
            a, g = out[k].astype(np.float64), case[k].astype(np.float64)
            print("%s %.3e" % (k, np.abs(a - g).max() / max(np.abs(g).max(), 1e-12)))


if __name__ == "__main__":
    main_check(sys.argv[1])
