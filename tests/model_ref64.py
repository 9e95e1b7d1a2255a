"""Functional float64 restatements, in torch autograd, of the train-mode networks and losses the fused plan differentiates
(usip_b200/engine.py: detector_backward, ablation_backward, descriptor_backward; the loss backward of ModelDetector /
ModelDescriptor).  Line numbers cite the original USIP code, as engine.py's docstrings do.

Every function takes the parameters as a dict keyed like the module's state_dict (`params64`) and runs on any device.
Every discrete decision of the forward is an ARGUMENT, held by a `Pins` object:
    min_idx   (B,N)      SOM assignment (util/som.py:35-39)
    knn_i     (B,M,Kn)   node kNN (layers.py:417-421)
    arg1/arg2 (B,C,M)    original point index of each (node, channel) segment max (networks.py:117-120, 130-133)
    sel_b/sel_a, sel3/sel5 (B,C,M)  row-in-group of each group pool: the row of max_k relu(bn(y_k)), i.e. the arg-max of
                         the raw y when the BN scale is >= 0 and its arg-min otherwise (engine.py's group_select)
    relu:<layer> (B,C,L) bool  the active set of each ReLU: an activation within rounding of 0 is as much a decision as
                         an arg-max, and one that flips moves a gradient sum by a whole term
    idx (B,M,K), perm (N,)  grouping indices (kNN / ball query) and the descriptor's point permutation
    i_sd/i_ds/i_src/i_dst, ipos/ineg  the arg-mins of the losses
With `Pins(strict=False)` a missing pool, ReLU or loss decision is derived from the values at hand -- the float64 arg-max /
arg-min / sign of the restatement itself, first index on ties like the kernels -- and recorded.  `pins.record` (when a
dict) receives every pool's and ReLU's float64 values with the decision taken, for the validity checks (pool_gaps,
relu_gaps, seg_gaps).
"""
import numpy as np
import torch
import torch.nn.functional as F

EPS = 1e-5


class Pins(dict):
    def __init__(self, *a, strict=True, record=None, **kw):
        super().__init__(*a, **kw)
        self.strict = strict
        self.record = record

    def need(self, key, derive):
        if key not in self:
            if self.strict:
                raise KeyError("decision %r is not pinned" % key)
            self[key] = derive()
        return self[key]


def params64(P, device="cpu", requires_grad=True):
    """state_dict-like mapping (numpy or torch) -> float64 leaf tensors; only floating entries that are parameters
    (conv weight / bias, norm weight / bias) get requires_grad."""
    out = {}
    for k, v in P.items():
        t = torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v.detach().cpu())
        if not t.is_floating_point():
            continue
        t = t.to(device=device, dtype=torch.float64).clone()
        if requires_grad and not (k.endswith("running_mean") or k.endswith("running_var")):
            t.requires_grad_(True)
        out[k] = t
    return out


def _gather_cols(t, idx):
    """t (B,C,L), idx (B,J) -> (B,C,J)."""
    return torch.gather(t, 2, idx.unsqueeze(1).expand(t.shape[0], t.shape[1], idx.shape[1]))


# ----------------------------------------------------------------------------- layers
def conv(x, P, name):
    """1x1 Conv1d / Conv2d on (B,Cin,L) (layers.py:178, 257)."""
    W = P[name + ".conv.weight"]
    return torch.einsum("oc,bcl->bol", W.reshape(W.shape[0], -1), x) + P[name + ".conv.bias"][None, :, None]


def bn_train(y, P, name):
    """Train-mode BatchNorm with batch statistics, biased variance (layers.py:69-71)."""
    mean = y.mean(dim=(0, 2), keepdim=True)
    var = y.var(dim=(0, 2), unbiased=False, keepdim=True)
    return (y - mean) / torch.sqrt(var + EPS) * P[name + ".norm.weight"][None, :, None] + P[name + ".norm.bias"][None, :, None]


def relu(pins, name, z):
    """ReLU at the pinned active set of layer `name` (pins["relu:" + name], bool like z): max(z, 0) with the same
    gradient wherever the set agrees with z > 0."""
    key = "relu:" + name
    on = pins.need(key, lambda: z.detach() > 0)
    if pins.record is not None:
        pins.record[key] = (z.detach(), on)
    return z * on.to(z.dtype)


def layer(x, P, name, pins, bn=True, act=True):
    """EquivariantLayer / MyConv2d forward (layers.py:289-303, 207-216)."""
    y = conv(x, P, name)
    if bn:
        y = bn_train(y, P, name)
    return relu(pins, name, y) if act else y


def group_pool(pins, key, y, act, gamma, K):
    """max over the K rows of each group of act = relu(bn(y)) (layers.py:433,438; networks.py:377,380) at the pinned row.
    y, act (B,C,M*K); gamma (C,) BN weight, or None for a linear layer (act = y, plain max).  -> (B,C,M)"""
    B, C, L = y.shape
    y4 = y.reshape(B, C, L // K, K)
    a4 = act.reshape(B, C, L // K, K)

    def derive():
        yd = y4.detach()
        if gamma is None:
            return yd.argmax(-1)
        return torch.where((gamma.detach() >= 0)[None, :, None], yd.argmax(-1), yd.argmin(-1))
    sel = pins.need(key, derive)
    if pins.record is not None:
        pins.record[key] = (a4.detach(), sel)
    return torch.gather(a4, 3, sel.unsqueeze(3)).squeeze(3)


def seg_pool(pins, key, feat, min_idx, M, mask):
    """index_max + gather + mask (networks.py:117-120, 130-133): feat (B,C,N) -> (B,C,M) at the pinned original point."""
    B, C, N = feat.shape

    def derive():
        f = feat.detach()
        cmax = torch.full((B, C, M), -torch.inf, dtype=f.dtype, device=f.device)
        cmax = cmax.scatter_reduce(2, min_idx.unsqueeze(1).expand(B, C, N), f, "amax", include_self=True)
        hit = f == torch.gather(cmax, 2, min_idx.unsqueeze(1).expand(B, C, N))
        n = torch.arange(N, device=f.device).expand(B, C, N)
        first = torch.full((B, C, M), N, dtype=torch.long, device=f.device)
        first = first.scatter_reduce(2, min_idx.unsqueeze(1).expand(B, C, N), torch.where(hit, n, N), "amin")
        return torch.where(first < N, first, 0)
    arg = pins.need(key, derive)
    if pins.record is not None:
        pins.record[key] = (feat.detach(), arg)
    return torch.gather(feat, 2, arg) * mask


# ----------------------------------------------------------------------------- detectors
def knn_fusion_head(P, pins, coords, feat, lb):
    """GeneralKNNFusionModule on the nodes (layers.py:401-440) + head mlp1/2/3, softplus (networks.py:143-154).
    coords (B,3,M) the nodes the kNN runs on and the offsets are added to; feat (B,C1,M).  -> keypoints, sigmas."""
    B, _, M = coords.shape
    ki = pins["knn_i"]
    Kn = ki.shape[2]
    kif = ki.reshape(B, M * Kn)
    nb_xyz = _gather_cols(coords, kif).reshape(B, 3, M, Kn) - coords[:, :, :, None]
    nb_feat = _gather_cols(feat, kif).reshape(B, -1, M, Kn)
    g = torch.cat([nb_xyz, nb_feat], 1).reshape(B, -1, M * Kn)            # layers.py:422-429
    nb = len({k.split(".")[2] for k in P if k.startswith("knnlayer_1.layers_before.")})
    na = len({k.split(".")[2] for k in P if k.startswith("knnlayer_1.layers_after.")})
    for i in range(nb - 1):
        g = layer(g, P, "knnlayer_1.layers_before.%d" % i, pins)
    name = "knnlayer_1.layers_before.%d" % (nb - 1)
    y = conv(g, P, name)
    g = relu(pins, name, bn_train(y, P, name))
    gmax = group_pool(pins, "sel_b", y, g, P[name + ".norm.weight"], Kn)  # layers.py:433
    h = torch.cat([gmax.unsqueeze(3).expand(-1, -1, -1, Kn).reshape(B, -1, M * Kn), g], 1)   # :435 (max first)
    for i in range(na - 1):
        h = layer(h, P, "knnlayer_1.layers_after.%d" % i, pins)
    name = "knnlayer_1.layers_after.%d" % (na - 1)
    y = conv(h, P, name)
    knn_feat = group_pool(pins, "sel_a", y, relu(pins, name, bn_train(y, P, name)), P[name + ".norm.weight"], Kn)  # :438
    agg = torch.cat([feat, knn_feat], 1)                                   # networks.py:143
    out = layer(layer(layer(agg, P, "mlp1", pins), P, "mlp2", pins), P, "mlp3", pins, bn=False, act=False)
    keypoints = out[:, 0:3, :] + coords                                    # :151
    sigmas = F.softplus(out[:, 3, :]) + lb                                 # :154 (Softplus beta 1, threshold 20)
    return keypoints, sigmas


def detector_forward(P, pins, x, sn, node, lb):
    """RPN_Detector / RPN_DetectorLite.forward, train mode (networks.py:75-162, k = 1).  x (B,3,N), sn (B,S,N) (S may be 0),
    node (B,3,M) are data.  -> (cluster_mean, keypoints, sigmas)."""
    B, _, N = x.shape
    M = node.shape[2]
    min_idx = pins["min_idx"]
    cnt = torch.zeros((B, M), dtype=x.dtype, device=x.device).scatter_add_(1, min_idx, torch.ones_like(x[:, 0]))
    csum = torch.zeros((B, 3, M), dtype=x.dtype, device=x.device).scatter_add_(2, min_idx.unsqueeze(1).expand(B, 3, N), x)
    cmean = csum / (cnt[:, None, :] + 1e-5)                                # networks.py:87-97
    x_dec = x - torch.gather(cmean, 2, min_idx.unsqueeze(1).expand(B, 3, N))   # :105-107
    x_aug = torch.cat([x_dec, sn], 1) if sn is not None and sn.shape[1] else x_dec
    mask = (cnt > 0).to(x.dtype)[:, None, :]                               # mask_row_max
    h = layer(x_aug, P, "first_pointnet.layers.0", pins)
    h = layer(h, P, "first_pointnet.layers.1", pins)
    first = layer(h, P, "first_pointnet.layers.2", pins, bn=False, act=False)   # layers.py:531-535
    pool1 = seg_pool(pins, "arg1", first, min_idx, M, mask)
    scattered = torch.gather(pool1, 2, min_idx.unsqueeze(1).expand(B, pool1.shape[1], N))
    h = layer(torch.cat([first, scattered], 1), P, "second_pointnet.layers.0", pins)   # :123-127
    second = layer(h, P, "second_pointnet.layers.1", pins, bn=False, act=False)
    pool2 = seg_pool(pins, "arg2", second, min_idx, M, mask)
    kp, sig = knn_fusion_head(P, pins, cmean, pool2, lb)
    return cmean, kp, sig


def group_net(P, pins, grp, bn5):
    """The grouped PointNet of DescriptorLiteOld (networks.py:375-381) and the ablation detectors (:567-572, 695-700):
    conv1..conv3, max_k, conv4 on cat(y, broadcast max) (max LAST), conv5, max_k.  grp (B,C,M,K).  -> (B,C5,M)"""
    B, C, M, K = grp.shape
    a = layer(grp.reshape(B, C, M * K), P, "conv1", pins)
    a = layer(a, P, "conv2", pins)
    y3 = conv(a, P, "conv3")
    a3 = relu(pins, "conv3", bn_train(y3, P, "conv3"))
    m3 = group_pool(pins, "sel3", y3, a3, P["conv3.norm.weight"], K)
    a4 = layer(torch.cat([a3, m3.unsqueeze(3).expand(-1, -1, -1, K).reshape(B, -1, M * K)], 1), P, "conv4", pins)
    y5 = conv(a4, P, "conv5")
    if bn5:
        return group_pool(pins, "sel5", y5, relu(pins, "conv5", bn_train(y5, P, "conv5")), P["conv5.norm.weight"], K)
    return group_pool(pins, "sel5", y5, y5, None, K)


def gather_groups(x_aug, centers, idx):
    """x_aug (B,C,N) gathered at idx (B,M,K), xyz minus the centre (networks.py:361-373, 565, 692) -> (B,C,M,K)."""
    B, C, _ = x_aug.shape
    _, M, K = idx.shape
    g = _gather_cols(x_aug, idx.reshape(B, M * K)).reshape(B, C, M, K)
    return torch.cat([g[:, :3] - centers[:, :, :, None], g[:, 3:]], 1)


def ablation_forward(P, pins, x, sn, node, lb):
    """RPN_Detector_KNN / RPN_Detector_Ball.forward, train mode (networks.py:545-608, 671-738): the grouping `pins["idx"]`
    (B,M,64) around the given nodes, the grouped PointNet, the node kNN fusion and head on the nodes.  -> keypoints, sigmas"""
    x_aug = torch.cat([x, sn], 1) if sn is not None and sn.shape[1] else x
    feat = group_net(P, pins, gather_groups(x_aug, node, pins["idx"]), bn5=True)
    return knn_fusion_head(P, pins, node, feat, lb)


def descriptor_forward(P, pins, x, sn, keypoints):
    """DescriptorLiteOld.forward, train mode (networks.py:333-385): points permuted by pins["perm"] (:345), balls
    pins["idx"] (B,M,K) into the permuted points (:355-362), grouped PointNet, max, L2 normalisation (:383)."""
    perm = pins["perm"]
    xp = x[:, :, perm]
    x_aug = torch.cat([xp, sn[:, :, perm]], 1) if sn is not None and sn.shape[1] else xp
    d = group_net(P, pins, gather_groups(x_aug, keypoints, pins["idx"]), bn5=False)
    return d / (torch.sqrt((d * d).sum(1, keepdim=True)) + 1e-5)


# ----------------------------------------------------------------------------- losses
def _argmin_dist(a, b):
    """arg-min_j ||a_i - b_j|| in float64, first index on ties: a (B,C,Ma), b (B,C,Nb) -> (B,Ma)."""
    a = a.detach(); b = b.detach()
    d2 = (a * a).sum(1)[:, :, None] + (b * b).sum(1)[:, None, :] - 2 * torch.einsum("bci,bcj->bij", a, b)
    return d2.argmin(2)


def pinned_min_dist(pins, key, a, b):
    """min_j ||a_i - b_j|| at the pinned arg-min (losses.py:62-66, 134-141): -> (B,Ma)."""
    arg = pins.need(key, lambda: _argmin_dist(a, b))
    return torch.sqrt(((a - _gather_cols(b, arg)) ** 2).sum(1))


def chamfer_sigma(pins, src, dst, sig_src, sig_dst):
    """ChamferLoss_Brute, sigma branch (losses.py:79-97): the loss (pure and weighted are not differentiated)."""
    d_sd = pinned_min_dist(pins, "i_sd", src, dst)
    d_ds = pinned_min_dist(pins, "i_ds", dst, src)
    s_sd = (sig_src + torch.gather(sig_dst, 1, pins["i_sd"])) / 2
    s_ds = (sig_dst + torch.gather(sig_src, 1, pins["i_ds"])) / 2
    return (torch.log(s_sd) + d_sd / s_sd).mean() + (torch.log(s_ds) + d_ds / s_ds).mean()


def point_on_surface(pins, key, kp, pc, sn):
    """PointOnSurfaceLoss (losses.py:146-183): squared cosine between the normal (sn[:, :3]) of the nearest cloud point
    and kp minus that point, the norm offset by 1e-7.  -> (B,M)"""
    arg = pins.need(key, lambda: _argmin_dist(kp, pc))
    d = kp - _gather_cols(pc, arg)
    n = _gather_cols(sn[:, :3], arg)
    s = (n * d).sum(1) / (torch.sqrt((d * d).sum(1)) + 1e-7)
    return s * s


def transform_keypoints(kp, R, scale, shift):
    """keypoint_detector.py:182-184: R @ kp * scale + shift."""
    return torch.matmul(R, kp) * scale.reshape(-1, 1, 1) + shift.reshape(-1, 3, 1)


def detector_loss(pins, kp, sig, src_pc, dst_pc, R, scale, shift, alpha, src_sn=None, dst_sn=None, on_pc="point_to_point"):
    """ModelDetector's train loss (keypoint_detector.py:182-204) on the siamese outputs kp (2B,3,M), sig (2B,M):
    chamfer(transform(src kp), dst kp) + alpha * mean keypoint-on-cloud term of each side."""
    B = src_pc.shape[0]
    kp_t = transform_keypoints(kp[:B], R, scale, shift)
    lc = chamfer_sigma(pins, kp_t, kp[B:], sig[:B], sig[B:])
    if on_pc == "point_to_point":
        ls = pinned_min_dist(pins, "i_src", kp[:B], src_pc).mean() * alpha
        ld = pinned_min_dist(pins, "i_dst", kp[B:], dst_pc).mean() * alpha
    else:
        ls = point_on_surface(pins, "i_src", kp[:B], src_pc, src_sn).mean() * alpha
        ld = point_on_surface(pins, "i_dst", kp[B:], dst_pc, dst_sn).mean() * alpha
    return lc + ls + ld, lc


def desc_pair_scan_loss(pins, anc, pos, neg, anc_sigmas, gamma=0.5, sigma_max=3.0):
    """DescPairScanLoss (losses.py:200-237) -> (loss (B,M), active (B)); the sigma weights carry no gradient."""
    dpos = pinned_min_dist(pins, "ipos", anc, pos)
    dneg = pinned_min_dist(pins, "ineg", anc, neg)
    before = dpos - dneg + gamma
    w = torch.clamp(sigma_max - anc_sigmas.detach(), min=0)
    w = w / w.mean(1, keepdim=True)
    return w * torch.clamp(before, min=0), (before > 0).to(before.dtype).mean(1)


def descriptor_train_loss(pins, desc, neg_idx, anc_sigmas, gamma=0.5, sigma_max=3.0):
    """ModelDescriptor.optimize's loss (keypoint_descriptor.py:126-157) on the siamese descriptors desc (2B,D,M): the
    triplet loss of anchors vs positives and the in-batch negatives anc[neg_idx], averaged."""
    B = desc.shape[0] // 2
    anc, pos = desc[:B], desc[B:]
    loss, active = desc_pair_scan_loss(pins, anc, pos, anc[neg_idx], anc_sigmas, gamma, sigma_max)
    return loss.mean(), active.mean()


# ----------------------------------------------------------------------------- decisions on the CPU
def cpu_detector_pins(x, node, Kn):
    """min_idx from oracle.som_assign (the fp32 arithmetic the reference runs) and the node kNN from oracle.knn on the fp32
    cluster means; the pools stay open for the float64 forward to derive.  x, node numpy (B,3,N), (B,3,M)."""
    from oracle import usip_oracle as orc
    min_idx = orc.som_assign(x, node).astype(np.int64)
    B, _, N = x.shape
    M = node.shape[2]
    cnt = np.stack([np.bincount(min_idx[b], minlength=M) for b in range(B)]).astype(np.float64)
    csum = np.stack([[np.bincount(min_idx[b], weights=x[b, c].astype(np.float64), minlength=M) for c in range(3)]
                     for b in range(B)])
    cmean = (csum / (cnt[:, None, :] + 1e-5)).astype(np.float32)
    knn_i, _ = orc.knn(cmean, cmean, Kn)
    return Pins(min_idx=torch.from_numpy(min_idx), knn_i=torch.from_numpy(knn_i.astype(np.int64)), strict=False)


def pool_gaps(record):
    """Decision validity from `Pins.record`: for every pinned pool choice, how far its float64 value lies below the float64
    maximum of its group, relative to the channel's largest |value|.  -> {key: (worst gap, number of choices that differ
    from the float64 arg-max, number of choices)}"""
    out = {}
    for key, (vals, sel) in record.items():
        if vals.dim() != 4 or key.startswith("relu:"):          # the segment maxima: seg_gaps; ReLUs: relu_gaps
            continue
        best = vals.max(-1).values
        got = torch.gather(vals, 3, sel.unsqueeze(3)).squeeze(3)
        scale = vals.abs().amax(dim=(0, 2, 3))[None, :, None]
        gap = (best - got) / torch.clamp(scale, min=1e-30)
        out[key] = (float(gap.max()), int((got < best).sum()), int(sel.numel()))
    return out


def relu_gaps(record):
    """Validity of pinned ReLU active sets: where one disagrees with the float64 z > 0, how close z is to 0 relative to the
    channel's largest |z|.  -> {key: (worst, number of disagreements, number of elements)}"""
    out = {}
    for key, (z, on) in record.items():
        if not key.startswith("relu:"):
            continue
        off = on != (z > 0)
        scale = z.abs().amax(dim=(0, 2), keepdim=True)
        gap = (z.abs() / torch.clamp(scale, min=1e-30))[off]
        out[key] = (float(gap.max()) if gap.numel() else 0.0, int(off.sum()), int(z.numel()))
    return out


def seg_gaps(record, min_idx, M):
    """pool_gaps for the two segment maxima (keys arg1, arg2): the pinned point's float64 value against the float64 maximum
    over its cluster (empty clusters are masked and skipped)."""
    out = {}
    for key in ("arg1", "arg2"):
        if key not in record:
            continue
        f, arg = record[key]
        B, C, N = f.shape
        ix = min_idx.unsqueeze(1).expand(B, C, N)
        cmax = torch.full((B, C, M), -torch.inf, dtype=f.dtype, device=f.device).scatter_reduce(2, ix, f, "amax")
        got = torch.gather(f, 2, arg)
        cnt = torch.zeros((B, M), dtype=f.dtype, device=f.device).scatter_add_(1, min_idx, torch.ones_like(f[:, 0]))
        live = (cnt > 0)[:, None, :].expand(B, C, M)
        own = torch.gather(min_idx, 1, arg.reshape(B, C * M)).reshape(B, C, M)
        assert bool((own == torch.arange(M, device=f.device)[None, None, :])[live].all()), key + ": pinned point outside its cluster"
        scale = f.abs().amax(dim=(0, 2))[None, :, None]
        gap = ((cmax - got) / torch.clamp(scale, min=1e-30))[live]
        out[key] = (float(gap.max()), int((gap > 0).sum()), int(live.sum()))
    return out
