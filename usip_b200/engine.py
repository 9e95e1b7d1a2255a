"""Fused H100 execution plan of the USIP detector / descriptor networks.

This is NOT a layer-by-layer translation of models/networks.py: the (B,C,N) activations of the reference
are replaced by point-major [rows, C] buffers over points SORTED BY NODE, so that
  * index_max + gather + mask (networks.py:117-120,130-133) is a contiguous segmented max,
  * the un-pool gather (networks.py:123-126) and the concat that follows become a per-node GEMM whose
    result is added in the consuming layer's epilogue (W [a;b] = Wa a + Wb b),
  * the kNN group tensor (B,3+C,M,K) of layers.py:422-429 is never built: W_feat @ feat is computed once
    per node and gathered; the broadcast-max half of layers.py:435 likewise,
  * train-mode BatchNorm (layers.py:69-71) is "epilogue emits statistics -> finalize -> next layer's
    prologue normalises": every pre-BN activation is written once and read once,
  * max_k relu(bn(y_k)) (layers.py:433,438) comes from per-group max/min of the raw GEMM output.
All arithmetic happens in libusip_b200.so; torch only owns memory / streams / autograd plumbing.
"""
import torch

from . import _lib, ops

f32 = torch.float32
i32 = torch.int32

# Optional per-op device timing (bench.py): set PROFILE = {} to record CUDA-event pairs around every op of the
# plan on the launching stream; collect_profile() turns them into mean milliseconds per op name.
PROFILE = None


class _Prof:
    def __init__(self, name, flops=None, nbytes=None, precision=None):
        self.on = PROFILE is not None
        if self.on:
            self.name, self.flops, self.nbytes, self.precision = name, flops, nbytes, precision

    def __enter__(self):
        if self.on:
            self.e0 = torch.cuda.Event(enable_timing=True); self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *a):
        if self.on:
            self.e1.record()
            rec = PROFILE.setdefault(self.name, dict(ev=[], flops=self.flops, bytes=self.nbytes, precision=self.precision))
            rec["ev"].append((self.e0, self.e1))
        return False


def collect_profile():
    out = {}
    if not PROFILE:
        return out
    torch.cuda.synchronize()
    for k, rec in PROFILE.items():
        ms = [a.elapsed_time(b) for a, b in rec["ev"]]
        out[k] = dict(ms=sum(ms) / len(ms), n=len(ms), flops=rec["flops"], bytes=rec["bytes"], precision=rec["precision"])
    return out


def _conv_w(layer, cols=None):
    """[Cout, Cin] view of the conv1x1 `layer`'s weight -- only the columns `cols` (a concat half) when given -- and the
    offset of its first column."""
    W = layer.conv.weight.detach().flatten(1)
    return (W, 0) if cols is None else (W[:, cols], cols.start)


class BNState:
    """Folded affine of one BatchNorm for the current step (+ what backward needs)."""
    __slots__ = ("scale", "shift", "mean", "invstd", "count")


# Packed (hi/lo TF32, pre-swizzled) weight tiles are cached on the weight Parameter and re-used while its autograd
# version counter is unchanged (inference / fwd-only loops); an optimizer step bumps the version and the next launch
# re-packs into the same workspace.
class _PackEntry:
    """One packed-weight workspace: the version it was packed at, and -- once the layer has run -- a copy of its descriptor,
    so that prepack_weights() can re-pack it together with all the others in one launch."""
    __slots__ = ("ver", "ws", "ptr", "desc", "keep", "used_step")

    def __init__(self, ver, ws, ptr):
        self.ver, self.ws, self.ptr, self.desc, self.keep, self.used_step = ver, ws, ptr, None, None, -1

    def remember(self, d, W):
        """Keep a copy of the descriptor `d` the layer launched with (its W / workspace pointers; the tensors are kept
        alive next to it), so that the pack can join the one-launch re-pack of a train step."""
        if self.desc is None:
            self.desc, self.keep = ops.LayerDesc.from_buffer_copy(d), (W, self.ws)


_PACK_STEP = [0]


def _tc_workspace(weight, col0, P, Cin, Cout, transposed):
    """-> (workspace, already_packed, entry) of the tensor-core tiles of the conv weight Parameter `weight` as one layer
    launch reads it: columns from col0 on, Cin x Cout as the launch sees them (swapped for a transposed use).  The key
    holds what the pack depends on; P is there because the column-tile width follows from P and Cout."""
    cache = weight.__dict__.setdefault("_usip_tc", {})  # lives and dies with the Parameter object
    key = (col0, P, Cin, Cout, bool(transposed))
    ver = (weight._version, _lib.WEIGHT_GEN[0])
    ent = cache.get(key)
    if ent is not None and ent.ver == ver and ent.ptr == weight.data_ptr():
        ent.used_step = _PACK_STEP[0]
        return ent.ws, True, ent
    if ent is None or ent.ptr != weight.data_ptr():
        ent = _PackEntry(ver, ent.ws if ent is not None else torch.empty((2 * Cin * Cout,), dtype=f32, device=weight.device),
                         weight.data_ptr())
        cache[key] = ent
    ent.ver = ver
    ent.used_step = _PACK_STEP[0]
    return ent.ws, False, ent


def prepack_weights(module):
    """Re-pack, in ONE launch (usip_layer_tc_pack_many), every tensor-core weight matrix of `module` that went stale since it
    was last packed (an optimizer step moved the weights) and was used by the previous step.  The train step calls this first:
    its 26 per-layer pack launches become one.  Layers that have not run yet are packed by their own first launch."""
    jobs = []
    step = _PACK_STEP[0]
    for p in module.parameters():
        cache = p.__dict__.get("_usip_tc")
        if not cache:
            continue
        ver = (p._version, _lib.WEIGHT_GEN[0])
        for ent in cache.values():
            if ent.desc is not None and ent.used_step == step and ent.ver != ver and ent.ptr == p.data_ptr():
                jobs.append((ent, ver))
    _PACK_STEP[0] = step + 1
    if not jobs:
        return 0
    arr = (ops.LayerDesc * len(jobs))(*[ent.desc for ent, _ in jobs])
    ops.check(_lib.load().usip_layer_tc_pack_many(arr, len(jobs), ops._stream()), "usip_layer_tc_pack_many")
    for ent, ver in jobs:
        ent.ver = ver
    return len(jobs)


def invalidate_packed_weights(module):
    """Drop every cached packed (hi/lo TF32) weight tile of `module`'s parameters.  The cache key follows the autograd
    version counter, which in-place writes through `.data` (legacy checkpoint loaders, EMA, weight clipping) do NOT bump:
    call this after such a write.  load_state_dict(), train()/eval() switches and the optimizer step invalidate by
    themselves (models/networks.py hooks; Adam bumps the version)."""
    for p in module.parameters():
        p.__dict__.pop("_usip_tc", None)


_TC_PREC = 1          # usip_layer_desc.precision of the wgmma 3xTF32 kernel


def _precision_for(P, Cin, Cout, use_tc, group=0):
    """Tensor-core kernel only for shapes it implements; everything else takes the fp32 SIMT kernel.  The wgmma group
    epilogue handles groups of 16/32/64/128 rows (the SIMT kernel any multiple of 4 dividing 128)."""
    if group and group not in (16, 32, 64, 128):
        return 0
    return _TC_PREC if (use_tc and Cin % 32 == 0 and Cout % 64 == 0 and P >= 1024) else 0


class LayerRunner:
    """Runs conv1x1(+BN) layers of one nn.Module tree through usip_layer_fwd / usip_bn_finalize."""

    def __init__(self, training, use_tc, dev):
        self.training = training
        self.use_tc = use_tc
        self.dev = dev

    def bn_state(self, norm, part, ntiles, count, momentum):
        C = norm.weight.numel()
        st = BNState()
        st.scale = torch.empty(C, dtype=f32, device=self.dev)
        st.shift = torch.empty(C, dtype=f32, device=self.dev)
        st.count = count
        if self.training:
            st.mean = torch.empty(C, dtype=f32, device=self.dev)
            st.invstd = torch.empty(C, dtype=f32, device=self.dev)
            ops.bn_finalize(part, ntiles, count, C, norm.weight.detach(), norm.bias.detach(), norm.eps, momentum,
                            norm.running_mean, norm.running_var, st.scale, st.shift, st.mean, st.invstd)
        else:
            st.mean = st.invstd = None
            ops.bn_eval_affine(norm.weight.detach(), norm.bias.detach(), norm.running_mean, norm.running_var, norm.eps,
                               st.scale, st.shift)
        return st

    def partials(self, P, Cout, prec=0, group=0, want_group=False):
        ntiles = ops.stat_slots(P, Cout, prec, group, want_group)
        if not self.training:
            return None, ntiles
        return torch.empty((ntiles, 2, Cout), dtype=f32, device=self.dev), ntiles

    def conv(self, layer, X, P, prev=None, epoch=None, cols=None, node=False, relu_in=None, write_y=True, addend=None,
             add_index=None, add_group=0, group=0, want_group=False, want_arg=False, name="layer"):
        """Forward of the conv1x1 `layer` over P rows: Y = act(X) W^T + b (+addend), followed by the layer's BatchNorm when
        it has one, its momentum scheduled by `epoch` (omitted where the reference calls the layer without it).  X is read
        through relu(bn(.)) with the BNState `prev` of the layer that produced it, raw when prev is None; cols: the slice
        of W's columns a concat half reads.  node=True: the per-node half of a concat, a plain GEMM (no bias, no
        BatchNorm).  Returns (Y, BNState or None, group dict or None)."""
        W, col0 = _conv_w(layer, cols)
        bias = None if node else layer.conv.bias.detach()
        norm = None if node else getattr(layer, "norm", None)
        Cout, Cin = W.shape
        Y = torch.empty((P, Cout), dtype=f32, device=self.dev) if write_y else None
        prec = _precision_for(P, Cin, Cout, self.use_tc, group if want_group else 0)
        part, ntiles = self.partials(P, Cout, prec, group, want_group) if norm is not None else (None, 0)
        grp = None
        if want_group:
            Q = P // group
            grp = dict(gmax=torch.empty((Q, Cout), dtype=f32, device=self.dev),
                       gmin=torch.empty((Q, Cout), dtype=f32, device=self.dev))
            if want_arg:
                grp["amax"] = torch.empty((Q, Cout), dtype=i32, device=self.dev)
                grp["amin"] = torch.empty((Q, Cout), dtype=i32, device=self.dev)
        ws, packed, ent = _tc_workspace(layer.conv.weight, col0, P, Cin, Cout, False) if prec else (None, False, None)
        with _Prof("%s[%dx%d->%d]" % (name, P, Cin, Cout), flops=2.0 * P * Cin * Cout,
                   precision="3xTF32 wgmma" if prec else "fp32 SIMT"):
            d = ops.layer_fwd(X, W, bias, P, Cin, Cout,
                              in_scale=None if prev is None else prev.scale, in_shift=None if prev is None else prev.shift,
                              in_relu=(prev is not None) if relu_in is None else relu_in,
                              addend=addend, add_index=add_index, add_group=add_group, Y=Y,
                              stat_partial=part,
                              gmax=None if grp is None else grp["gmax"], gmin=None if grp is None else grp["gmin"],
                              garg_max=None if grp is None else grp.get("amax"),
                              garg_min=None if grp is None else grp.get("amin"),
                              group=group, precision=prec, tc_ws=ws, tc_packed=packed)
        if ent is not None:
            ent.remember(d, W)
        st = None
        if norm is not None:
            with _Prof("bn_finalize"):
                st = self.bn_state(norm, part, ntiles, P, norm.scheduled_momentum(epoch))
        return Y, st, grp


def _knn_head_forward(R, net, AGG, C1, coords, Bp, M, Kn, epoch, keep):
    """GeneralKNNFusionModule on the nodes (layers.py:401-440) + head mlp1/2/3 + softplus (networks.py:143-154).
    AGG [Q, C1+C2]: columns [0,C1) hold the per-node feature (pool 2) on entry, columns [C1,C1+C2) receive the fused kNN
    feature.  coords (B,3,M) are the nodes the kNN runs on and the keypoint offsets are added to.  Shared by RPN_Detector /
    RPN_DetectorLite (coords = cluster means) and the ablation networks RPN_Detector_KNN / _Ball (coords = the given nodes)."""
    opt = net.opt
    dev = AGG.device
    Q = Bp * M
    G = Q * Kn
    kb = net.knnlayer_1.layers_before
    ka = net.knnlayer_1.layers_after
    C2 = ka[-1].conv.weight.shape[0]
    pool2 = AGG[:, :C1]
    # ---- GeneralKNNFusionModule (layers.py:401-440)
    with _Prof("knn_nodes"):
        knn_i = ops.knn_nodes(coords, Kn)
    W5, _ = _conv_w(kb[0])
    Cb = W5.shape[0]
    Z, _, _ = R.conv(kb[0], pool2, Q, cols=slice(3, None), node=True, name="knn_b0_node")
    Y5 = torch.empty((G, Cb), dtype=f32, device=dev)
    part5, nt5 = R.partials(G, Cb)
    with _Prof("knn_combine", nbytes=8.0 * G * Cb):
        ops.knn_combine(Z, coords, knn_i, W5, W5.stride(0), kb[0].conv.bias.detach(), Y5, part5, Bp, M, Kn, Cb)
    bn5 = R.bn_state(kb[0].norm, part5, nt5, G, kb[0].norm.scheduled_momentum(epoch))
    prev, Yprev = bn5, Y5
    saved_before = [(Y5, bn5)]
    grp_b = None
    for li in range(1, len(kb)):
        last = li == len(kb) - 1
        Yn, bnn, grp = R.conv(kb[li], Yprev, G, prev=prev, epoch=epoch, group=Kn, want_group=last, want_arg=last and keep,
                              name="knn_b%d" % li)
        prev, Yprev = bnn, Yn
        saved_before.append((Yn, bnn))
        grp_b = grp if last else grp_b
    # max over K of the activated features (layers.py:433): from group max/min of the raw output
    amax = torch.empty((Q, Cb), dtype=f32, device=dev)
    with _Prof("group_select"):
        ops.group_select(grp_b["gmax"], grp_b["gmin"], prev.scale, prev.shift, amax, Q, Cb)
    U, _, _ = R.conv(ka[0], amax, Q, cols=slice(0, Cb), node=True, name="knn_a0_node")        # max half (layers.py:435)
    Y8, bn8, _ = R.conv(ka[0], Yprev, G, prev=prev, epoch=epoch, cols=slice(Cb, None), addend=U, add_group=Kn,
                        name="knn_a0")
    saved_after = [(Y8, bn8)]
    prevA, YA = bn8, Y8
    grp_a = None
    for li in range(1, len(ka)):
        last = li == len(ka) - 1
        Yn, bnn, grp = R.conv(ka[li], YA, G, prev=prevA, epoch=epoch, group=Kn, want_group=last, want_arg=last and keep,
                              write_y=(not last) or keep, name="knn_a%d" % li)
        prevA, YA = bnn, Yn
        saved_after.append((Yn, bnn))
        grp_a = grp if last else grp_a
    ops.group_select(grp_a["gmax"], grp_a["gmin"], prevA.scale, prevA.shift, AGG[:, C1:], Q, C2)   # layers.py:438

    # ---- head (networks.py:143-154); mlp1/mlp2 are called WITHOUT epoch in the reference
    Y10, bn10, _ = R.conv(net.mlp1, AGG, Q, name="mlp1")
    Y11, bn11, _ = R.conv(net.mlp2, Y10, Q, prev=bn10, name="mlp2")
    OUT, _, _ = R.conv(net.mlp3, Y11, Q, prev=bn11, name="mlp3")
    with _Prof("head_finalize"):
        keypoints, sigmas = ops.head_finalize(OUT, coords, opt.loss_sigma_lower_bound, Bp, M)

    kctx = dict(knn_i=knn_i)
    if keep:
        kctx.update(Kn=Kn, C1=C1, C2=C2, Cb=Cb, AGG=AGG, Z=Z, before=saved_before, grp_b=grp_b, amax=amax, U=U,
                    after=saved_after, grp_a=grp_a, Y10=Y10, bn10=bn10, Y11=Y11, bn11=bn11, OUT=OUT, coords=coords)
    return keypoints, sigmas, kctx


def detector_forward(net, x, sn, node, epoch=None, use_tc=True, keep=False):
    """RPN_Detector.forward (models/networks.py:75-162) on the fused plan.

    x (B,3,N), sn (B,S,N), node (B,3,M) CUDA f32 contiguous.  Returns
    (cluster_mean (B,3,M), keypoints (B,3,M), sigmas (B,M), ctx) -- ctx holds everything backward needs when
    keep=True."""
    opt = net.opt
    assert opt.k == 1, "only k=1 is supported (every shipped config; networks.py:91-92)"
    if keep and not net.training:
        raise NotImplementedError("gradients through eval-mode BatchNorm are not part of the hot path "
                                  "(the reference only back-propagates in train mode, keypoint_detector.py:170)")
    assert len(net.knnlayer_1.layers_before) >= 2 and len(net.knnlayer_1.layers_after) >= 2
    dev = x.device
    Bp, _, N = x.shape
    M = node.shape[2]
    S = opt.surface_normal_len if opt.surface_normal_len >= 1 else 0
    Kn = opt.node_knn_k_1
    P, Q = Bp * N, Bp * M
    G = Q * Kn
    training = net.training
    R = LayerRunner(training, use_tc, dev)
    x = x.detach().contiguous(); node = node.detach().contiguous()
    snc = sn.detach().contiguous() if S else None

    # ---- grouping (som.query_topk + networks.py:87-108)
    with _Prof("som_assign", nbytes=4.0 * Bp * (4 * N + 3 * M)):
        min_idx, count = ops.som_assign(x, node)
    with _Prof("cluster_sort"):
        seg_off, perm, row_seg = ops.cluster_sort(min_idx, M)
    with _Prof("cluster_mean_decenter", nbytes=4.0 * Bp * N * (3 + S + 8 + 1)):
        cmean, X0 = ops.cluster_mean_decenter(x, snc, seg_off, perm, M, ldx=8)

    # ---- first PointNet (3+S -> C1/2 -> C1/2 -> C1/2), networks.py:111-114
    fp = net.first_pointnet.layers
    H = fp[0].conv.weight.shape[0]
    Y0, bn0, _ = R.conv(fp[0], X0, P, epoch=epoch, name="pn1.0")
    Y1, bn1, _ = R.conv(fp[1], Y0, P, prev=bn0, epoch=epoch, name="pn1.1")
    F1, _, _ = R.conv(fp[2], Y1, P, prev=bn1, name="pn1.2")
    # ---- pool 1 (index_max + gather * mask, networks.py:117-120)
    with _Prof("segmax1", nbytes=4.0 * P * H):
        pool1, arg1 = ops.segmax(F1, H, seg_off, perm, Bp, N, M, want_arg=keep)
    # ---- second PointNet on cat(first, scattered max) (networks.py:123-127): W [f; s] = Wa f + Wb s
    sp = net.second_pointnet.layers
    C1 = sp[0].conv.weight.shape[0]
    V, _, _ = R.conv(sp[0], pool1, Q, cols=slice(H, None), node=True, name="pn2.0_node")
    Y3, bn3, _ = R.conv(sp[0], F1, P, epoch=epoch, cols=slice(0, H), addend=V, add_index=row_seg, name="pn2.0")
    F2, _, _ = R.conv(sp[1], Y3, P, prev=bn3, name="pn2.1")
    # ---- pool 2 -> first C1 columns of the head input (networks.py:130-133,143)
    C2 = net.knnlayer_1.layers_after[-1].conv.weight.shape[0]
    AGG = torch.empty((Q, C1 + C2), dtype=f32, device=dev)
    pool2 = AGG[:, :C1]
    with _Prof("segmax2", nbytes=4.0 * P * C1):
        _, arg2 = ops.segmax(F2, C1, seg_off, perm, Bp, N, M, out=pool2, want_arg=keep)

    keypoints, sigmas, kctx = _knn_head_forward(R, net, AGG, C1, cmean, Bp, M, Kn, epoch, keep)
    knn_i = kctx["knn_i"]

    ctx = None
    if keep:
        ctx = dict(kctx)
        ctx.update(Bp=Bp, N=N, M=M, S=S, H=H,
                   seg_off=seg_off, perm=perm, row_seg=row_seg, min_idx=min_idx, count=count, cmean=cmean,
                   X0=X0, Y0=Y0, bn0=bn0, Y1=Y1, bn1=bn1, F1=F1, pool1=pool1, arg1=arg1, V=V,
                   Y3=Y3, bn3=bn3, F2=F2, arg2=arg2, use_tc=use_tc)
    aux = dict(min_idx=min_idx, count=count, perm=perm, seg_off=seg_off, knn_i=knn_i)
    return cmean, keypoints, sigmas, ctx, aux


# ----------------------------------------------------------------------------- losses (forward)
def chamfer_prob_forward(src, dst, sig_src, sig_dst):
    """ChamferLoss_Brute sigma branch (losses.py:79-97).  Returns (out3, saved)."""
    src = src.contiguous(); dst = dst.contiguous()
    d_sd, i_sd = ops.pairwise_min(src, dst)
    d_ds, i_ds = ops.pairwise_min(dst, src)
    out3 = ops.chamfer_prob_reduce(d_sd, i_sd, d_ds, i_ds, sig_src.contiguous(), sig_dst.contiguous())
    return out3, (d_sd, i_sd, d_ds, i_ds)


class _Bwd:
    """Small helper bundle for the backward plans: raw C-ABI calls + gradient bookkeeping."""

    def __init__(self, net, dev, use_tc):
        self.lib = _lib.load()
        self.check = _lib.check
        self.dev = dev
        self.use_tc = use_tc
        # opt.backward_precision: "3xtf32" (default, fp32-equivalent like the forward) or "tf32" -- the dgrad / wgrad GEMMs as
        # ONE TF32 MMA per MAC, the arithmetic PyTorch's default cuDNN path gives the reference's backward
        self.tf32_bwd = str(getattr(getattr(net, "opt", None), "backward_precision", "3xtf32")).lower() == "tf32"
        params = list(net.parameters())
        # usip_b200.optim.FlatAdam publishes a view of its flat gradient buffer on every parameter: accumulate straight
        # into it (autograd's own semantics for an existing .grad) and hand autograd nothing to add.  Without it (a
        # caller's own optimizer) the gradients are fresh tensors returned through autograd.
        self.direct = all(getattr(p, "_usip_flat_grad", None) is not None for p in params)
        if self.direct:
            for p in params:
                if p.grad is None or p.grad.data_ptr() != p._usip_flat_grad.data_ptr():   # module.zero_grad(set_to_none=True)
                    p._usip_flat_grad.zero_()
                    p.grad = p._usip_flat_grad
            self.grads = {p: p._usip_flat_grad for p in params}
        else:
            self.grads = {p: torch.zeros_like(p, memory_format=torch.contiguous_format) for p in params}

    def result(self, net):
        """What the autograd Function returns for the parameters."""
        if self.direct:
            return [None for _ in net.parameters()]
        return [self.grads[q] for q in net.parameters()]

    def g2d(self, w):
        g = self.grads[w]
        return g.view(g.shape[0], -1)

    def bn_bwd(self, G, Y, st, norm, P, C, relu=True, name="bn_bwd"):
        """g_y of a train-mode BN(+ReLU) layer; writes g_gamma / g_beta; returns GY [P,C] (new buffer)."""
        nt = (P + 127) // 128
        part = torch.empty((nt, 2, C), dtype=f32, device=self.dev)
        c1 = torch.empty(C, dtype=f32, device=self.dev); c2 = torch.empty(C, dtype=f32, device=self.dev)
        GY = torch.empty((P, C), dtype=f32, device=self.dev)
        s = ops._stream(); p = ops._p
        with _Prof(name, nbytes=4.0 * P * C * 5):
            self.check(self.lib.usip_bn_bwd_reduce(p(G), G.stride(0), p(Y), Y.stride(0), p(st.scale), p(st.shift), p(st.mean),
                                                   p(st.invstd), 1 if relu else 0, p(part), P, C, s), "usip_bn_bwd_reduce")
            self.check(self.lib.usip_bn_bwd_finalize(p(part), nt, P, C, p(self.grads[norm.weight]), p(self.grads[norm.bias]),
                                                     p(c1), p(c2), 1, s), "usip_bn_bwd_finalize")
            self.check(self.lib.usip_bn_bwd_apply(p(G), G.stride(0), p(Y), Y.stride(0), p(st.scale), p(st.shift), p(st.mean),
                                                  p(st.invstd), p(c1), p(c2), 1 if relu else 0, p(GY), GY.stride(0), P, C, s),
                       "usip_bn_bwd_apply")
        return GY

    def groupmax_select(self, Gout, grp, st, Qn, C, with_stats):
        """Gradient of out = max_k relu(bn(y_k)) at the selected row of each group: gz [Qn,C] (ReLU-masked), argsel [Qn,C]
        and, with_stats, the BN-backward partial sums over the selected entries."""
        p, s = ops._p, ops._stream
        gz = torch.empty((Qn, C), dtype=f32, device=self.dev)
        argsel = torch.empty((Qn, C), dtype=i32, device=self.dev)
        nt = (Qn + 127) // 128
        part = torch.empty((nt, 2, C), dtype=f32, device=self.dev) if with_stats else None
        self.check(self.lib.usip_groupmax_bwd_select(p(Gout), Gout.stride(0), p(grp["gmax"]), p(grp["gmin"]), p(grp["amax"]),
                                                     p(grp["amin"]), p(st.scale), p(st.shift), p(st.mean), p(st.invstd), p(gz),
                                                     p(argsel), p(part), Qn, C, s()), "usip_groupmax_bwd_select")
        return gz, argsel, part, nt

    def groupmax_bn_bwd(self, Gout, Y, grp, st, norm, K, Q, C):
        """g_y [Q*K, C] of a layer whose ONLY consumer is max_k relu(bn(y)) (layers.py:433,438; networks.py:572,700)."""
        p, s = ops._p, ops._stream
        G = Q * K
        gz, arg, part, nt = self.groupmax_select(Gout, grp, st, Q, C, True)
        c1 = torch.empty(C, dtype=f32, device=self.dev); c2 = torch.empty(C, dtype=f32, device=self.dev)
        self.check(self.lib.usip_bn_bwd_finalize(p(part), nt, G, C, p(self.grads[norm.weight]), p(self.grads[norm.bias]),
                                                 p(c1), p(c2), 1, s()), "usip_bn_bwd_finalize")
        GY = torch.empty((G, C), dtype=f32, device=self.dev)
        with _Prof("groupmax_bwd_apply", nbytes=8.0 * G * C):
            self.check(self.lib.usip_groupmax_bwd_apply(p(Y), Y.stride(0), p(gz), p(arg), p(st.scale), p(st.mean), p(st.invstd),
                                                        p(c1), p(c2), p(GY), GY.stride(0), K, G, C, s()), "usip_groupmax_bwd_apply")
        return GY

    def wgrad(self, GY, X, gW, P, Cout, Cin, prev=None, relu=False, name="wgrad"):
        s = ops._stream(); p = ops._p
        tc = self.use_tc and Cout % 4 == 0 and Cout >= 64 and Cin % 64 == 0 and P >= 4096
        with _Prof("%s[%dx%d->%d]" % (name, P, Cin, Cout), flops=2.0 * P * Cin * Cout,
                   precision="3xTF32 wgmma" if tc else "fp32 SIMT"):
            self.check(self.lib.usip_wgrad(p(GY), GY.stride(0), p(X), X.stride(0), None if prev is None else p(prev.scale),
                                           None if prev is None else p(prev.shift), 1 if (relu or prev is not None) else 0,
                                           p(gW), gW.stride(0), P, Cout, Cin, (4 if self.tf32_bwd else 1) if self.use_tc else 0, s), "usip_wgrad")

    def dgrad(self, GY, layer, P, cols=None, name="dgrad"):
        """G_in[P,Cin] = GY[P,Cout] @ W[Cout,Cin], W the forward weight of the conv1x1 `layer` (its columns `cols` when
        given), used transposed by the layer kernel."""
        W2d, col0 = _conv_w(layer, cols)
        Cout, Cin = W2d.shape
        out = torch.empty((P, Cin), dtype=f32, device=self.dev)
        prec = _precision_for(P, Cout, Cin, self.use_tc)
        ws, packed, ent = _tc_workspace(layer.conv.weight, col0, P, Cout, Cin, True) if prec else (None, False, None)
        with _Prof("%s[%dx%d->%d]" % (name, P, Cout, Cin), flops=2.0 * P * Cin * Cout,
                   precision="3xTF32 wgmma" if prec else "fp32 SIMT"):
            d = ops.layer_fwd(GY, W2d, None, P, Cout, Cin, Y=out, precision=prec, w_transposed=True, tc_ws=ws, tc_packed=packed,
                              debug_flags=8 if (self.tf32_bwd and prec) else 0)
        if ent is not None:
            ent.remember(d, W2d)
        return out

    def colsum(self, G, out, P, C):
        self.check(self.lib.usip_colsum(ops._p(G), G.stride(0), ops._p(out), P, C, ops._stream()), "usip_colsum")

    def conv_bwd(self, GY, layer, P, X, prev=None, norm=None, name="", in_name="", cols=None, grad_in=True):
        """Backward of the conv1x1 `layer` (y = act(X) W^T + b over P rows) from GY [P, Cout], the gradient of its pre-BN
        output (of its output when it has no BatchNorm).  X: the saved input, read through relu(bn(.)) with the BNState
        `prev` of the layer that produced it, or raw when prev is None; cols: the slice of W's columns a concat half reads.
        Accumulates the weight (and bias) gradient and returns the gradient of act(X) -- or, given the input layer's
        BatchNorm `norm`, of that layer's pre-BN output (profile record "bn_bwd_<in_name>"); GY is consumed then, its buffer
        released before bn_bwd allocates the next one.  grad_in=False (a plan's first layer): the weight gradient only."""
        gW = self.g2d(layer.conv.weight)
        if cols is not None:
            gW = gW[:, cols]
        Cout, Cin = gW.shape
        self.wgrad(GY, X, gW, P, Cout, Cin, prev=prev, name="wgrad_" + name)
        # a conv bias in front of a train-mode BatchNorm receives exactly zero gradient (BN removes the mean): it stays
        # zero-initialised in self.grads
        if getattr(layer, "norm", None) is None:
            self.colsum(GY, self.grads[layer.conv.bias], P, Cout)
        if not grad_in:
            return None
        G_in = self.dgrad(GY, layer, P, cols, name="dgrad_" + name)
        if norm is None:
            return G_in
        GY.set_()                                   # frees GY's buffer even though the caller still holds the tensor
        return self.bn_bwd(G_in, X, prev, norm, P, Cin, name="bn_bwd_" + in_name)

    def max_concat_bwd(self, GY, layer, X, prev, grp, amax, dense, node, K, Q, name):
        """Backward of a layer on cat(a, broadcast max over each group of K rows of a), a = relu(bn(X)) (layers.py:435,
        networks.py:377): y = a W[:, dense]^T + (amax W[:, node]^T)[row / K] + b, from GY [Q*K, Cout], the gradient of
        its pre-BN output, which is consumed.  grp / prev: the group max/min/arg and BNState of the layer that produced
        X.  Returns the gradient [Q*K, Cin] of a, the max path scattered to each group's selected row (the ReLU mask is
        applied by the bn_bwd that follows)."""
        p, s = ops._p, ops._stream
        Cout = GY.shape[1]
        G_a = self.conv_bwd(GY, layer, Q * K, X, prev, cols=dense, name=name)
        G_U = torch.empty((Q, Cout), dtype=f32, device=self.dev)
        self.check(self.lib.usip_group_sum(p(GY), GY.stride(0), p(G_U), G_U.stride(0), K, Q, Cout, s()), "usip_group_sum")
        GY.set_()                                   # frees GY's buffer even though the caller still holds the tensor
        G_amax = self.conv_bwd(G_U, layer, Q, amax, cols=node, name=name + "_node")
        Cin = G_amax.shape[1]
        _, arg, _, _ = self.groupmax_select(G_amax, grp, prev, Q, Cin, False)
        self.check(self.lib.usip_groupmax_scatter_add(p(G_a), G_a.stride(0), p(G_amax), p(arg), K, Q, Cin, s()),
                   "usip_groupmax_scatter_add")
        return G_a


def _knn_head_backward(bw, net, ctx, g_kp, g_sig):
    """Backward of _knn_head_forward: parameter gradients of mlp1/2/3 and knnlayer_1 are accumulated into bw.grads; returns
    the gradient [Q, C1] of the per-node feature that entered AGG[:, :C1] (head path + kNN path)."""
    dev = bw.dev
    Bp, M = ctx["Bp"], ctx["M"]
    Kn, C1, C2, Cb = ctx["Kn"], ctx["C1"], ctx["C2"], ctx["Cb"]
    Q = Bp * M
    G = Q * Kn
    lib, check, p, s = bw.lib, bw.check, ops._p, ops._stream
    kb, ka = net.knnlayer_1.layers_before, net.knnlayer_1.layers_after
    g_kp = None if g_kp is None else g_kp.contiguous()
    g_sig = None if g_sig is None else g_sig.contiguous()
    # ---- head (networks.py:143-154)
    G_OUT = torch.empty((Q, 4), dtype=f32, device=dev)
    check(lib.usip_head_bwd(p(g_kp), p(g_sig), p(ctx["OUT"]), ctx["OUT"].stride(0), p(G_OUT), Bp, M, s()), "usip_head_bwd")
    GY = bw.conv_bwd(G_OUT, net.mlp3, Q, ctx["Y11"], ctx["bn11"], net.mlp2.norm, "mlp3", "mlp2")
    GY = bw.conv_bwd(GY, net.mlp2, Q, ctx["Y10"], ctx["bn10"], net.mlp1.norm, "mlp2", "mlp1")
    G_AGG = bw.conv_bwd(GY, net.mlp1, Q, ctx["AGG"], name="mlp1")          # [Q, C1+C2]

    # ---- kNN fusion, layers_after (layers.py:435-438), last -> first
    Ya_last, bna_last = ctx["after"][-1]
    GY = bw.groupmax_bn_bwd(G_AGG[:, C1:], Ya_last, ctx["grp_a"], bna_last, ka[-1].norm, Kn, Q, C2)
    for li in range(len(ka) - 1, 0, -1):
        GY = bw.conv_bwd(GY, ka[li], G, *ctx["after"][li - 1], ka[li - 1].norm, "knn_a%d" % li, "knn_a%d" % (li - 1))
    # ka[0] on cat(broadcast max, a7): the max half is first
    Yb_last, bnb_last = ctx["before"][-1]
    GY = bw.max_concat_bwd(GY, ka[0], Yb_last, bnb_last, ctx["grp_b"], ctx["amax"], slice(Cb, None), slice(0, Cb), Kn, Q,
                           "knn_a0")
    # ---- layers_before, last -> 1
    GY = bw.bn_bwd(GY, Yb_last, bnb_last, kb[-1].norm, G, Cb, name="bn_bwd_knn_b%d" % (len(kb) - 1))
    for li in range(len(kb) - 1, 0, -1):
        GY = bw.conv_bwd(GY, kb[li], G, *ctx["before"][li - 1], kb[li - 1].norm, "knn_b%d" % li, "knn_b%d" % (li - 1))
    # kb[0] = knn_combine: Y5 = Z[nbr] + Wxyz*delta + b, Z = pool2 Wf^T
    gW5 = bw.g2d(kb[0].conv.weight)
    G_Z = torch.zeros((Q, Cb), dtype=f32, device=dev)
    with _Prof("knn_combine_bwd"):
        check(lib.usip_knn_combine_bwd(p(GY), GY.stride(0), p(ctx["coords"]), p(ctx["knn_i"]), p(G_Z), G_Z.stride(0), p(gW5),
                                       gW5.stride(0), Bp, M, Kn, Cb, s()), "usip_knn_combine_bwd")
    del GY
    G_pool2 = bw.conv_bwd(G_Z, kb[0], Q, ctx["AGG"][:, :C1], cols=slice(3, None), name="knn_b0_node")     # [Q, C1]
    G_pool2 += G_AGG[:, :C1]                                               # tiny [Q,C1] plumbing add
    return G_pool2


def detector_backward(net, ctx, g_kp, g_sig):
    """Backward of detector_forward.  Returns the gradients of net.parameters() in order."""
    dev = ctx["cmean"].device
    Bp, N, M = ctx["Bp"], ctx["N"], ctx["M"]
    H, C1 = ctx["H"], ctx["C1"]
    P, Q = Bp * N, Bp * M
    bw = _Bwd(net, dev, ctx["use_tc"])
    lib, check, p, s = bw.lib, bw.check, ops._p, ops._stream
    fp, sp = net.first_pointnet.layers, net.second_pointnet.layers

    G_pool2 = _knn_head_backward(bw, net, ctx, g_kp, g_sig)

    # ---- pool 2 un-pool (index_max gather backward), second PointNet
    G_F2 = torch.zeros((P, C1), dtype=f32, device=dev)
    check(lib.usip_unpool_scatter(p(G_F2), G_F2.stride(0), p(G_pool2), G_pool2.stride(0), p(ctx["arg2"]), Q, C1, 0, s()),
          "usip_unpool_scatter")
    GY3 = bw.conv_bwd(G_F2, sp[1], P, ctx["Y3"], ctx["bn3"], sp[0].norm, "pn2.1", "pn2.0")
    # pn2.0 on cat(F1, un-pooled pool1): the per-node half's gradient is the segment sum
    G_F1 = bw.conv_bwd(GY3, sp[0], P, ctx["F1"], cols=slice(0, H), name="pn2.0")                     # [P, H]
    G_V = torch.empty((Q, C1), dtype=f32, device=dev)
    check(lib.usip_seg_sum(p(GY3), GY3.stride(0), p(ctx["seg_off"]), p(G_V), G_V.stride(0), Bp, N, M, C1, s()), "usip_seg_sum")
    del GY3
    G_pool1 = bw.conv_bwd(G_V, sp[0], Q, ctx["pool1"], cols=slice(H, None), name="pn2.0_node")     # [Q, H]
    check(lib.usip_unpool_scatter(p(G_F1), G_F1.stride(0), p(G_pool1), G_pool1.stride(0), p(ctx["arg1"]), Q, H, 1, s()),
          "usip_unpool_scatter")
    # ---- first PointNet
    GY = bw.conv_bwd(G_F1, fp[2], P, ctx["Y1"], ctx["bn1"], fp[1].norm, "pn1.2", "pn1.1")
    GY = bw.conv_bwd(GY, fp[1], P, ctx["Y0"], ctx["bn0"], fp[0].norm, "pn1.1", "pn1.0")
    bw.conv_bwd(GY, fp[0], P, ctx["X0"], name="pn1.0", grad_in=False)
    return bw.result(net)


def _combine_sub_groups(grp, ratio, sub, keep):
    """Reduce the sub-group max / min (and, with keep, their args) of a group-max layer to whole groups, in place."""
    with _Prof("group_max_combine"):
        if keep:
                grp["gmax"], grp["gmin"], grp["amax"], grp["amin"] = ops.group_max_combine_arg(
                grp["gmax"], ratio, grp["gmin"], grp["amax"], grp["amin"], sub)
        else:
            grp["gmax"], grp["gmin"] = ops.group_max_combine(grp["gmax"], ratio, grp["gmin"])


def _group_net_forward(R, net, rows, Bp, M, K, keep, out=None):
    """The grouped PointNet shared by DescriptorLiteOld (networks.py:375-381) and the ablation detectors
    RPN_Detector_KNN / RPN_Detector_Ball (networks.py:567-572, 695-700):
        conv1 -> conv2 -> conv3 -> max_k -> conv4 on cat(y, broadcast max) -> conv5 -> max_k
    on point-major rows [Bp*M*K, ld] of the gathered, decentred groups.  conv1..conv4 carry BN+ReLU; conv5 is linear in the
    descriptor (the raw group max is returned) and BN+ReLU in the detectors (max_k relu(bn(.)) is written to `out`).
    The reference calls these convolutions WITHOUT epoch: their BN momentum never decays.
    Balls of more than 128 rows (K a multiple of 64) take the layer epilogue's group max over 64-row sub-groups and reduce
    each run of K/64 of them with usip_group_max_combine -- with keep, usip_group_max_combine_arg, whose args are rows of
    the whole ball, so the backward sees the same [Q, C] amax / amin as for a direct group max."""
    dev = rows.device
    G, Q = Bp * M * K, Bp * M
    sub = K if K <= 128 else 64
    if K % sub != 0:
        raise NotImplementedError("group of %d rows: groups above 128 must be a multiple of 64" % K)
    c1, c2, c3, c4, c5 = net.conv1, net.conv2, net.conv3, net.conv4, net.conv5
    D = c3.conv.weight.shape[0]
    Y1, bn1, _ = R.conv(c1, rows, G, name="grp.conv1")
    Y2, bn2, _ = R.conv(c2, Y1, G, prev=bn1, name="grp.conv2")
    Y3, bn3, grp3 = R.conv(c3, Y2, G, prev=bn2, group=sub, want_group=True, want_arg=keep, name="grp.conv3")
    if sub != K:
        _combine_sub_groups(grp3, K // sub, sub, keep)
    amax = torch.empty((Q, D), dtype=f32, device=dev)
    ops.group_select(grp3["gmax"], grp3["gmin"], bn3.scale, bn3.shift, amax, Q, D)          # y_first_max (networks.py:377)
    C4 = c4.conv.weight.shape[0]
    U, _, _ = R.conv(c4, amax, Q, cols=slice(D, None), node=True, name="grp.conv4_node")   # cat(y_first, max): max is LAST
    Y4, bn4, _ = R.conv(c4, Y3, G, prev=bn3, cols=slice(0, D), addend=U, add_group=K, name="grp.conv4")
    last_bn = getattr(c5, "norm", None) is not None
    Y5, bn5, grp5 = R.conv(c5, Y4, G, prev=bn4, group=sub, want_group=True, want_arg=keep, write_y=last_bn and keep,
                           name="grp.conv5")
    if sub != K:
        if not last_bn:                                    # a linear conv5 is pooled by its max only
            grp5["gmin"] = grp5["amin"] = None
        _combine_sub_groups(grp5, K // sub, sub, keep)
    result = grp5["gmax"]
    if last_bn:
        C5 = c5.conv.weight.shape[0]
        if out is None:
            out = torch.empty((Q, C5), dtype=f32, device=dev)
        ops.group_select(grp5["gmax"], grp5["gmin"], bn5.scale, bn5.shift, out, Q, C5)
        result = out
    gctx = dict(D=D)
    if keep:
        gctx.update(Bp=Bp, M=M, K=K, C4=C4, rows=rows, Y1=Y1, bn1=bn1, Y2=Y2, bn2=bn2, Y3=Y3, bn3=bn3, grp3=grp3, amax=amax,
                    Y4=Y4, bn4=bn4, Y5=Y5, bn5=bn5, grp5=grp5)
    return result, gctx


ABLATION_K = 64             # networks.py:554, 680: `k = 64` is hard-coded in both ablation detectors
ABLATION_RADIUS = 2.0       # networks.py:681


def ablation_forward(net, x, sn, node, epoch=None, use_tc=True, keep=False, mode="knn"):
    """RPN_Detector_KNN.forward (models/networks.py:545-608, mode="knn") / RPN_Detector_Ball.forward (:671-738, mode="ball")
    on the fused plan: group the points around the GIVEN nodes (64 nearest points / first 64 points within radius 2, both
    without the (B,M,N) distance matrix), the grouped PointNet conv1..conv5 with two max-pools over the group, then the same
    node-level kNN fusion module and head as RPN_Detector -- on the nodes themselves, which are also returned in place of the
    recomputed cluster means.  Returns (node, keypoints, sigmas, ctx)."""
    opt = net.opt
    if keep and not net.training:
        raise NotImplementedError("gradients through eval-mode BatchNorm are not part of the hot path")
    dev = x.device
    Bp, _, N = x.shape
    M = node.shape[2]
    S = opt.surface_normal_len if opt.surface_normal_len >= 1 else 0
    Kn = opt.node_knn_k_1
    K = ABLATION_K
    Q = Bp * M
    R = LayerRunner(net.training, use_tc, dev)
    x = x.detach().contiguous(); node = node.detach().contiguous()
    snc = sn.detach().contiguous() if S else None
    with _Prof("group_%s" % mode):
        if mode == "knn":
            _, _, rows = ops.knn_group(x, snc, node, K, want_group=False, rows_ld=8)
        else:
            _, _, rows = ops.ball_group(x, snc, node, ABLATION_RADIUS, K, want_group=False, rows_ld=8)
    C1 = net.conv5.conv.weight.shape[0]
    C2 = net.knnlayer_1.layers_after[-1].conv.weight.shape[0]
    AGG = torch.empty((Q, C1 + C2), dtype=f32, device=dev)
    _, gctx = _group_net_forward(R, net, rows, Bp, M, K, keep, out=AGG[:, :C1])      # second_pn_out_max (networks.py:572)
    keypoints, sigmas, kctx = _knn_head_forward(R, net, AGG, C1, node, Bp, M, Kn, epoch, keep)
    ctx = None
    if keep:
        ctx = dict(kctx)                                        # (both plans keep an "amax": the grouped PointNet's state is nested)
        ctx.update(Bp=Bp, M=M, use_tc=use_tc, group_net=gctx)
    return node, keypoints, sigmas, ctx


def ablation_backward(net, ctx, g_kp, g_sig):
    """Backward of ablation_forward: gradients of net.parameters() in order (points and nodes carry none)."""
    dev = ctx["AGG"].device
    gctx = ctx["group_net"]
    Bp, M, K = ctx["Bp"], ctx["M"], gctx["K"]
    bw = _Bwd(net, dev, ctx["use_tc"])
    G_pool = _knn_head_backward(bw, net, ctx, g_kp, g_sig)                  # gradient of max_k relu(bn5(conv5)) [Q, C1]
    C5 = net.conv5.conv.weight.shape[0]
    GY5 = bw.groupmax_bn_bwd(G_pool, gctx["Y5"], gctx["grp5"], gctx["bn5"], net.conv5.norm, K, Bp * M, C5)
    _group_net_backward(bw, net, gctx, GY5)
    return bw.result(net)


def descriptor_forward(net, x, sn, keypoints, epoch, permute_idx, use_tc=True, keep=False):
    """DescriptorLiteOld.forward (models/networks.py:333-385) on the fused plan.
    Returns (descriptor (B,C,M), x_features (B,3+S,M,K), ctx) -- ctx holds what descriptor_backward needs (keep=True)."""
    opt = net.opt
    dev = x.device
    if keep and not net.training:
        raise NotImplementedError("gradients through eval-mode BatchNorm are not part of the hot path "
                                  "(the reference only back-propagates in train mode, keypoint_descriptor.py:138)")
    Bp, M, K = x.shape[0], keypoints.shape[2], opt.ball_nsamples
    R = LayerRunner(net.training, use_tc, dev)
    feats, rows = _descriptor_balls(opt, x, sn, keypoints, permute_idx)
    gmax5, gctx = _group_net_forward(R, net, rows, Bp, M, K, keep, out=None)
    D = gctx["D"]
    desc = torch.empty((Bp, D, M), dtype=f32, device=dev)
    _lib.check(_lib.load().usip_l2norm_to_bcm(ops._p(gmax5), gmax5.stride(0), ops._p(desc), None, Bp, M, D,
                                              ops._stream()), "usip_l2norm_to_bcm")
    ctx = None
    if keep:
        ctx = dict(gctx)
        ctx.update(use_tc=use_tc)
    return desc, feats, ctx


def _descriptor_balls(opt, x, sn, keypoints, permute_idx):
    """networks.py:345-373: the balls of both descriptors -> (x_features (B,3+S,M,K), point-major rows [B*M*K, 8])."""
    Bp, _, N = x.shape
    M = keypoints.shape[2]
    K = opt.ball_nsamples
    S = opt.surface_normal_len if opt.surface_normal_len > 0 else 0
    # permute the points on the host-drawn permutation: the ball query keeps the FIRST K hits in index order
    x = x.detach()[:, :, permute_idx].contiguous()
    snp = sn.detach()[:, :, permute_idx].contiguous() if S else None
    kp = keypoints.detach().contiguous()
    with _Prof("ball_group", nbytes=4.0 * Bp * (N * (3 + S) + 3 * M + M * K + (3 + S) * M * K)):
        _, feats, rows = ops.ball_group(x, snp, kp, float(opt.ball_radius), K, want_group=True, rows_ld=8)
    return feats, rows


def descriptor_global_forward(net, x, sn, keypoints, epoch, permute_idx, use_tc=True, keep=False):
    """DescriptorLiteOldGlobal.forward (models/networks.py:433-479) on the fused plan.  The grouped PointNet
    is DescriptorLiteOld's; then PPFNet's global context:
        g = max over the M keypoints of each cloud of the raw conv5 max          (usip_group_max_combine, ratio M)
        fc1 on cat(desc, g) = desc W1[:, :D]^T + (g W1[:, D:]^T)[row / M] + b  -> BN + ReLU
        fc2 -> BN + ReLU, fc3 linear, L2 normalisation.
    The EquivariantLayers are called without epoch, like the convolutions: their BN momentum never decays.
    Returns (descriptor (B,D,M), x_features (B,3+S,M,K), ctx) -- ctx holds what descriptor_global_backward needs (keep=True:
    every pool's arg, the global max's keypoint included)."""
    opt = net.opt
    dev = x.device
    if keep and not net.training:
        raise NotImplementedError("gradients through eval-mode BatchNorm are not part of the hot path "
                                  "(the reference only back-propagates in train mode, keypoint_descriptor.py:466)")
    Bp, M, K = x.shape[0], keypoints.shape[2], opt.ball_nsamples
    Q = Bp * M
    R = LayerRunner(net.training, use_tc, dev)
    feats, rows = _descriptor_balls(opt, x, sn, keypoints, permute_idx)
    local, gctx = _group_net_forward(R, net, rows, Bp, M, K, keep, out=None)         # [Q, D] raw max of conv5
    D = gctx["D"]
    with _Prof("global_max"):
        if keep:
            glob, _, glob_arg, _ = ops.group_max_combine_arg(local, M)                # [Bp, D], keypoint of each max
        else:
            glob, _ = ops.group_max_combine(local, M)
    f1, f2, f3 = net.fc1, net.fc2, net.fc3
    U, _, _ = R.conv(f1, glob, Bp, cols=slice(D, None), node=True, name="fc1_global")   # cat(desc, global): global is LAST
    Y1, bn1, _ = R.conv(f1, local, Q, cols=slice(0, D), addend=U, add_group=M, name="fc1")
    Y2, bn2, _ = R.conv(f2, Y1, Q, prev=bn1, name="fc2")
    OUT, _, _ = R.conv(f3, Y2, Q, prev=bn2, name="fc3")
    desc = torch.empty((Bp, OUT.shape[1], M), dtype=f32, device=dev)
    _lib.check(_lib.load().usip_l2norm_to_bcm(ops._p(OUT), OUT.stride(0), ops._p(desc), None, Bp, M, OUT.shape[1],
                                              ops._stream()), "usip_l2norm_to_bcm")
    ctx = None
    if keep:
        ctx = dict(gctx)
        ctx.update(use_tc=use_tc, local=local, glob=glob, glob_arg=glob_arg, Y1f=Y1, bn1f=bn1, Y2f=Y2, bn2f=bn2, OUT=OUT)
    return desc, feats, ctx


def _group_net_backward(bw, net, ctx, GY5):
    """Backward of _group_net_forward from GY5 [G, C5], the gradient of conv5's raw output rows, which is consumed
    (parameter gradients are accumulated into bw.grads; points / centres carry no gradient)."""
    Bp, M, K, D = ctx["Bp"], ctx["M"], ctx["K"], ctx["D"]
    Q, G = Bp * M, Bp * M * K
    c1, c2, c3, c4, c5 = net.conv1, net.conv2, net.conv3, net.conv4, net.conv5
    GY = bw.conv_bwd(GY5, c5, G, ctx["Y4"], ctx["bn4"], c4.norm, "grp.conv5", "grp.conv4")
    # conv4 on cat(a3, broadcast max): the max half is last
    GY = bw.max_concat_bwd(GY, c4, ctx["Y3"], ctx["bn3"], ctx["grp3"], ctx["amax"], slice(0, D), slice(D, None), K, Q,
                           "grp.conv4")
    GY = bw.bn_bwd(GY, ctx["Y3"], ctx["bn3"], c3.norm, G, D, name="bn_bwd_grp.conv3")
    GY = bw.conv_bwd(GY, c3, G, ctx["Y2"], ctx["bn2"], c2.norm, "grp.conv3", "grp.conv2")
    GY = bw.conv_bwd(GY, c2, G, ctx["Y1"], ctx["bn1"], c1.norm, "grp.conv2", "grp.conv1")
    bw.conv_bwd(GY, c1, G, ctx["rows"], name="grp.conv1", grad_in=False)


def descriptor_backward(net, ctx, g_desc):
    """Backward of descriptor_forward (points / keypoints carry no gradient): gradients of net.parameters() in order.

    desc = l2norm(max_k conv5(a4)),  a4 = relu(bn4(a3 WA^T + (amax WB^T)[row/K])),  amax = max_k a3,
    a3 = relu(bn3(conv3(a2))), a2 = relu(bn2(conv2(a1))), a1 = relu(bn1(conv1(rows)))      (networks.py:375-383)."""
    dev = g_desc.device
    Bp, M, K, D = ctx["Bp"], ctx["M"], ctx["K"], ctx["D"]
    Q, G = Bp * M, Bp * M * K
    bw = _Bwd(net, dev, ctx["use_tc"])
    lib, check, p, s = bw.lib, bw.check, ops._p, ops._stream
    grp5 = ctx["grp5"]
    # ---- l2 normalisation and the max over the ball (conv5 is linear: the max of the raw output routes to its arg row)
    G_y = torch.empty((Q, D), dtype=f32, device=dev)
    check(lib.usip_l2norm_bwd(p(g_desc.contiguous()), p(grp5["gmax"]), grp5["gmax"].stride(0), p(G_y), G_y.stride(0), Bp, M, D, s()),
          "usip_l2norm_bwd")
    GY5 = torch.zeros((G, D), dtype=f32, device=dev)
    check(lib.usip_groupmax_scatter_add(p(GY5), GY5.stride(0), p(G_y), p(grp5["amax"]), K, Q, D, s()), "usip_groupmax_scatter_add")
    _group_net_backward(bw, net, ctx, GY5)
    # conv1..conv4 biases sit in front of a train-mode BatchNorm: exactly zero gradient (left zero-initialised)
    return bw.result(net)


def descriptor_global_backward(net, ctx, g_desc):
    """Backward of descriptor_global_forward (points / keypoints carry no gradient): gradients of net.parameters() in order.

    desc = l2norm(fc3(a2)),  a2 = relu(bn2(fc2(a1))),  a1 = relu(bn1(local W1A^T + (g W1B^T)[row/M])),
    g = max over the cloud's M keypoints of local,  local = max_k conv5(a4) (the grouped PointNet, networks.py:433-479)."""
    dev = g_desc.device
    Bp, M, K, D = ctx["Bp"], ctx["M"], ctx["K"], ctx["D"]
    Q, G = Bp * M, Bp * M * K
    bw = _Bwd(net, dev, ctx["use_tc"])
    lib, check, p, s = bw.lib, bw.check, ops._p, ops._stream
    f1, f2, f3 = net.fc1, net.fc2, net.fc3
    OUT = ctx["OUT"]
    # ---- L2 normalisation, fc3 (linear), fc2
    G_out = torch.empty((Q, OUT.shape[1]), dtype=f32, device=dev)
    check(lib.usip_l2norm_bwd(p(g_desc.contiguous()), p(OUT), OUT.stride(0), p(G_out), G_out.stride(0), Bp, M, OUT.shape[1],
                              s()), "usip_l2norm_bwd")
    GY = bw.conv_bwd(G_out, f3, Q, ctx["Y2f"], ctx["bn2f"], f2.norm, "fc3", "fc2")
    GY = bw.conv_bwd(GY, f2, Q, ctx["Y1f"], ctx["bn1f"], f1.norm, "fc2", "fc1")
    # ---- fc1 on cat(local, broadcast global max): the dense half, then the global half summed over each cloud's keypoints
    local, glob = ctx["local"], ctx["glob"]
    G_local = bw.conv_bwd(GY, f1, Q, local, cols=slice(0, D), name="fc1")                       # [Q, D]
    G_U = torch.empty((Bp, GY.shape[1]), dtype=f32, device=dev)
    check(lib.usip_group_sum(p(GY), GY.stride(0), p(G_U), G_U.stride(0), M, Bp, GY.shape[1], s()), "usip_group_sum")
    GY.set_()                                   # frees GY's buffer even though the caller still holds the tensor
    G_glob = bw.conv_bwd(G_U, f1, Bp, glob, cols=slice(D, None), name="fc1_global")             # [Bp, D]
    # the global max is of the raw local descriptors: its gradient goes to each cloud's arg-max keypoint
    check(lib.usip_groupmax_scatter_add(p(G_local), G_local.stride(0), p(G_glob), p(ctx["glob_arg"]), M, Bp, D, s()),
          "usip_groupmax_scatter_add")
    # ---- the max over each ball (conv5 is linear: the max of the raw output routes to its arg row)
    GY5 = torch.zeros((G, D), dtype=f32, device=dev)
    check(lib.usip_groupmax_scatter_add(p(GY5), GY5.stride(0), p(G_local), p(ctx["grp5"]["amax"]), K, Q, D, s()),
          "usip_groupmax_scatter_add")
    del G_local
    _group_net_backward(bw, net, ctx, GY5)
    return bw.result(net)
