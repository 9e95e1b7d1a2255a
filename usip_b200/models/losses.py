"""Host-side mirror of the hot-path losses of models/losses.py (same class names / signatures / returns):

  ChamferLoss_Brute            losses.py:44-99    probabilistic chamfer (sigma branch) + plain branch
  KeypointOnPCLoss             losses.py:102-116  (point_to_point -> SingleSideChamferLoss_Brute)
  SingleSideChamferLoss_Brute  losses.py:119-143
  DescPairScanLoss             losses.py:190-237  outdoor descriptor triplet loss
  DescCGFLoss                  losses.py:240-369  indoor descriptor triplet loss (CGF sampling)

The (B,3,M,N) / (B,M,N) temporaries of the reference are never built: one tiled pairwise-L2 arg-min kernel
(usip_pairwise_min_f32) serves all three, the reductions and the backward passes are small fused kernels.  The descriptor
losses likewise never build their (B,C,M,M) descriptor differences.
"""
import ctypes

import torch
import torch.nn as nn

from usip_b200 import _lib, ops
from usip_b200.ops import _p, _stream


# ---- functional cores: used by the autograd Functions below and by the autograd-free train step of ModelDetector ----
def pairmin_bwd(a, b, d, arg, g, want_b=False, scale=1.0):
    """Gradient of d_i = min_j ||a_i - b_j|| w.r.t. a (and b): g (B,Ma) upstream, times `scale`."""
    B, _, Ma = a.shape
    ga = torch.empty_like(a)
    gb = torch.zeros_like(b) if want_b else None
    _lib.check(_lib.load().usip_pairwise_min_bwd(_p(a), _p(b), _p(d), _p(arg), _p(g.contiguous()), float(scale), _p(ga),
                                                 _p(gb), B, Ma, b.shape[2], _stream()), "usip_pairwise_min_bwd")
    return ga, gb


def chamfer_prob_fwd(src, dst, sig_src, sig_dst):
    """ChamferLoss_Brute sigma branch (losses.py:79-97): -> (out3 = [loss, pure, weighted], saved)."""
    d_sd, i_sd = ops.pairwise_min(src, dst)
    d_ds, i_ds = ops.pairwise_min(dst, src)
    out3 = ops.chamfer_prob_reduce(d_sd, i_sd, d_ds, i_ds, sig_src, sig_dst)
    return out3, (src, dst, sig_src, sig_dst, d_sd, i_sd, d_ds, i_ds)


def chamfer_prob_bwd(saved, g_loss):
    """-> (g_src, g_dst, g_sig_src, g_sig_dst) for the upstream gradient g_loss (1-element tensor) of the chamfer loss."""
    src, dst, sig_src, sig_dst, d_sd, i_sd, d_ds, i_ds = saved
    B, _, M = src.shape
    N = dst.shape[2]
    g_src = torch.zeros_like(src); g_dst = torch.zeros_like(dst)
    g_ss = torch.zeros_like(sig_src); g_sd = torch.zeros_like(sig_dst)
    gout = g_loss.reshape(1).to(torch.float32).contiguous()
    _lib.check(_lib.load().usip_chamfer_prob_bwd(_p(src), _p(dst), _p(sig_src), _p(sig_dst), _p(d_sd), _p(i_sd),
                                                 _p(d_ds), _p(i_ds), _p(gout), _p(g_src), _p(g_dst), _p(g_ss),
                                                 _p(g_sd), B, M, N, _stream()), "usip_chamfer_prob_bwd")
    return g_src, g_dst, g_ss, g_sd


def transform_bwd(g, R, scale):
    g = g.contiguous()
    B, _, M = g.shape
    gk = torch.empty_like(g)
    _lib.check(_lib.load().usip_transform_points_bwd(_p(g), _p(R), _p(scale), _p(gk), B, M, _stream()),
               "usip_transform_points_bwd")
    return gk


def point_on_surface_fwd(kp, pc, sn):
    B, _, M = kp.shape
    _, arg = ops.pairwise_min(kp, pc)                       # nearest cloud point of every keypoint (not differentiated)
    loss = torch.empty((B, M), dtype=torch.float32, device=kp.device)
    _lib.check(_lib.load().usip_point_on_surface(_p(kp), _p(pc), _p(sn), _p(arg), None, _p(loss), None, B, M, pc.shape[2],
                                                 sn.shape[1], _stream()), "usip_point_on_surface")
    return loss, arg


def point_on_surface_bwd(kp, pc, sn, arg, g):
    B, _, M = kp.shape
    g_kp = torch.empty_like(kp)
    _lib.check(_lib.load().usip_point_on_surface(_p(kp), _p(pc), _p(sn), _p(arg), _p(g.reshape(B, M).contiguous().float()),
                                                 None, _p(g_kp), B, M, pc.shape[2], sn.shape[1], _stream()),
               "usip_point_on_surface")
    return g_kp


class _PairMinFn(torch.autograd.Function):
    """min_j ||a_i - b_j|| (B,Ma); differentiable w.r.t. both point sets (sub-gradient 0 at d == 0)."""

    @staticmethod
    def forward(ctx, a, b):
        a = a.contiguous(); b = b.contiguous()
        from usip_b200 import engine
        with engine._Prof("pairwise_min[%dx%dx%d]" % (a.shape[0], a.shape[2], b.shape[2])):
            d, arg = ops.pairwise_min(a, b)
        ctx.save_for_backward(a, b, d, arg)
        return d

    @staticmethod
    def backward(ctx, g):
        a, b, d, arg = ctx.saved_tensors
        ga, gb = pairmin_bwd(a, b, d, arg, g, want_b=ctx.needs_input_grad[1])
        return (ga if ctx.needs_input_grad[0] else None), gb


class _ChamferProbFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, dst, sig_src, sig_dst):
        src = src.contiguous(); dst = dst.contiguous()
        sig_src = sig_src.contiguous(); sig_dst = sig_dst.contiguous()
        from usip_b200 import engine
        with engine._Prof("chamfer_prob"):
            out3, saved = chamfer_prob_fwd(src, dst, sig_src, sig_dst)
        ctx.save_for_backward(*saved)
        loss, pure, weighted = out3[0], out3[1], out3[2]
        ctx.mark_non_differentiable(pure, weighted)
        return loss, pure, weighted

    @staticmethod
    def backward(ctx, g_loss, g_pure, g_weighted):
        return chamfer_prob_bwd(ctx.saved_tensors, g_loss)


class _TransformFn(torch.autograd.Function):
    """R @ kp * scale + shift (keypoint_detector.py:182-184); gradient only w.r.t. kp."""

    @staticmethod
    def forward(ctx, kp, R, scale, shift):
        kp = kp.contiguous(); R = R.contiguous()
        scale = scale.reshape(-1).contiguous(); shift = shift.reshape(shift.shape[0], 3).contiguous()
        ctx.save_for_backward(R, scale)
        return ops.transform_points(kp, R, scale, shift)

    @staticmethod
    def backward(ctx, g):
        R, scale = ctx.saved_tensors
        return transform_bwd(g, R, scale), None, None, None


class _MeanScaleFn(torch.autograd.Function):
    """mean(d) * alpha (keypoint_detector.py:193-197)."""

    @staticmethod
    def forward(ctx, d, alpha):
        ctx.alpha = alpha; ctx.n = d.numel(); ctx.shape = d.shape
        return ops.mean_scale(d.contiguous(), alpha)[0]

    @staticmethod
    def backward(ctx, g):
        return (g * (ctx.alpha / ctx.n)).expand(ctx.shape), None


def transform_keypoints(kp, R, scale, shift):
    return _TransformFn.apply(kp, R, scale, shift)


def mean_scale(d, alpha):
    return _MeanScaleFn.apply(d, float(alpha))


class ChamferLoss_Brute(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.dimension = 3

    def forward(self, pc_src_input, pc_dst_input, sigma_src=None, sigma_dst=None):
        """pc_src (B,3,M), pc_dst (B,3,N), sigma (B,M)/(B,N) -> (loss, chamfer_pure, chamfer_weighted);
        without sigmas: un-reduced (B,M) tensors (losses.py:68-78)."""
        if sigma_src is None or sigma_dst is None:
            forward_loss = _PairMinFn.apply(pc_src_input, pc_dst_input)
            backward_loss = _PairMinFn.apply(pc_dst_input, pc_src_input)
            chamfer_pure = forward_loss + backward_loss
            return forward_loss + backward_loss, chamfer_pure, chamfer_pure
        return _ChamferProbFn.apply(pc_src_input, pc_dst_input, sigma_src, sigma_dst)


class SingleSideChamferLoss_Brute(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.dimension = 3

    def forward(self, pc_src_input, pc_dst_input):
        """(B,3,M), (B,3,N) -> (B,M) min distances (losses.py:125-143)."""
        return _PairMinFn.apply(pc_src_input, pc_dst_input)


class _PointOnSurfaceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoint, pc, sn):
        kp = keypoint.contiguous(); pc = pc.contiguous(); sn = sn.contiguous()
        B, _, M = kp.shape
        loss, arg = point_on_surface_fwd(kp, pc, sn)
        ctx.save_for_backward(kp, pc, sn, arg)
        return loss.view(B, M, 1, 1)                            # the reference returns the (B,M,1,1) matmul result

    @staticmethod
    def backward(ctx, g):
        kp, pc, sn, arg = ctx.saved_tensors
        return point_on_surface_bwd(kp, pc, sn, arg, g), None, None


class PointOnSurfaceLoss(nn.Module):
    """models/losses.py:146-183 ('point_to_plane'): squared cosine between the surface normal of the nearest cloud point
    and the direction from that point to the keypoint; gradient w.r.t. the keypoint only."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt

    def forward(self, keypoint, pc, sn):
        return _PointOnSurfaceFn.apply(keypoint, pc.detach(), sn.detach())


class KeypointOnPCLoss(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.single_side_chamfer = SingleSideChamferLoss_Brute(opt)
        self.keypoint_on_surface = PointOnSurfaceLoss(opt)

    def forward(self, keypoint, pc, sn=None):
        if sn is None:
            return self.single_side_chamfer(keypoint, pc)
        return self.keypoint_on_surface(keypoint, pc, sn)


class _DescTripletFn(torch.autograd.Function):
    """loss (B,M), active (B) of DescPairScanLoss; backward through the two descriptor-space nearest neighbours."""

    @staticmethod
    def forward(ctx, anc, pos, neg, sigmas, gamma, sigma_max):
        lib = _lib.load()
        a = anc.contiguous(); p_ = pos.contiguous(); n_ = neg.contiguous(); sg = sigmas.contiguous().float()
        B, C, M = a.shape
        dev = a.device
        dpos = torch.empty((B, M), dtype=torch.float32, device=dev); dneg = torch.empty_like(dpos)
        ipos = torch.empty((B, M), dtype=torch.int32, device=dev); ineg = torch.empty_like(ipos)
        _lib.check(lib.usip_desc_pairmin_f32(_p(a), _p(p_), _p(dpos), _p(ipos), B, C, M, p_.shape[2], _stream()), "usip_desc_pairmin_f32")
        _lib.check(lib.usip_desc_pairmin_f32(_p(a), _p(n_), _p(dneg), _p(ineg), B, C, M, n_.shape[2], _stream()), "usip_desc_pairmin_f32")
        loss = torch.empty_like(dpos); active = torch.empty((B,), dtype=torch.float32, device=dev)
        _lib.check(lib.usip_desc_triplet(_p(dpos), _p(dneg), _p(sg), float(gamma), float(sigma_max), _p(loss), _p(active),
                                         B, M, _stream()), "usip_desc_triplet")
        ctx.save_for_backward(a, p_, n_, sg, dpos, ipos, dneg, ineg)
        ctx.gamma, ctx.sigma_max = float(gamma), float(sigma_max)
        ctx.mark_non_differentiable(active)
        return loss, active

    @staticmethod
    def backward(ctx, g_loss, g_active):
        a, p_, n_, sg, dpos, ipos, dneg, ineg = ctx.saved_tensors
        B, C, M = a.shape
        g_a = torch.zeros_like(a); g_p = torch.zeros_like(p_); g_n = torch.zeros_like(n_)
        _lib.check(_lib.load().usip_desc_triplet_bwd(_p(a), _p(p_), _p(n_), _p(dpos), _p(ipos), _p(dneg), _p(ineg), _p(sg),
                                                     ctx.gamma, ctx.sigma_max, _p(g_loss.contiguous().float()), _p(g_a), _p(g_p),
                                                     _p(g_n), B, C, M, p_.shape[2], n_.shape[2], _stream()),
                   "usip_desc_triplet_bwd")
        return g_a, g_p, g_n, None, None, None


class DescPairScanLoss(nn.Module):
    """Triplet loss over scan pairs (models/losses.py:190-237): for every anchor keypoint the closest descriptor in
    the positive and in the negative scan (two fused C-dimensional pairwise-min kernels instead of two (B,C,M,M)
    difference tensors), sigma-derived (detached) weights; backward through the matched pairs (SURVEY 8 f-1)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt

    def forward(self, anc_descriptors, pos_descriptors, neg_descriptors, anc_sigmas):
        return _DescTripletFn.apply(anc_descriptors, pos_descriptors, neg_descriptors, anc_sigmas.detach(),
                                    self.opt.triple_loss_gamma, self.opt.sigma_max)


class _DescCGFFn(torch.autograd.Function):
    """loss (B,M), active (B) of DescCGFLoss (usip_desc_cgf_f32); backward (usip_desc_cgf_bwd) to both descriptor sets
    through the three selected pairs of every anchor."""

    @staticmethod
    def forward(ctx, module, anc_kp, anc_desc, pos_kp, pos_desc, sigmas, u_near, u_out, u_sel, radius, gamma, sigma_max):
        a, p_ = anc_desc.contiguous(), pos_desc.contiguous()
        sg = sigmas.contiguous()
        from usip_b200 import engine
        with engine._Prof("desc_cgf"):
            loss, active, saved = ops.desc_cgf(anc_kp.contiguous(), pos_kp.contiguous(), a, p_, sg, (u_near, u_out, u_sel),
                                               radius, gamma, sigma_max)
        ctx.save_for_backward(a, p_, sg, *saved)
        ctx.sigma_max = float(sigma_max)
        module.last_picks = saved[0]
        ctx.mark_non_differentiable(active)
        return loss, active

    @staticmethod
    def backward(ctx, g_loss, g_active):
        a, p_, sg, sel, aux, cloud = ctx.saved_tensors
        from usip_b200 import engine
        with engine._Prof("desc_cgf_bwd"):
            g_a, g_p = ops.desc_cgf_bwd(a, p_, sg, (sel, aux, cloud), g_loss, ctx.sigma_max)
        return None, None, g_a, None, g_p, None, None, None, None, None, None, None


class DescCGFLoss(nn.Module):
    """CGF triplet loss of the indoor descriptor (models/losses.py:240-369).  For every anchor keypoint (already mapped into
    the positive frame): a random positive keypoint within CGF_radius, the closest one beyond it and a random one beyond
    it; the negative is one of the latter two by a coin flip.  Loss (B,M) weighted by the anchor sigmas and rescaled by
    the share of anchors that have a positive; active (B).  One kernel scans the (B,M,M) keypoint pairs without storing
    them and computes only the three selected descriptor distances per anchor; the backward goes through those pairs.

    The three random tensors are the reference's own torch.rand calls, same shapes, order and device (`draws`): with the
    same CUDA seed the same GPU draws the same numbers.  `last_picks` holds the (B,M,4) int32 picks of the last call:
    near, far, out and flags (bit 0: the anchor has a positive, bit 1: the negative is `far`)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.last_picks = None

    def draws(self, B, M, device):
        """losses.py:279, 293, 298: u_near (B,M,M), u_out (B,M,M), u_sel (B,M), uniform in [0, 1)."""
        u_near = torch.rand((B, M, M), dtype=torch.float32, device=device, requires_grad=False)
        u_out = torch.rand((B, M, M), dtype=torch.float32, device=device, requires_grad=False)
        u_sel = torch.rand((B, M), dtype=torch.float32, device=device, requires_grad=False)
        return u_near, u_out, u_sel

    def forward(self, anc_keypoints, anc_descriptors, pos_keypoints, pos_descriptors, anc_sigmas, anc_pc=None, pos_pc=None):
        """anc_keypoints (B,3,M) in the positive frame, anc_descriptors (B,C,M), pos_keypoints (B,3,M), pos_descriptors
        (B,C,M), anc_sigmas (B,M) -> (loss (B,M), active_percentage (B)).  anc_pc / pos_pc are accepted and unused, as in
        the reference."""
        B, _, M = anc_keypoints.shape
        if not anc_descriptors.is_cuda:
            raise NotImplementedError("the DescCGFLoss training step runs on CUDA tensors only; there is no CPU path")
        u_near, u_out, u_sel = self.draws(B, M, anc_keypoints.device)
        return _DescCGFFn.apply(self, anc_keypoints.detach(), anc_descriptors, pos_keypoints.detach(), pos_descriptors,
                                anc_sigmas.detach().float(), u_near, u_out, u_sel, float(self.opt.CGF_radius),
                                float(self.opt.triple_loss_gamma), float(self.opt.sigma_max))
