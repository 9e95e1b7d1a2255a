"""Host-side mirror of the hot-path networks of models/networks.py: same class names, constructor
(`opt`), forward signatures, return conventions and state_dict keys; the arithmetic is the fused H100 plan
in usip_b200/engine.py.

  RPN_Detector      models/networks.py:20-162   (C1=128, C2=512)
  RPN_DetectorLite  models/networks.py:165-307  (C1=64,  C2=256; same graph)
  DescriptorLiteOld models/networks.py:310-385
  DescriptorLiteOldGlobal models/networks.py:388-479  (indoor: PPFNet global context)
  RPN_Detector_KNN  models/networks.py:482-608  (ablation: 64 nearest points per node instead of the SOM assignment)
  RPN_Detector_Ball models/networks.py:611-738  (ablation: first 64 points within radius 2 of each node)
"""
import numpy as np
import torch
import torch.nn as nn

from .layers import EquivariantLayer, GeneralKNNFusionModule, MyConv2d, PointNet
from usip_b200 import engine


def _check_group(k, name):
    """The fused group-max epilogues (usip_layer_fwd) take groups that are a multiple of 4 and divide 128."""
    if k % 4 != 0 or 128 % k != 0:
        raise NotImplementedError("%s=%d: the H100 plan supports group sizes 4, 8, 16, 32, 64, 128 "
                                  "(every shipped configuration uses 16, 32 or 64)" % (name, k))


def _check_ball(k, name):
    """Balls of at most 128 rows go through the layer epilogue's group max directly; larger ones as 64-row sub-groups that
    usip_group_max_combine reduces (engine._group_net_forward)."""
    if k > 128 and k % 64 == 0:
        return
    if k % 4 != 0 or 128 % k != 0:
        raise NotImplementedError("%s=%d: the H100 plan supports balls of 4, 8, 16, 32, 64 or 128 samples, or a multiple "
                                  "of 64 above 128 (the indoor options use 448)" % (name, k))


class _PackedWeightHooks:
    """Mixin: keeps the packed tensor-core weight cache (engine._tc_workspace) honest across the writes that do not bump
    the parameters' autograd version -- load_state_dict and mode switches re-pack; `invalidate_packed_weights()` is the
    explicit hook for in-place `.data` edits (EMA, clipping, legacy loaders)."""

    def _install_weight_hooks(self):
        self.register_load_state_dict_post_hook(lambda module, incompatible: engine.invalidate_packed_weights(module))

    def invalidate_packed_weights(self):
        engine.invalidate_packed_weights(self)

    def train(self, mode=True):
        if mode != self.training:
            engine.invalidate_packed_weights(self)
        return super().train(mode)


class _DetectorFn(torch.autograd.Function):
    """Whole-network autograd node: forward = engine.detector_forward, backward = engine.detector_backward.
    Inputs carry no gradient (x, sn, node are detached data in the reference, networks.py:96-107);
    gradients flow to the parameters."""

    @staticmethod
    def forward(ctx, net, x, sn, node, epoch, *params):
        keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        # autograd.Function.forward runs under no_grad; `keep` was decided by the caller
        cmean, kp, sig, saved, aux = engine.detector_forward(net, x, sn, node, epoch, use_tc=net.use_tc, keep=net._keep)
        ctx.net = net
        ctx.saved_plan = saved
        ctx.mark_non_differentiable(cmean)
        net._last_aux = aux
        return cmean, kp, sig

    @staticmethod
    def backward(ctx, g_cmean, g_kp, g_sig):
        if ctx.saved_plan is None:
            raise RuntimeError("detector forward ran without saving activations (no_grad / frozen)")
        grads = engine.detector_backward(ctx.net, ctx.saved_plan, g_kp, g_sig)
        ctx.saved_plan = None
        return (None, None, None, None, None) + tuple(grads)


class _RPNBase(_PackedWeightHooks, nn.Module):
    C1 = 128
    C2 = 512

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        C1, C2 = self.C1, self.C2
        kw = dict(momentum=opt.bn_momentum, bn_momentum_decay_step=opt.bn_momentum_decay_step,
                  bn_momentum_decay=opt.bn_momentum_decay)
        self.first_pointnet = PointNet(3 + self.opt.surface_normal_len, [C1 // 2, C1 // 2, C1 // 2],
                                       activation=opt.activation, normalization=opt.normalization, **kw)
        self.second_pointnet = PointNet(C1, [C1, C1], activation=opt.activation, normalization=opt.normalization, **kw)
        assert self.opt.node_knn_k_1 >= 2
        _check_group(self.opt.node_knn_k_1, "node_knn_k_1")
        self.knnlayer_1 = GeneralKNNFusionModule(3 + C1, (C2 // 2, C2 // 2, C2 // 2), (C2, C2),
                                                 activation=opt.activation, normalization=opt.normalization, **kw)
        self.mlp1 = EquivariantLayer(C1 + C2, 512, activation=opt.activation, normalization=opt.normalization, **kw)
        self.mlp2 = EquivariantLayer(512, 256, activation=opt.activation, normalization=opt.normalization, **kw)
        self.mlp3 = EquivariantLayer(256, 4, activation=None, normalization=None)
        self.mlp3.conv.weight.data.normal_(0, 1e-4)          # networks.py:70-71
        self.mlp3.conv.bias.data.zero_()
        self.softplus = torch.nn.Softplus()                  # kept for attribute parity; evaluated in-kernel
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False
        self._last_aux = None
        self._install_weight_hooks()
        if opt.activation != "relu" or opt.normalization != "batch":
            raise NotImplementedError("the H100 plan implements activation='relu', normalization='batch'")

    def forward(self, x, sn, node, is_train=False, epoch=None):
        """-> (som_node_cluster_mean (B,3,M), keypoints (B,3,M), sigmas (B,M), None)   networks.py:156-162"""
        if not x.is_cuda:
            raise RuntimeError("usip_b200 runs on CUDA tensors only (no CPU fallback)")
        params = tuple(self.parameters())
        self._keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        with torch.cuda.device(x.device):
            cmean, kp, sig = _DetectorFn.apply(self, x, sn, node, epoch, *params)
        return cmean, kp, sig, None


class RPN_Detector(_RPNBase):
    C1 = 128
    C2 = 512


class RPN_DetectorLite(_RPNBase):
    C1 = 64
    C2 = 256


class _AblationFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, x, sn, node, epoch, *params):
        node_out, kp, sig, saved = engine.ablation_forward(net, x, sn, node, epoch, use_tc=net.use_tc, keep=net._keep,
                                                           mode=net.GROUPING)
        ctx.net = net
        ctx.saved_plan = saved
        return kp, sig

    @staticmethod
    def backward(ctx, g_kp, g_sig):
        if ctx.saved_plan is None:
            raise RuntimeError("detector forward ran without saving activations (no_grad / frozen)")
        grads = engine.ablation_backward(ctx.net, ctx.saved_plan, g_kp, g_sig)
        ctx.saved_plan = None
        return (None, None, None, None, None) + tuple(grads)


class _RPNAblationBase(_PackedWeightHooks, nn.Module):
    """Shared body of the two ablation detectors (identical constructors in the reference, networks.py:483-543, 612-669):
    conv1..conv5 grouped PointNet, the node kNN fusion module, the head.  The nodes are used as given -- no SOM
    re-assignment, no recomputed cluster means -- and are returned as the first output (networks.py:608, 738)."""
    GROUPING = None

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.C1, self.C2 = 128, 512
        C1, C2 = self.C1, self.C2
        bn = dict(momentum=opt.bn_momentum, bn_momentum_decay_step=opt.bn_momentum_decay_step,
                  bn_momentum_decay=opt.bn_momentum_decay)
        kw = dict(kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=opt.activation,
                  normalization=opt.normalization, **bn)
        self.conv1 = MyConv2d(3 + opt.surface_normal_len, C1 // 2, **kw)
        self.conv2 = MyConv2d(C1 // 2, C1 // 2, **kw)
        self.conv3 = MyConv2d(C1 // 2, C1 // 2, **kw)
        self.conv4 = MyConv2d(C1, C1, **kw)
        self.conv5 = MyConv2d(C1, C1, **kw)
        assert opt.node_knn_k_1 >= 2
        _check_group(opt.node_knn_k_1, "node_knn_k_1")
        self.knnlayer_1 = GeneralKNNFusionModule(3 + C1, (C2 // 2, C2 // 2, C2 // 2), (C2, C2),
                                                 activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp1 = EquivariantLayer(C1 + C2, 512, activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp2 = EquivariantLayer(512, 256, activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp3 = EquivariantLayer(256, 4, activation=None, normalization=None)
        self.mlp3.conv.weight.data.normal_(0, 1e-4)
        self.mlp3.conv.bias.data.zero_()
        self.softplus = torch.nn.Softplus()
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False
        self._install_weight_hooks()
        if opt.activation != "relu" or opt.normalization != "batch":
            raise NotImplementedError("the H100 plan implements activation='relu', normalization='batch'")

    def forward(self, x, sn, node, is_train=False, epoch=None):
        """-> (node (B,3,M), keypoints (B,3,M), sigmas (B,M), None)"""
        if not x.is_cuda:
            raise RuntimeError("usip_b200 runs on CUDA tensors only (no CPU fallback)")
        params = tuple(self.parameters())
        self._keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        with torch.cuda.device(x.device):
            kp, sig = _AblationFn.apply(self, x, sn, node, epoch, *params)
        return node, kp, sig, None


class RPN_Detector_KNN(_RPNAblationBase):
    GROUPING = "knn"


class RPN_Detector_Ball(_RPNAblationBase):
    GROUPING = "ball"


class _DescriptorFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, x, sn, keypoints, epoch, permute_idx, *params):
        desc, feats, saved = engine.descriptor_forward(net, x, sn, keypoints, epoch, permute_idx,
                                                       use_tc=net.use_tc, keep=net._keep)
        ctx.net = net
        ctx.saved_plan = saved
        ctx.mark_non_differentiable(feats)
        return desc, feats

    @staticmethod
    def backward(ctx, g_desc, g_feats):
        if ctx.saved_plan is None:
            raise RuntimeError("descriptor forward ran without saving activations")
        grads = engine.descriptor_backward(ctx.net, ctx.saved_plan, g_desc)
        ctx.saved_plan = None
        return (None, None, None, None, None, None) + tuple(grads)


class DescriptorLiteOld(_PackedWeightHooks, nn.Module):
    """models/networks.py:310-385.  forward(x, sn, keypoints, is_train, epoch) -> (descriptor (B,C,M),
    x_features (B,3+S,M,K))."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        cin = 3 + opt.surface_normal_len
        D = opt.descriptor_len
        kw = dict(kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=opt.activation,
                  normalization=opt.normalization, momentum=opt.bn_momentum,
                  bn_momentum_decay_step=opt.bn_momentum_decay_step, bn_momentum_decay=opt.bn_momentum_decay)
        self.conv1 = MyConv2d(cin, D // 4, **kw)
        self.conv2 = MyConv2d(D // 4, D // 2, **kw)
        self.conv3 = MyConv2d(D // 2, D, **kw)
        self.conv4 = MyConv2d(D * 2, D, **kw)
        self.conv5 = MyConv2d(D, D, kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=None, normalization=None)
        _check_group(opt.ball_nsamples, "ball_nsamples")
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False
        self._install_weight_hooks()

    def forward(self, x, sn, keypoints, is_train=False, epoch=None):
        if not x.is_cuda:
            raise RuntimeError("usip_b200 runs on CUDA tensors only (no CPU fallback)")
        N = x.size()[2]
        # host-side permutation, same RNG stream as the reference (networks.py:345)
        permute_idx = torch.from_numpy(np.random.permutation(N).astype(np.int64)).to(x.device)
        params = tuple(self.parameters())
        self._keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        with torch.cuda.device(x.device):
            desc, feats = _DescriptorFn.apply(self, x, sn, keypoints, epoch, permute_idx, *params)
        return desc, feats


class _DescriptorGlobalFn(torch.autograd.Function):
    """Whole-network autograd node of DescriptorLiteOldGlobal: forward = engine.descriptor_global_forward(keep=True),
    backward = engine.descriptor_global_backward; gradients flow to the parameters only."""

    @staticmethod
    def forward(ctx, net, x, sn, keypoints, epoch, permute_idx, *params):
        desc, feats, saved = engine.descriptor_global_forward(net, x, sn, keypoints, epoch, permute_idx,
                                                              use_tc=net.use_tc, keep=True)
        ctx.net = net
        ctx.saved_plan = saved
        ctx.mark_non_differentiable(feats)
        return desc, feats

    @staticmethod
    def backward(ctx, g_desc, g_feats):
        if ctx.saved_plan is None:
            raise RuntimeError("descriptor forward ran without saving activations")
        grads = engine.descriptor_global_backward(ctx.net, ctx.saved_plan, g_desc)
        ctx.saved_plan = None
        return (None, None, None, None, None, None) + tuple(grads)


class DescriptorLiteOldGlobal(_PackedWeightHooks, nn.Module):
    """models/networks.py:388-479, the indoor descriptor: DescriptorLiteOld's grouped PointNet, then PPFNet's global
    context -- the max of the descriptors over the M keypoints of each cloud, concatenated to every keypoint's descriptor,
    fc1 (2D->2D), fc2 (2D->D), fc3 (D->D, linear) -- and L2 normalisation.  The global context is taken over the keypoints
    the forward is given.  forward(x, sn, keypoints, is_train, epoch) -> (descriptor (B,D,M), x_features (B,3+S,M,K)).
    With gradients enabled and trainable parameters the forward keeps its activations and pool args, and autograd runs
    engine.descriptor_global_backward (_DescriptorGlobalFn)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        cin = 3 + opt.surface_normal_len
        D = int(opt.descriptor_len)                           # the indoor options declare descriptor_len as a float
        bn = dict(momentum=opt.bn_momentum, bn_momentum_decay_step=opt.bn_momentum_decay_step,
                  bn_momentum_decay=opt.bn_momentum_decay)
        kw = dict(kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=opt.activation,
                  normalization=opt.normalization, **bn)
        self.conv1 = MyConv2d(cin, D // 4, **kw)
        self.conv2 = MyConv2d(D // 4, D // 2, **kw)
        self.conv3 = MyConv2d(D // 2, D, **kw)
        self.conv4 = MyConv2d(D * 2, D, **kw)
        self.conv5 = MyConv2d(D, D, kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=None, normalization=None)
        self.fc1 = EquivariantLayer(D * 2, D * 2, activation=opt.activation, normalization=opt.normalization, **bn)
        self.fc2 = EquivariantLayer(D * 2, D, activation=opt.activation, normalization=opt.normalization, **bn)
        self.fc3 = EquivariantLayer(D, D, activation=None, normalization=None)
        _check_ball(opt.ball_nsamples, "ball_nsamples")
        if opt.activation != "relu" or opt.normalization != "batch":
            raise NotImplementedError("the H100 plan implements activation='relu', normalization='batch'")
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False
        self._install_weight_hooks()

    def forward(self, x, sn, keypoints, is_train=False, epoch=None):
        params = tuple(self.parameters())
        self._keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        if not x.is_cuda:
            if self._keep:
                raise NotImplementedError("DescriptorLiteOldGlobal with gradients: the DescCGFLoss training step runs on "
                                          "CUDA tensors only; there is no CPU path")
            raise RuntimeError("usip_b200 runs on CUDA tensors only (no CPU fallback)")
        if self._keep and self.conv1.conv.weight.shape[0] < 32:
            raise NotImplementedError("DescriptorLiteOldGlobal with gradients needs descriptor_len >= 128: the BatchNorm "
                                      "backward kernels take layers of at least 32 channels (conv1 has descriptor_len/4)")
        N = x.size()[2]
        # host-side permutation, same RNG stream as the reference (networks.py:443)
        permute_idx = torch.from_numpy(np.random.permutation(N).astype(np.int64)).to(x.device)
        with torch.cuda.device(x.device):
            if self._keep:
                return _DescriptorGlobalFn.apply(self, x, sn, keypoints, epoch, permute_idx, *params)
            desc, feats, _ = engine.descriptor_global_forward(self, x, sn, keypoints, epoch, permute_idx, use_tc=self.use_tc)
            return desc, feats
