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


class _FusedNet(nn.Module):
    """Base of the networks below.  Their forward and backward are the fused plans of usip_b200/engine.py, run through
    one whole-network autograd node (_NetFn).  Each network states its plans, `_forward_plan(x, sn, points, epoch) ->
    (outputs, saved plan)` and `_backward_plan(saved plan, *output gradients) -> parameter gradients`, and `_NON_DIFF`,
    the indices of the outputs that carry no gradient.

    It also keeps the packed tensor-core weight cache (engine._tc_workspace) honest across the writes that do not bump
    the parameters' autograd version -- load_state_dict and mode switches re-pack; `invalidate_packed_weights()` is the
    explicit hook for in-place `.data` edits (EMA, clipping, legacy loaders)."""
    _NON_DIFF = ()

    def _install_weight_hooks(self):
        self.register_load_state_dict_post_hook(lambda module, incompatible: engine.invalidate_packed_weights(module))

    def invalidate_packed_weights(self):
        engine.invalidate_packed_weights(self)

    def train(self, mode=True):
        if mode != self.training:
            engine.invalidate_packed_weights(self)
        return super().train(mode)

    def _check_input(self, x):
        if not x.is_cuda:
            raise RuntimeError("usip_b200 runs on CUDA tensors only (no CPU fallback)")

    def _run(self, x, sn, points, epoch):
        """The forward plan's outputs.  The plan keeps its activations for a backward (`_keep`) only when autograd
        will ask for parameter gradients."""
        params = tuple(self.parameters())
        self._keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        self._check_input(x)
        with torch.cuda.device(x.device):
            return _NetFn.apply(self, x, sn, points, epoch, *params)


class _NetFn(torch.autograd.Function):
    """Whole-network autograd node: forward = net._forward_plan, backward = net._backward_plan.
    Inputs carry no gradient (x, sn, nodes / keypoints are detached data in the reference, networks.py:96-107, 345);
    gradients flow to the parameters."""

    @staticmethod
    def forward(ctx, net, x, sn, points, epoch, *params):
        # autograd.Function.forward runs under no_grad; whether to keep activations was decided by the caller (net._keep)
        outs, saved = net._forward_plan(x, sn, points, epoch)
        ctx.net = net
        ctx.saved_plan = saved
        ctx.mark_non_differentiable(*(outs[i] for i in net._NON_DIFF))
        return outs

    @staticmethod
    def backward(ctx, *grads):
        if ctx.saved_plan is None:
            raise RuntimeError("%s forward ran without saving activations (no_grad / frozen)" % type(ctx.net).__name__)
        param_grads = ctx.net._backward_plan(ctx.saved_plan, *grads)
        ctx.saved_plan = None
        return (None, None, None, None, None) + tuple(param_grads)


def _bn_kwargs(opt):
    return dict(momentum=opt.bn_momentum, bn_momentum_decay_step=opt.bn_momentum_decay_step,
                bn_momentum_decay=opt.bn_momentum_decay)


class _DetectorBase(_FusedNet):
    C1 = 128
    C2 = 512

    def _build_head(self, opt):
        """The node kNN fusion module and the head of every detector (networks.py:43-72, and the same lines of the other
        three); built after the point stage, so that each layer draws the same initial weights as the reference's."""
        C1, C2, bn = self.C1, self.C2, _bn_kwargs(opt)
        assert opt.node_knn_k_1 >= 2
        _check_group(opt.node_knn_k_1, "node_knn_k_1")
        self.knnlayer_1 = GeneralKNNFusionModule(3 + C1, (C2 // 2, C2 // 2, C2 // 2), (C2, C2),
                                                 activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp1 = EquivariantLayer(C1 + C2, 512, activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp2 = EquivariantLayer(512, 256, activation=opt.activation, normalization=opt.normalization, **bn)
        self.mlp3 = EquivariantLayer(256, 4, activation=None, normalization=None)
        self.mlp3.conv.weight.data.normal_(0, 1e-4)          # networks.py:70-71
        self.mlp3.conv.bias.data.zero_()
        self.softplus = torch.nn.Softplus()                  # kept for attribute parity; evaluated in-kernel
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False
        self._install_weight_hooks()
        if opt.activation != "relu" or opt.normalization != "batch":
            raise NotImplementedError("the H100 plan implements activation='relu', normalization='batch'")


class _RPNBase(_DetectorBase):
    _NON_DIFF = (0,)                                         # the cluster means

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        C1, bn = self.C1, _bn_kwargs(opt)
        self.first_pointnet = PointNet(3 + opt.surface_normal_len, [C1 // 2, C1 // 2, C1 // 2],
                                       activation=opt.activation, normalization=opt.normalization, **bn)
        self.second_pointnet = PointNet(C1, [C1, C1], activation=opt.activation, normalization=opt.normalization, **bn)
        self._build_head(opt)
        self._last_aux = None

    def forward(self, x, sn, node, is_train=False, epoch=None):
        """-> (som_node_cluster_mean (B,3,M), keypoints (B,3,M), sigmas (B,M), None)   networks.py:156-162"""
        cmean, kp, sig = self._run(x, sn, node, epoch)
        return cmean, kp, sig, None

    def _forward_plan(self, x, sn, node, epoch):
        cmean, kp, sig, saved, self._last_aux = engine.detector_forward(self, x, sn, node, epoch, use_tc=self.use_tc,
                                                                         keep=self._keep)
        return (cmean, kp, sig), saved

    def _backward_plan(self, saved, g_cmean, g_kp, g_sig):
        return engine.detector_backward(self, saved, g_kp, g_sig)


class RPN_Detector(_RPNBase):
    C1 = 128
    C2 = 512


class RPN_DetectorLite(_RPNBase):
    C1 = 64
    C2 = 256


class _RPNAblationBase(_DetectorBase):
    """Shared body of the two ablation detectors (identical constructors in the reference, networks.py:483-543, 612-669):
    conv1..conv5 grouped PointNet, the node kNN fusion module, the head.  The nodes are used as given -- no SOM
    re-assignment, no recomputed cluster means -- and are returned as the first output (networks.py:608, 738)."""
    GROUPING = None

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        C1 = self.C1
        kw = dict(kernel_size=(1, 1), stride=1, padding=0, bias=True, activation=opt.activation,
                  normalization=opt.normalization, **_bn_kwargs(opt))
        self.conv1 = MyConv2d(3 + opt.surface_normal_len, C1 // 2, **kw)
        self.conv2 = MyConv2d(C1 // 2, C1 // 2, **kw)
        self.conv3 = MyConv2d(C1 // 2, C1 // 2, **kw)
        self.conv4 = MyConv2d(C1, C1, **kw)
        self.conv5 = MyConv2d(C1, C1, **kw)
        self._build_head(opt)

    def forward(self, x, sn, node, is_train=False, epoch=None):
        """-> (node (B,3,M), keypoints (B,3,M), sigmas (B,M), None)"""
        kp, sig = self._run(x, sn, node, epoch)
        return node, kp, sig, None

    def _forward_plan(self, x, sn, node, epoch):
        _, kp, sig, saved = engine.ablation_forward(self, x, sn, node, epoch, use_tc=self.use_tc, keep=self._keep,
                                                    mode=self.GROUPING)
        return (kp, sig), saved

    def _backward_plan(self, saved, g_kp, g_sig):
        return engine.ablation_backward(self, saved, g_kp, g_sig)


class RPN_Detector_KNN(_RPNAblationBase):
    GROUPING = "knn"


class RPN_Detector_Ball(_RPNAblationBase):
    GROUPING = "ball"


class _DescriptorBase(_FusedNet):
    """The grouped PointNet both descriptors start with (conv1..conv5, networks.py:315-331 and 393-410) and their
    forward: forward(x, sn, keypoints, is_train, epoch) -> (descriptor (B,D,M), x_features (B,3+S,M,K))."""
    _NON_DIFF = (1,)                                         # the ball features

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        D = int(opt.descriptor_len)                          # the indoor options declare descriptor_len as a float
        kw = dict(kernel_size=(1, 1), stride=1, padding=0, bias=True)
        act = dict(activation=opt.activation, normalization=opt.normalization, **_bn_kwargs(opt))
        self.conv1 = MyConv2d(3 + opt.surface_normal_len, D // 4, **kw, **act)
        self.conv2 = MyConv2d(D // 4, D // 2, **kw, **act)
        self.conv3 = MyConv2d(D // 2, D, **kw, **act)
        self.conv4 = MyConv2d(D * 2, D, **kw, **act)
        self.conv5 = MyConv2d(D, D, **kw, activation=None, normalization=None)
        self.use_tc = bool(getattr(opt, "use_tensor_cores", True))
        self._keep = False

    def forward(self, x, sn, keypoints, is_train=False, epoch=None):
        return self._run(x, sn, keypoints, epoch)

    def _forward_plan(self, x, sn, keypoints, epoch):
        # host-side permutation, same RNG stream as the reference (networks.py:345, 443)
        permute_idx = torch.from_numpy(np.random.permutation(x.size()[2]).astype(np.int64)).to(x.device)
        desc, feats, saved = self._plan_forward(self, x, sn, keypoints, epoch, permute_idx, use_tc=self.use_tc,
                                                keep=self._keep)
        return (desc, feats), saved

    def _backward_plan(self, saved, g_desc, g_feats):
        return self._plan_backward(self, saved, g_desc)


class DescriptorLiteOld(_DescriptorBase):
    """models/networks.py:310-385."""
    _plan_forward = staticmethod(engine.descriptor_forward)
    _plan_backward = staticmethod(engine.descriptor_backward)

    def __init__(self, opt):
        super().__init__(opt)
        _check_group(opt.ball_nsamples, "ball_nsamples")
        self._install_weight_hooks()


class DescriptorLiteOldGlobal(_DescriptorBase):
    """models/networks.py:388-479, the indoor descriptor: DescriptorLiteOld's grouped PointNet, then PPFNet's global
    context -- the max of the descriptors over the M keypoints of each cloud, concatenated to every keypoint's descriptor,
    fc1 (2D->2D), fc2 (2D->D), fc3 (D->D, linear) -- and L2 normalisation.  The global context is taken over the keypoints
    the forward is given.  With gradients enabled and trainable parameters the forward keeps its activations and pool
    args, and autograd runs engine.descriptor_global_backward."""
    _plan_forward = staticmethod(engine.descriptor_global_forward)
    _plan_backward = staticmethod(engine.descriptor_global_backward)

    def __init__(self, opt):
        super().__init__(opt)
        D, bn = int(opt.descriptor_len), _bn_kwargs(opt)
        self.fc1 = EquivariantLayer(D * 2, D * 2, activation=opt.activation, normalization=opt.normalization, **bn)
        self.fc2 = EquivariantLayer(D * 2, D, activation=opt.activation, normalization=opt.normalization, **bn)
        self.fc3 = EquivariantLayer(D, D, activation=None, normalization=None)
        _check_ball(opt.ball_nsamples, "ball_nsamples")
        if opt.activation != "relu" or opt.normalization != "batch":
            raise NotImplementedError("the H100 plan implements activation='relu', normalization='batch'")
        self._install_weight_hooks()

    def _check_input(self, x):
        if not x.is_cuda and self._keep:
            raise NotImplementedError("DescriptorLiteOldGlobal with gradients: the DescCGFLoss training step runs on "
                                      "CUDA tensors only; there is no CPU path")
        super()._check_input(x)
        if self._keep and self.conv1.conv.weight.shape[0] < 32:
            raise NotImplementedError("DescriptorLiteOldGlobal with gradients needs descriptor_len >= 128: the BatchNorm "
                                      "backward kernels take layers of at least 32 channels (conv1 has descriptor_len/4)")
