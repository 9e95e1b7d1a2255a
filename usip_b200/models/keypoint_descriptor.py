"""`ModelDescriptor` -- API surface of models/keypoint_descriptor.py:14-318 (outdoor descriptor: DescriptorLiteOld +
DescPairScanLoss) on the fused H100 plan: `forward`, `forward_siamese`, `run_model`, `test_model` and the train step
`optimize()` (backward plan in engine.descriptor_backward, loss backward in losses._DescTripletFn; SURVEY.md 8 f-1).

`ModelDescriptorIndoor` -- models/keypoint_descriptor.py:321-603 (indoor descriptor: DescriptorLiteOldGlobal, 448-sample
balls and a global context, DescCGFLoss): `set_input`, `forward`, `forward_siamese`, `run_model`, `freeze_model` and the
train step `optimize()` / `test_model()` (backward plan in engine.descriptor_global_backward, loss backward in
losses._DescCGFFn), on CUDA only.  The reference network calls operations.ball_query_wrapper, which the reference ships
commented out (operations.py:295-366); this plan follows that commented-out code, whose semantics are those of the
reference's ball_query extension."""
import os
from collections import OrderedDict

import torch

from usip_b200 import ops
from usip_b200.optim import FlatAdam

from . import losses, networks
from ._common import random_point_dropout


class ModelDescriptor():
    def __init__(self, opt):
        self.opt = opt
        if opt.gpu_ids[0] < 0:
            raise RuntimeError("usip_b200.ModelDescriptor needs a CUDA device: there is no CPU path")
        self.descriptor = networks.DescriptorLiteOld(opt).to(opt.device)
        self.triplet_criteria = losses.DescPairScanLoss(opt)
        self.old_lr_descriptor = self.opt.lr
        self.optimizer_descriptor = FlatAdam(self.descriptor.parameters(), lr=self.old_lr_descriptor,
                                             betas=(0.9, 0.999), weight_decay=0)        # keypoint_descriptor.py:32-35
        dev = opt.device
        B, N, M = opt.batch_size, opt.input_pc_num, opt.node_num
        self.anc_pc = torch.empty(B, 3, N, device=dev).uniform_(); self.anc_sn = torch.empty(B, 3, N, device=dev).uniform_()
        self.anc_keypoints = torch.empty(B, 3, M, device=dev); self.anc_sigmas = torch.empty(B, M, device=dev)
        self.pos_pc = torch.empty(B, 3, N, device=dev).uniform_(); self.pos_sn = torch.empty(B, 3, N, device=dev).uniform_()
        self.pos_keypoints = torch.empty(B, 3, M, device=dev); self.pos_sigmas = torch.empty(B, M, device=dev)
        self.neg_idx = torch.zeros(B, dtype=torch.long, device=dev)
        z = lambda: torch.tensor([0], dtype=torch.float32, requires_grad=False, device=dev)
        self.test_loss_average = z(); self.test_loss_triplet_average = z(); self.test_active_percentage_average = z()

    _INPUT_FIELDS = ("anc_pc", "anc_sn", "anc_keypoints", "anc_sigmas", "pos_pc", "pos_sn", "pos_keypoints",
                     "pos_sigmas", "neg_idx")

    def set_input(self, anc_pc, anc_sn, anc_keypoints, anc_sigmas, pos_pc, pos_sn, pos_keypoints, pos_sigmas, neg_idx):
        """keypoint_descriptor.py:77-107.  If the same tensors were staged by prefetch_input(), the staged device copies
        are adopted with a stream-side wait instead of nine copies and a host synchronisation."""
        args = (anc_pc, anc_sn, anc_keypoints, anc_sigmas, pos_pc, pos_sn, pos_keypoints, pos_sigmas, neg_idx)
        st = getattr(self, "_staged", None)
        if st is not None and len(st[0]) == len(args) and all(a is b for a, b in zip(st[0], args)):
            cur = torch.cuda.current_stream()
            cur.wait_event(st[2])
            for k, v in zip(self._INPUT_FIELDS, st[1]):
                v.record_stream(cur)                                  # allocated on another stream, consumed here
                setattr(self, k, v)
            self._staged = None
            return
        dev = self.opt.device
        self.anc_pc = anc_pc.float().to(dev); self.anc_sn = anc_sn.float().to(dev)
        self.anc_keypoints = anc_keypoints.float().to(dev); self.anc_sigmas = anc_sigmas.float().to(dev)
        self.pos_pc = pos_pc.float().to(dev); self.pos_sn = pos_sn.float().to(dev)
        self.pos_keypoints = pos_keypoints.float().to(dev); self.pos_sigmas = pos_sigmas.float().to(dev)
        self.neg_idx = neg_idx.long().to(dev)
        torch.cuda.synchronize()

    def prefetch_input(self, *args, after=None):
        """Not in the reference: stage the NEXT batch (the nine set_input tensors) with asynchronous host-to-device
        copies on a dedicated stream, so that the transfer overlaps the running step; the following set_input() with the
        same tensor objects adopts the staged copies.  `after`: a CUDA event the staging waits for (device tensors
        produced on another stream, e.g. by KittiDescriptorPairSource).  neg_idx stays int64."""
        if len(args) != len(self._INPUT_FIELDS):
            raise TypeError("prefetch_input takes the nine set_input tensors, got %d" % len(args))
        dev = self.opt.device
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        if after is not None:
            self._copy_stream.wait_event(after)
        with torch.cuda.stream(self._copy_stream):
            staged = [a.float().to(dev, non_blocking=True).detach() for a in args[:-1]]
            staged.append(args[-1].long().to(dev, non_blocking=True).detach())
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        self._staged = (tuple(args), staged, ev)

    def forward(self, pc, sn, keypoints, is_train=False, epoch=None):
        with torch.cuda.device(pc.get_device()):
            return self.descriptor(pc, sn, keypoints, is_train, epoch)

    def forward_siamese(self, pc_tuple, sn_tuple, keypoints_tuple, is_train=False, epoch=None):
        n = pc_tuple[0].size()[0]
        descriptors, x_aug_ball = self.descriptor(torch.cat(pc_tuple, dim=0), torch.cat(sn_tuple, dim=0),
                                                  torch.cat(keypoints_tuple, dim=0), is_train, epoch)
        return torch.split(descriptors, n, dim=0), torch.split(x_aug_ball, n, dim=0)

    def _loss(self):
        triplet_loss, active_percentage = self.triplet_criteria(self.anc_descriptors, self.pos_descriptors,
                                                                self.anc_descriptors[self.neg_idx, :, :], self.anc_sigmas)
        self.triplet_loss = torch.mean(triplet_loss)
        self.active_percentage = torch.mean(active_percentage)
        self.loss = self.triplet_loss

    def optimize(self, epoch=None):
        """keypoint_descriptor.py:126-157: optional random point dropout (same RNG streams), train-mode forward of the
        (anchor, positive) batch, triplet loss against the in-batch negatives, backward, Adam."""
        with torch.cuda.device(self.anc_pc.get_device()):
            self.anc_pc, self.anc_sn, self.pos_pc, self.pos_sn = random_point_dropout(
                self.opt, self.anc_pc, self.anc_sn, self.pos_pc, self.pos_sn)
            self.descriptor.train()
            (self.anc_descriptors, self.pos_descriptors), _ = self.forward_siamese(
                (self.anc_pc, self.pos_pc), (self.anc_sn, self.pos_sn), (self.anc_keypoints, self.pos_keypoints),
                is_train=True, epoch=epoch)
            self.optimizer_descriptor.zero_grad()
            self._loss()
            self.loss.backward()
            self.optimizer_descriptor.step()

    def test_model(self):
        self.descriptor.eval()
        with torch.cuda.device(self.anc_pc.device), torch.no_grad():
            (self.anc_descriptors, self.pos_descriptors), _ = self.forward_siamese(
                (self.anc_pc, self.pos_pc), (self.anc_sn, self.pos_sn), (self.anc_keypoints, self.pos_keypoints),
                is_train=False, epoch=None)
            self._loss()

    def freeze_model(self):
        for p in self.descriptor.parameters():
            p.requires_grad = False

    def run_model(self, pc, sn, keypoints):
        self.descriptor.eval()
        with torch.cuda.device(pc.device), torch.no_grad():
            descriptors, _ = self.descriptor(pc, sn, keypoints, False, None)
        return descriptors

    def get_negative_samples(self):
        return (self.anc_pc[self.neg_idx, :, :], self.anc_sn[self.neg_idx, :, :],
                self.anc_keypoints[self.neg_idx, :, :], self.anc_sigmas[self.neg_idx, :])

    def get_current_visuals(self):
        raise NotImplementedError("visdom payloads (keypoint_descriptor.py:241-289) are outside the hot path")

    def get_current_errors(self):
        return OrderedDict([('O_loss', self.loss.item()), ('O_triplet', self.triplet_loss.item()),
                            ('O_active_perc', self.active_percentage.item()), ('E_loss', self.test_loss_average.item()),
                            ('E_triplet', self.test_loss_triplet_average.item()),
                            ('E_active_perc', self.test_active_percentage_average.item())])

    def save_network(self, network, network_label, epoch_label, gpu_id):
        torch.save(network.state_dict(), os.path.join(self.opt.checkpoints_dir, '%s_net_%s.pth' % (epoch_label, network_label)))

    def update_learning_rate(self, ratio):
        lr = max(self.old_lr_descriptor * ratio, 0.00001)
        for g in self.optimizer_descriptor.param_groups:
            g['lr'] = lr
        print('update descriptor learning rate: %f -> %f' % (self.old_lr_descriptor, lr))
        self.old_lr_descriptor = lr


class ModelDescriptorIndoor():
    """models/keypoint_descriptor.py:321-603: DescriptorLiteOldGlobal and DescCGFLoss on the fused plan.  A module built on
    a CPU device constructs (for state_dict work) but has no optimizer and does not train."""

    _NO_CPU = "the DescCGFLoss training step runs on CUDA tensors only; there is no CPU path"

    def __init__(self, opt):
        self.opt = opt
        if opt.gpu_ids[0] < 0:
            raise RuntimeError("usip_b200.ModelDescriptorIndoor needs a CUDA device: there is no CPU path")
        self.descriptor = networks.DescriptorLiteOldGlobal(opt).to(opt.device)
        self.triplet_criteria = losses.DescCGFLoss(opt)
        self.old_lr_descriptor = self.opt.lr
        dev = opt.device
        self.optimizer_descriptor = None
        if torch.device(dev).type == "cuda":                  # FlatAdam re-points CUDA parameters only
            self.optimizer_descriptor = FlatAdam(self.descriptor.parameters(), lr=self.old_lr_descriptor,
                                                 betas=(0.9, 0.999), weight_decay=0)    # keypoint_descriptor.py:340-343
        B, N, M = opt.batch_size, opt.input_pc_num, opt.node_num
        self.anc_pc = torch.empty(B, 3, N, device=dev).uniform_(); self.anc_sn = torch.empty(B, 3, N, device=dev).uniform_()
        self.anc_keypoints = torch.empty(B, 3, M, device=dev); self.anc_sigmas = torch.empty(B, M, device=dev)
        self.pos_pc = torch.empty(B, 3, N, device=dev).uniform_(); self.pos_sn = torch.empty(B, 3, N, device=dev).uniform_()
        self.pos_keypoints = torch.empty(B, 3, M, device=dev); self.pos_sigmas = torch.empty(B, M, device=dev)
        self.anc_R_pos = torch.zeros((B, 3, 3), dtype=torch.float32, device=dev)
        self.anc_scale_pos = torch.zeros((B, 1), dtype=torch.float32, device=dev)
        self.anc_shift_pos = torch.zeros((B, 3, 1), dtype=torch.float32, device=dev)
        z = lambda: torch.tensor([0], dtype=torch.float32, requires_grad=False, device=dev)
        self.test_loss_average = z(); self.test_loss_triplet_average = z(); self.test_active_percentage_average = z()

    _INPUT_FIELDS = ("anc_pc", "anc_sn", "anc_keypoints", "anc_sigmas", "pos_pc", "pos_sn", "pos_keypoints",
                     "pos_sigmas", "anc_R_pos", "anc_scale_pos", "anc_shift_pos")

    def set_input(self, anc_pc, anc_sn, anc_keypoints, anc_sigmas, pos_pc, pos_sn, pos_keypoints, pos_sigmas,
                  anc_R_pos, anc_scale_pos, anc_shift_pos):
        """keypoint_descriptor.py:369-389.  If the same tensors were staged by prefetch_input(), the staged device copies
        are adopted with a stream-side wait instead of eleven copies and a host synchronisation."""
        args = (anc_pc, anc_sn, anc_keypoints, anc_sigmas, pos_pc, pos_sn, pos_keypoints, pos_sigmas, anc_R_pos,
                anc_scale_pos, anc_shift_pos)
        st = getattr(self, "_staged", None)
        if st is not None and len(st[0]) == len(args) and all(a is b for a, b in zip(st[0], args)):
            cur = torch.cuda.current_stream()
            cur.wait_event(st[2])
            for k, v in zip(self._INPUT_FIELDS, st[1]):
                v.record_stream(cur)                                  # allocated on another stream, consumed here
                setattr(self, k, v)
            self._staged = None
            return
        dev = self.opt.device
        self.anc_pc = anc_pc.float().to(dev); self.anc_sn = anc_sn.float().to(dev)
        self.anc_keypoints = anc_keypoints.float().to(dev); self.anc_sigmas = anc_sigmas.float().to(dev)
        self.pos_pc = pos_pc.float().to(dev); self.pos_sn = pos_sn.float().to(dev)
        self.pos_keypoints = pos_keypoints.float().to(dev); self.pos_sigmas = pos_sigmas.float().to(dev)
        self.anc_R_pos = anc_R_pos.float().to(dev); self.anc_scale_pos = anc_scale_pos.float().to(dev)
        self.anc_shift_pos = anc_shift_pos.float().to(dev)
        torch.cuda.synchronize()

    def prefetch_input(self, *args, after=None):
        """Not in the reference: stage the NEXT batch (the eleven set_input tensors) with asynchronous host-to-device
        copies on a dedicated stream, so that the transfer overlaps the running step; the following set_input() with the
        same tensor objects adopts the staged copies.  `after`: a CUDA event the staging waits for (device tensors
        produced on another stream, e.g. by SceneNNDescriptorPairSource)."""
        if len(args) != len(self._INPUT_FIELDS):
            raise TypeError("prefetch_input takes the eleven set_input tensors, got %d" % len(args))
        dev = self.opt.device
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        if after is not None:
            self._copy_stream.wait_event(after)
        with torch.cuda.stream(self._copy_stream):
            staged = [a.float().to(dev, non_blocking=True).detach() for a in args]
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        self._staged = (tuple(args), staged, ev)

    def forward(self, pc, sn, keypoints, is_train=False, epoch=None):
        with torch.cuda.device(pc.get_device()):
            return self.descriptor(pc, sn, keypoints, is_train, epoch)

    def forward_siamese(self, pc_tuple, sn_tuple, keypoints_tuple, is_train=False, epoch=None):
        n = pc_tuple[0].size()[0]
        descriptors, x_aug_ball = self.descriptor(torch.cat(pc_tuple, dim=0), torch.cat(sn_tuple, dim=0),
                                                  torch.cat(keypoints_tuple, dim=0), is_train, epoch)
        return torch.split(descriptors, n, dim=0), torch.split(x_aug_ball, n, dim=0)

    def _require_cuda(self):
        if not self.anc_pc.is_cuda or self.optimizer_descriptor is None:
            raise NotImplementedError("ModelDescriptorIndoor: " + self._NO_CPU)

    def _transform_anchor_keypoints(self):
        """keypoint_descriptor.py:474-477: R @ kp * scale + shift (the keypoints are data: no gradient)."""
        B = self.anc_keypoints.shape[0]
        self.anc_keypoints_transformed = ops.transform_points(
            self.anc_keypoints.contiguous(), self.anc_R_pos.contiguous(), self.anc_scale_pos.reshape(B).contiguous(),
            self.anc_shift_pos.reshape(B, 3).contiguous())

    def _loss(self):
        """keypoint_descriptor.py:483-491: DescCGFLoss of the anchors (mapped into the positive frame) against the
        positives, averaged.  The reference also maps the anchor cloud, which the loss does not read; that is skipped."""
        self._transform_anchor_keypoints()
        triplet_loss, active_percentage = self.triplet_criteria(self.anc_keypoints_transformed, self.anc_descriptors,
                                                                self.pos_keypoints, self.pos_descriptors, self.anc_sigmas)
        self.triplet_loss = torch.mean(triplet_loss)
        self.active_percentage = torch.mean(active_percentage)
        self.loss = self.triplet_loss

    def optimize(self, epoch=None):
        """keypoint_descriptor.py:451-497: optional random point dropout (same RNG streams), train-mode forward of the
        (anchor, positive) batch, DescCGFLoss, backward, Adam.  Nothing before the loss draws from the CUDA generator, so
        the loss's three draws are the reference's."""
        self._require_cuda()
        if self.opt.random_pc_dropout_lower_limit < 0.99 and self.anc_pc.shape[2] != self.opt.input_pc_num:
            raise ValueError("ModelDescriptorIndoor.optimize: the staged batch has %d points, not input_pc_num=%d -- point "
                             "dropout thins the batch in place, so set_input() a new batch before every step"
                             % (self.anc_pc.shape[2], self.opt.input_pc_num))
        with torch.cuda.device(self.anc_pc.get_device()):
            self.anc_pc, self.anc_sn, self.pos_pc, self.pos_sn = random_point_dropout(
                self.opt, self.anc_pc, self.anc_sn, self.pos_pc, self.pos_sn)
            self.descriptor.train()
            (self.anc_descriptors, self.pos_descriptors), _ = self.forward_siamese(
                (self.anc_pc, self.pos_pc), (self.anc_sn, self.pos_sn), (self.anc_keypoints, self.pos_keypoints),
                is_train=True, epoch=epoch)
            self.optimizer_descriptor.zero_grad()
            self._loss()
            self.loss.backward()
            self.optimizer_descriptor.step()

    def test_model(self):
        """keypoint_descriptor.py:499-519: eval-mode forward and the loss; no parameter or running statistic changes."""
        self._require_cuda()
        self.descriptor.eval()
        with torch.cuda.device(self.anc_pc.device), torch.no_grad():
            (self.anc_descriptors, self.pos_descriptors), _ = self.forward_siamese(
                (self.anc_pc, self.pos_pc), (self.anc_sn, self.pos_sn), (self.anc_keypoints, self.pos_keypoints),
                is_train=False, epoch=None)
            self._loss()

    def freeze_model(self):
        for p in self.descriptor.parameters():
            p.requires_grad = False

    def run_model(self, pc, sn, keypoints):
        self.descriptor.eval()
        with torch.cuda.device(pc.device), torch.no_grad():
            descriptors, _ = self.descriptor(pc, sn, keypoints, False, None)
        return descriptors

    def get_current_visuals(self):
        raise NotImplementedError("visdom payloads (keypoint_descriptor.py:540-572) are outside the hot path")

    def get_current_errors(self):
        return OrderedDict([('O_loss', self.loss.item()), ('O_triplet', self.triplet_loss.item()),
                            ('O_active_perc', self.active_percentage.item()), ('E_loss', self.test_loss_average.item()),
                            ('E_triplet', self.test_loss_triplet_average.item()),
                            ('E_active_perc', self.test_active_percentage_average.item())])

    def save_network(self, network, network_label, epoch_label, gpu_id):
        torch.save(network.state_dict(), os.path.join(self.opt.checkpoints_dir, '%s_net_%s.pth' % (epoch_label, network_label)))

    def update_learning_rate(self, ratio):
        lr = max(self.old_lr_descriptor * ratio, 0.00001)
        for g in self.optimizer_descriptor.param_groups:
            g['lr'] = lr
        print('update descriptor learning rate: %f -> %f' % (self.old_lr_descriptor, lr))
        self.old_lr_descriptor = lr
