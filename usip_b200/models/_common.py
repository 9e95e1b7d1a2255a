"""Host-side helpers shared by ModelDetector, ModelDescriptor and ModelDescriptorIndoor."""
import random

import numpy as np
import torch


def random_point_dropout(opt, *clouds):
    """Training-time point dropout of both model wrappers (keypoint_detector.py:161-169, keypoint_descriptor.py:128-137):
    unless `random_pc_dropout_lower_limit >= 0.99`, keep round(u * input_pc_num) randomly chosen point columns, the same
    ones in every (B, C, N) tensor given.  The random numbers are drawn like the reference does -- one random.uniform,
    then one np.random.choice without replacement -- so seeded runs keep the same points."""
    if opt.random_pc_dropout_lower_limit >= 0.99:
        return clouds
    n_keep = round(random.uniform(opt.random_pc_dropout_lower_limit, 1.0) * opt.input_pc_num)
    columns = torch.from_numpy(np.random.choice(opt.input_pc_num, n_keep, replace=False)).to(opt.device)
    return tuple(torch.index_select(c, 2, columns) for c in clouds)


class StagedInput:
    """set_input / prefetch_input of the three models.  A batch is the tensors named in the model's `_INPUT_FIELDS`, in
    set_input's order; they are stored on `opt.device` as float32, except the fields in `_INT64_FIELDS`."""
    _INPUT_FIELDS = ()
    _INT64_FIELDS = ()

    def _to_device(self, field, a):
        a = a.long() if field in self._INT64_FIELDS else a.float()
        return a.to(self.opt.device, non_blocking=True).detach()

    def _set_input(self, args):
        """The reference's set_input: copy the batch to the device, then synchronise.  If the same tensors were staged by
        prefetch_input(), the staged device copies are adopted with a stream-side wait instead."""
        st = getattr(self, "_staged", None)
        if st is not None and len(st[0]) == len(args) and all(a is b for a, b in zip(st[0], args)):
            cur = torch.cuda.current_stream()
            cur.wait_event(st[2])
            for k, v in zip(self._INPUT_FIELDS, st[1]):
                v.record_stream(cur)                                  # allocated on the copy stream, consumed here
                setattr(self, k, v)
            self._staged = None
            return
        for k, a in zip(self._INPUT_FIELDS, args):
            setattr(self, k, self._to_device(k, a))
        torch.cuda.synchronize()

    def prefetch_input(self, *args, after=None):
        """Not in the reference: stage the NEXT batch (the set_input tensors, ideally pinned if on the host) with
        asynchronous copies on a dedicated stream, so that the transfer overlaps the step that is running.  The following
        set_input() with the same tensor objects adopts the staged copies.  `after`: a CUDA event the staging waits for
        (device tensors produced on another stream, e.g. by a pair builder)."""
        if len(args) != len(self._INPUT_FIELDS):
            raise TypeError("prefetch_input takes the %d set_input tensors, got %d" % (len(self._INPUT_FIELDS), len(args)))
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.opt.device)
        if after is not None:
            self._copy_stream.wait_event(after)
        with torch.cuda.stream(self._copy_stream):
            staged = [self._to_device(k, a) for k, a in zip(self._INPUT_FIELDS, args)]
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        self._staged = (tuple(args), staged, ev)
