"""The training loop's meters on the device (replaces the AverageMeter updates of ssn_train.py:213-233 / :317-337 and
binary_train.py:170-180 / :235-243, with accuracy() of ssn_train.py:401-415 / binary_train.py:308-321).

The reference reads loss.data[0] and accuracy()[0].data[0] on every step: one host synchronisation each.  StepMeters
keeps the (sum, count) pairs of every meter in one fp64 device buffer that ssnb_train_meters updates with one launch per
step, so a step (or a CUDA graph of it) never waits for the host; read() synchronises once.

    meters = StepMeters("ssn", device)
    losses = model.fused_step(..., meters=meters)         # or meters.update_ssn(losses, ...) after a step of your own
    ...
    print(meters.read())                                  # {'loss': ..., 'act_acc': ..., ...}: AverageMeter.avg of each
    meters.reset()
"""
import ctypes as C

import torch

from ._lib import lib, check

# meter names in buffer order: the losses as fused_step returns them, then top-1 accuracy over all activity rows, the fg
# rows and the bg rows
_LOSSES = {"ssn": ("act_loss", "comp_loss", "reg_loss", "loss"), "binary": ("loss",)}
_ACC = ("act_acc", "fg_acc", "bg_acc")


class StepMeters:
    def __init__(self, kind, device):
        if kind not in _LOSSES:
            raise ValueError("kind must be 'ssn' or 'binary', got %r" % (kind,))
        self.kind = kind
        self.names = _LOSSES[kind] + _ACC
        self.device = torch.device(device)
        self.buf = torch.zeros(len(self.names), 2, dtype=torch.float64, device=self.device)

    def reset(self):
        self.buf.zero_()

    def _update(self, losses, scores, target, prop_type, batch_size):
        n_losses = len(_LOSSES[self.kind])
        losses = losses.reshape(-1)
        if losses.numel() != n_losses or losses.dtype != torch.float32:
            raise ValueError("%s meters take %d fp32 losses, got %s %s" % (self.kind, n_losses, tuple(losses.shape), losses.dtype))
        if scores.dim() != 2 or scores.dtype != torch.float32 or not scores.is_contiguous():
            raise ValueError("scores must be a contiguous fp32 [rows, classes] tensor")
        rows = scores.shape[0]
        target = target.reshape(-1).to(torch.int64).contiguous()
        if target.numel() != rows:
            raise ValueError("%d targets for %d score rows" % (target.numel(), rows))
        if prop_type is not None:
            prop_type = prop_type.reshape(-1).to(torch.int64).contiguous()
            if prop_type.numel() != rows:
                raise ValueError("%d proposal types for %d score rows" % (prop_type.numel(), rows))
        for t in (losses, scores, target) + ((prop_type,) if prop_type is not None else ()):
            if t.device != self.device:
                raise ValueError("meters live on %s, got a tensor on %s" % (self.device, t.device))
        with torch.cuda.device(self.device):
            check(lib.ssnb_train_meters(scores.data_ptr(), rows, scores.shape[1], target.data_ptr(),
                                        None if prop_type is None else prop_type.data_ptr(), losses.data_ptr(), n_losses,
                                        float(batch_size), self.buf.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  None, "train_meters")

    def update_ssn(self, losses, raw_act, target, prop_type, batch_size):
        """one SSN step: losses [4] (act, comp, reg, total) as fused_step returns them, raw_act [n, K+1] of every proposal
        (fused_step keeps it in last_fused), target and prop_type [n] (the activity rows are those of type 0 or 2), and the
        reference's out_frames.size(0), the videos of the batch.  fg / bg accuracy pair the activity rows two by two; an
        odd count (where the reference's view(-1, 2) raises) leaves the last one in act_acc only"""
        if self.kind != "ssn":
            raise ValueError("these are %s meters" % self.kind)
        self._update(losses, raw_act, target, prop_type, batch_size)

    def update_binary(self, loss, scores, target, batch_size):
        """one BinaryClassifier step: the mean loss [1], the scores [n, 2] of every proposal (last_fused['logits']), the
        targets [n] and out_frames.size(0)"""
        if self.kind != "binary":
            raise ValueError("these are %s meters" % self.kind)
        self._update(loss, scores, target, None, batch_size)

    def read(self):
        """AverageMeter.avg of every meter (0 for a meter that has seen nothing, as AverageMeter starts), with one
        synchronisation"""
        b = self.buf.cpu().tolist()
        return {n: (s / c if c else 0.0) for n, (s, c) in zip(self.names, b)}
