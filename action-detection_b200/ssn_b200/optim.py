"""Fused SGD-momentum over flat fp32 buffers (replaces torch.optim.SGD as configured by ssn_train.py:141-144 with the
parameter groups of SSN.get_optim_policies and the per-group lr_mult / decay_mult of adjust_learning_rate, :391-398).

All parameters live in ONE flat buffer (p.data are views), all gradients in another (p.grad are views: one ncclAllReduce
exchanges them, ssn_b200/dp.py), the momentum in a third; a step is ONE kernel launch (ssnb_sgd_step_groups) instead of
~6 foreach launches per group.  Same arithmetic as torch.optim.SGD(momentum, weight_decay, dampening=0, nesterov=False).

step(max_norm=...) and clip_grad_norm add the rest of the reference's update block (ssn_train.py:238-250,
binary_train.py:185-197): the iter_size division and clip_grad_norm, with the norm left on the device, so the whole step
stays capturable in a CUDA graph."""
import ctypes as C

import torch

from ._lib import lib, check, ExtraGrads, GRAD_NORM_CTAS, MAX_EXTRA_GRADS


def _extra_grads(tensors, device):
    """ssnb_extra_grads of gradient tensors the flat buffer does not hold (fp32, contiguous, on the optimiser's device)"""
    tensors = list(tensors)
    if len(tensors) > MAX_EXTRA_GRADS:
        raise ValueError("at most %d extra gradients, got %d" % (MAX_EXTRA_GRADS, len(tensors)))
    ex = ExtraGrads()
    ex.count = len(tensors)
    for i, t in enumerate(tensors):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
            raise ValueError("extra gradient %d must be a contiguous fp32 tensor on %s" % (i, device))
        ex.grad[i], ex.numel[i] = t.data_ptr(), t.numel()
    return ex


class FusedSGD:
    def __init__(self, policies, lr, momentum=0.9, weight_decay=5e-4, on_step=None, order=None):
        """policies: list of dicts with 'params', 'lr_mult', 'decay_mult' (SSN.get_optim_policies()).  on_step: callables run
        after every step (e.g. BNInception.invalidate_packed: the kernels' packed weight copies are stale).  order: the
        parameters in the order they should occupy the flat buffers (default: group by group; model.parameters() order
        puts each layer's weight and bias side by side, which ssn_b200.dp.GradSync's buckets need)."""
        self.param_groups = []
        for g in policies:
            ps = [p for p in g["params"] if p.requires_grad]
            if ps:
                d = dict(g)
                d["params"] = ps
                d["lr"] = lr * g.get("lr_mult", 1)
                d["weight_decay"] = weight_decay * g.get("decay_mult", 1)
                self.param_groups.append(d)
        self.momentum = float(momentum)
        self.on_step = list(on_step or [])
        params = [p for g in self.param_groups for p in g["params"]]
        self._group_of = {id(p): g for g in self.param_groups for p in g["params"]}
        if order is not None:
            order = [p for p in order if id(p) in self._group_of]
            assert len(order) == len(params), "order must list exactly the parameters of the groups"
            params = order
        self.params = params
        assert params and all(p.is_cuda and p.dtype == torch.float32 for p in params), "FusedSGD: fp32 CUDA parameters"
        dev = params[0].device
        self.device = dev
        n = sum(p.numel() for p in params)
        self.flat_param = torch.empty(n, device=dev)
        self.flat_grad = torch.zeros(n, device=dev)
        self.flat_mom = torch.zeros(n, device=dev)
        self.views = []
        off = 0
        for p in params:
            k = p.numel()
            self.flat_param[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat_param[off:off + k].view_as(p)
            p.grad = self.flat_grad[off:off + k].view_as(p)
            self.views.append((p, off, k))
            off += k
        self.n = n
        self._seg_end = torch.tensor([o + k for (_p, o, k) in self.views], dtype=torch.int64, device=dev)
        self._seg_lr = torch.empty(len(self.views), device=dev)
        self._seg_wd = torch.empty(len(self.views), device=dev)
        # the gradient norm of step(max_norm=...) and clip_grad_norm: one device scalar, rewritten by every call (a CUDA graph
        # replays into the same tensor), and the fp64 per-CTA partials it is reduced from
        self.norm = torch.zeros((), device=dev)
        self._norm_partials = torch.empty(GRAD_NORM_CTAS, dtype=torch.float64, device=dev)
        self.refresh_groups()

    def refresh_groups(self):
        """re-read lr / weight_decay of every group (call after adjust_learning_rate changed them)"""
        lr = [float(self._group_of[id(p)]["lr"]) for p in self.params]
        wd = [float(self._group_of[id(p)]["weight_decay"]) for p in self.params]
        self._seg_lr.copy_(torch.tensor(lr)); self._seg_wd.copy_(torch.tensor(wd))

    def rebind_grads(self):
        """p.grad must alias the flat gradient buffer (zero_grad(set_to_none=True) or an assignment breaks it): re-attach,
        keeping whatever gradient the parameter holds"""
        for p, off, k in self.views:
            view = self.flat_grad[off:off + k].view_as(p)
            if p.grad is None:
                view.zero_()
                p.grad = view
            elif p.grad.data_ptr() != view.data_ptr():
                view.copy_(p.grad)
                p.grad = view

    def zero_grad(self, set_to_none=False):
        self.flat_grad.zero_()
        self.rebind_grads()

    def ungrouped(self, params):
        """the parameters of `params` (model.parameters()) that need a gradient but no group holds: the extra_grads of
        step() and clip_grad_norm (the first BatchNorm2d's weight and bias under bn_mode='partial')"""
        return [p for p in params if p.requires_grad and id(p) not in self._group_of]

    def _grad_norm(self, grad_mult, ex):
        check(lib.ssnb_grad_norm(self.flat_grad.data_ptr(), self.n, float(grad_mult), C.byref(ex), self._norm_partials.data_ptr(),
                                 self.norm.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "grad_norm")

    def step(self, grad_mult=1.0, max_norm=None, extra_grads=(), write_back=True):
        """One update.  grad_mult multiplies every gradient of the groups (1 / iter_size for the reference's p.grad /=
        iter_size).  max_norm: clip_grad_norm(model.parameters(), max_norm) first, over the groups' gradients after that
        division plus extra_grads (gradient tensors of parameters no group holds, see ungrouped(); not divided, as in the
        reference); the norm is computed and applied on the device and returned as a 0-d fp32 tensor (self.norm, rewritten
        by every call), else None.  write_back: leave the divided and clipped gradients in .grad and extra_grads, as the
        reference's .grad holds them before optimizer.step(); False leaves them as they were.  Under ssn_b200.dp.GradSync
        call it after sync.finish(): the norm is then that of the exchanged gradients, the same on every rank."""
        self.rebind_grads()
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        with torch.cuda.device(self.device):
            if max_norm is None:
                check(lib.ssnb_sgd_step_groups(self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.flat_mom.data_ptr(), self.n,
                                               self._seg_end.data_ptr(), self._seg_lr.data_ptr(), self._seg_wd.data_ptr(), len(self.views),
                                               self.momentum, float(grad_mult), stream), None, "sgd_step_groups")
                norm = None
            else:
                ex = _extra_grads(extra_grads, self.device)
                self._grad_norm(grad_mult, ex)
                check(lib.ssnb_sgd_step_groups_clipped(self.flat_param.data_ptr(), self.flat_grad.data_ptr(), self.flat_mom.data_ptr(),
                                                       self.n, self._seg_end.data_ptr(), self._seg_lr.data_ptr(), self._seg_wd.data_ptr(),
                                                       len(self.views), self.momentum, float(grad_mult), self.norm.data_ptr(),
                                                       float(max_norm), 1 if write_back else 0, C.byref(ex), stream), None,
                      "sgd_step_groups_clipped")
                norm = self.norm
        for f in self.on_step:
            f()
        return norm


def clip_grad_norm(optimizer, max_norm, extra_grads=()):
    """torch.nn.utils.clip_grad_norm_ over the gradients a FusedSGD holds plus extra_grads, for loops that keep a separate
    optimizer.step(): the total L2 norm as a 0-d fp32 device tensor (optimizer.norm), and every gradient multiplied in
    place by max_norm / (norm + 1e-6) where that is < 1 (torch 0.3's rule, the reference's clip_grad_norm).  No host
    synchronisation: the `if total_norm > clip: print(...)` of the reference can read the returned tensor when it wants."""
    optimizer.rebind_grads()
    ex = _extra_grads(extra_grads, optimizer.device)
    with torch.cuda.device(optimizer.device):
        optimizer._grad_norm(1.0, ex)
        check(lib.ssnb_grad_clip(optimizer.norm.data_ptr(), float(max_norm), optimizer.flat_grad.data_ptr(), optimizer.n, C.byref(ex),
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "grad_clip")
    return optimizer.norm
