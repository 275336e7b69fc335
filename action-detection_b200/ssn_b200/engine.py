"""Host-side wrappers over the C ABI: engine lifetime, autograd bridges.  PyTorch is plumbing here
(device memory, streams, autograd bookkeeping); every arithmetic op runs in libssn_b200.so."""
import ctypes as C

import torch

from . import _lib
from ._lib import lib, check


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: libssn_b200 has no CPU path" % name)


def conv_table(in_channels):
    """[(name, cin, cout, k, stride, pad)] straight from the library (graph order)."""
    out = []
    buf = C.create_string_buffer(128)
    v = [C.c_int() for _ in range(5)]
    for i in range(lib.ssnb_num_convs()):
        check(lib.ssnb_conv_info(i, in_channels, buf, 128, *[C.byref(x) for x in v]), None, "conv_info")
        out.append((buf.value.decode(),) + tuple(x.value for x in v))
    return out


class PlannedEngine:
    """A planned backbone engine handle `h` of `workspace_bytes` and what every such handle needs: its workspace on `device`
    (1024-byte aligned, as the library requires), the BatchNorm-folded weight pack, and destruction with the object.  A
    subclass names its library functions and says where the library keeps its errors: on the handle (ssnb_*) or per
    thread (ssnb_iv3_*, read with ssnb_last_error(NULL))."""
    _set_workspace_fn = _pack_fn = _destroy_fn = None
    _errors_on_handle = True

    def _err(self):
        return self.h if self._errors_on_handle else None

    def _call(self, fn, *args):
        check(getattr(lib, fn)(self.h, *args), self._err(), fn[len("ssnb_"):])

    def _set_workspace(self):
        with torch.cuda.device(self.device):
            self._ws = torch.empty(self.workspace_bytes + 1024, dtype=torch.uint8, device=self.device)
            base = self._ws.data_ptr()
            self.ws_ptr = base + ((-base) % 1024)
            self._call(self._set_workspace_fn, C.c_void_p(self.ws_ptr), self.workspace_bytes)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                getattr(lib, self._destroy_fn)(self.h)
                self.h = None
        except Exception:
            pass

    def pack(self, w, b, gamma, beta, mean, var):
        """lists of one tensor per convolution each, reference shapes (graph order)"""
        with torch.cuda.device(self.device):
            self._call(self._pack_fn, *[_lib.ptr_array(x) for x in (w, b, gamma, beta, mean, var)], _stream())


class BackboneEngine(PlannedEngine):
    """One planned BNInception instance for a fixed frame count (ssnb_create .. ssnb_destroy).  A forward-only engine
    (training=False) also runs any smaller frame count on the same workspace.  device=None plans without allocating (the
    plan needs no GPU)."""
    _set_workspace_fn, _pack_fn, _destroy_fn = "ssnb_set_workspace", "ssnb_pack_weights", "ssnb_destroy"

    def __init__(self, in_channels, frames, precision, training, grad_scale, device, bn1_train=False):
        self.device = None if device is None else torch.device(device)
        self.frames, self.in_channels, self.precision, self.training = frames, in_channels, precision, training
        self.bn1_train = bool(bn1_train)
        cfg = _lib.Config(in_channels, frames, precision, 1 if training else 0, float(grad_scale), 1 if bn1_train else 0)
        self.h = C.c_void_p()
        check(lib.ssnb_create(C.byref(cfg), C.byref(self.h)), None, "ssnb_create")
        self.workspace_bytes = lib.ssnb_workspace_bytes(self.h)
        if self.device is not None:
            self._set_workspace()
        self.packed_version = None
        self.generation = 0        # bumped by every forward: the saved activations belong to the latest one only

    def set_bn1(self, bn, dgamma=None, dbeta=None):
        """bn1_train engines: the first BatchNorm2d module's tensors (training-mode statistics, running-stat update, gradients)"""
        check(lib.ssnb_set_bn1(self.h, bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                               None if dgamma is None else dgamma.data_ptr(), None if dbeta is None else dbeta.data_ptr(),
                               float(bn.momentum if bn.momentum is not None else 0.1), float(bn.eps)), self.h, "set_bn1")

    def forward(self, x):
        """x [n, C, 224, 224] -> feat [n, 1024]; n < frames (forward-only engines) runs the first n frames of the plan"""
        _need_cuda(x, "input")
        x = x.contiguous().float()
        n = x.shape[0]
        assert 1 <= n <= self.frames and x.shape[1] == self.in_channels and tuple(x.shape[2:]) == (224, 224), \
            "engine planned for [<=%d,%d,224,224], got %s" % (self.frames, self.in_channels, tuple(x.shape))
        feat = torch.empty(n, 1024, dtype=torch.float32, device=x.device)
        self.generation += 1
        with torch.cuda.device(self.device):
            if n == self.frames:
                check(lib.ssnb_backbone_fwd(self.h, C.c_void_p(x.data_ptr()), C.c_void_p(feat.data_ptr()), _stream()),
                      self.h, "backbone_fwd")
            else:
                check(lib.ssnb_backbone_fwd_frames(self.h, C.c_void_p(x.data_ptr()), n, C.c_void_p(feat.data_ptr()), _stream()),
                      self.h, "backbone_fwd_frames")
        return feat

    def backward(self, dfeat, dw, db, accumulate=False, buckets=None, on_bucket=None):
        """buckets: list of (op_hi, op_lo) ranges from the top of the network down (see bucket_ranges); on_bucket(i) runs
        after range i has been enqueued -- its convolutions' gradients are final then (bucketed gradient exchange)."""
        dfeat = dfeat.contiguous().float()
        check(lib.ssnb_set_grad_accumulate(self.h, int(accumulate)), self.h, "set_grad_accumulate")
        with torch.cuda.device(self.device):
            if not buckets:
                check(lib.ssnb_backbone_bwd(self.h, C.c_void_p(dfeat.data_ptr()), _lib.ptr_array(dw), _lib.ptr_array(db),
                                            _stream()), self.h, "backbone_bwd")
                return
            pw, pb = _lib.ptr_array(dw), _lib.ptr_array(db)
            for i, (hi, lo) in enumerate(buckets):
                check(lib.ssnb_backbone_bwd_range(self.h, C.c_void_p(dfeat.data_ptr()), pw, pb, hi, lo, _stream()), self.h, "backbone_bwd_range")
                if on_bucket is not None:
                    on_bucket(i)

    def bucket_ranges(self, first_ops):
        """first_ops: names of the convolutions that start a bucket, top of the network first (e.g. ['inception_4e_3x3_reduce',
        'inception_3c_3x3_reduce']); returns [(op_hi, op_lo)] covering all ops and, per bucket, the index of its first conv in
        graph order (for slicing a flat gradient buffer laid out in parameter order)."""
        ops = self.ops()
        conv_idx, k = {}, 0
        first_of = {}
        for i, (kind, _iname, oname) in enumerate(ops):
            if kind == "conv":
                conv_idx[oname[:-3]] = (i, k)
                k += 1
        cuts = sorted([conv_idx[n] for n in first_ops], reverse=True)       # (op index, conv index), top first
        ranges, convs = [], []
        hi = len(ops) - 1
        for (oi, ci) in cuts:
            ranges.append((hi, oi)); convs.append(ci)
            hi = oi - 1
        if hi >= 0:
            ranges.append((hi, 0)); convs.append(0)
        return ranges, convs

    # ---- introspection used by the per-layer parity tests ----
    def ops(self):
        out = []
        k, i, o = (C.create_string_buffer(64), C.create_string_buffer(128), C.create_string_buffer(128))
        for n in range(lib.ssnb_num_ops(self.h)):
            check(lib.ssnb_op_info(self.h, n, k, 64, i, 128, o, 128), self.h, "op_info")
            out.append((k.value.decode(), i.value.decode(), o.value.decode()))
        return out

    def value_shape(self, name):
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        check(lib.ssnb_value_shape(self.h, name.encode(), C.byref(c), C.byref(h), C.byref(w)), self.h, "value_shape")
        return c.value, h.value, w.value

    def write(self, name, t, grad=False):
        c, h, w = self.value_shape(name)
        t = t.contiguous().float()
        assert tuple(t.shape) == (self.frames, c, h, w), (name, tuple(t.shape), (self.frames, c, h, w))
        with torch.cuda.device(self.device):
            check(lib.ssnb_value_write(self.h, name.encode(), int(grad), C.c_void_p(t.data_ptr()), _stream()), self.h, "value_write")

    def read(self, name, grad=False, planes=False):
        """planes=True (EXACT_TC only): hi + lo of the value's fp16 operand planes instead of the fp32 tensor."""
        c, h, w = self.value_shape(name)
        t = torch.empty(self.frames, c, h, w, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib.ssnb_value_read(self.h, name.encode(), int(grad) | (2 if planes else 0), C.c_void_p(t.data_ptr()), _stream()),
                  self.h, "value_read")
        return t

    def run_op(self, idx, backward=False):
        with torch.cuda.device(self.device):
            check(lib.ssnb_run_op(self.h, idx, int(backward), _stream()), self.h, "run_op")

    def bind_grads(self, dw, db):
        check(lib.ssnb_bind_grads(self.h, _lib.ptr_array(dw), _lib.ptr_array(db)), self.h, "bind_grads")

    def grad_overflow(self, clear=True):
        """EXACT_TC: True when a gradient operand plane left the fp16 range under the current grad_scale (device sync)."""
        return lib.ssnb_grad_overflow(self.h, int(clear)) == 1

    def launch_count(self):
        return lib.ssnb_launch_count(self.h)


class BackboneFunction(torch.autograd.Function):
    """autograd bridge: feat = BNInception(x); backward produces the Conv2d weight/bias gradients
    (BatchNorm2d is frozen, ssn_models.py:156-174, so it gets none).

    With direct_grad (default) the kernels add straight into each parameter's .grad (allocating it
    when it is None), exactly what autograd's AccumulateGrad would do with returned gradients, but
    without 138 temporary tensors and 138 tiny add kernels per step; the Function then returns None
    for the parameters.  That shortcut is only taken when it is indistinguishable from autograd: every
    parameter is a leaf tensor without hooks (nn.DataParallel replicas are non-leaf; DDP and user code
    register hooks) -- otherwise, or with BackboneFunction.direct_grad = False, ordinary gradients are
    returned (also needed for torch.autograd.grad).

    The engine keeps ONE set of saved activations per frame count: a second forward through the same
    engine before this node's backward overwrites them, which is detected (generation counter) and raised."""
    direct_grad = True

    @staticmethod
    def forward(ctx, x, engine, n_conv, bn1, *wb):
        # wb = 69 conv weights, 69 conv biases (+ the weight and bias of bn1, the first BatchNorm2d module, for a bn1_train engine)
        ctx.engine, ctx.n_conv, ctx.bn1 = engine, n_conv, bn1
        ctx.params = wb
        feat = engine.forward(x)
        ctx.generation = engine.generation
        return feat

    @staticmethod
    def _direct_ok(params):
        for p in params:
            if not p.requires_grad:
                continue
            if not p.is_leaf or getattr(p, "_backward_hooks", None) or getattr(p, "_post_accumulate_grad_hooks", None):
                return False
        return True

    @staticmethod
    def backward(ctx, dfeat):
        eng, n = ctx.engine, ctx.n_conv
        dev = dfeat.device
        if ctx.generation != eng.generation:
            raise RuntimeError("BNInception(H100): another forward of %d frames ran through this engine after the one being "
                               "differentiated; its saved activations are gone.  Run backward before the next forward of the same "
                               "shape (or use different frame counts / a second model instance)." % eng.frames)
        bn1 = getattr(ctx, "bn1", None)
        if BackboneFunction.direct_grad and BackboneFunction._direct_ok(ctx.params):
            grads = []
            for p in ctx.params:
                if not p.requires_grad:
                    grads.append(None)
                    continue
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
                grads.append(p.grad)
            if bn1 is not None:
                eng.set_bn1(bn1, grads[2 * n], grads[2 * n + 1])
            eng.backward(dfeat, grads[:n], grads[n:2 * n], accumulate=True)
            return (None, None, None, None) + (None,) * len(ctx.params)
        grads = [torch.empty(p.shape, dtype=torch.float32, device=dev) if p.requires_grad else None for p in ctx.params]
        if bn1 is not None:
            eng.set_bn1(bn1, grads[2 * n], grads[2 * n + 1])
        eng.backward(dfeat, grads[:n], grads[n:2 * n])
        return (None, None, None, None) + tuple(grads)


# ---- STPP ---------------------------------------------------------------------------------------------
def parse_stage_config(cfg):
    if isinstance(cfg, int):
        return (cfg,), cfg
    if isinstance(cfg, (tuple, list)):
        return tuple(cfg), sum(cfg)
    raise ValueError("Incorrect STPP config {}".format(cfg))


def stpp_part_table(parts, norm_num, seg_split):
    """Integer part boundaries for ops/ssn_ops.py:49-53 — same float arange + int() truncation."""
    x1, x2, n_seg = seg_split
    bounds = ((0, x1, 0), (x1, x2, -1), (x2, n_seg, 1))
    lo, hi, nm, col = [], [], [], []
    for (a, b, c), stage_parts, norm in zip(bounds, parts, norm_num):
        stage_len = b - a
        for n_part in stage_parts:
            ticks = torch.arange(0, stage_len + 1e-5, stage_len / n_part)
            for i in range(n_part):
                lo.append(a + int(ticks[i])); hi.append(a + int(ticks[i + 1])); nm.append(norm); col.append(c)
    return lo, hi, nm, col


class STPPFunction(torch.autograd.Function):
    """(course_ft, stpp_ft) = STPP(ft).  An empty part table means the course mean alone (BinaryClassifier's segment mean);
    scaling may then be None and stpp_ft is [n, 0]."""

    @staticmethod
    def forward(ctx, ft, scaling, table, n_seg, course):
        _need_cuda(ft, "ft")
        lo, hi, nm, col = table
        ft = ft.contiguous().float()
        if scaling is not None:
            scaling = scaling.contiguous().float().view(-1, 2)
        D = ft.shape[1]
        n = ft.shape[0] // n_seg
        act = torch.empty(n, D, dtype=torch.float32, device=ft.device)
        comp = torch.empty(n, len(lo) * D, dtype=torch.float32, device=ft.device)
        with torch.cuda.device(ft.device):
            check(lib.ssnb_stpp_fwd(ft.data_ptr(), None if scaling is None else scaling.data_ptr(), n, n_seg, D, len(lo),
                                    _lib.int_array(lo), _lib.int_array(hi), _lib.int_array(nm), _lib.int_array(col), course[0],
                                    course[1], act.data_ptr(), comp.data_ptr() if lo else None, _stream()), None, "stpp_fwd")
        ctx.save_for_backward(scaling)
        ctx.meta = (table, n_seg, course, n, D)
        return act, comp

    @staticmethod
    def backward(ctx, d_act, d_comp):
        (scaling,) = ctx.saved_tensors
        (lo, hi, nm, col), n_seg, course, n, D = ctx.meta
        d_act = d_act.contiguous().float()
        d_comp = d_comp.contiguous().float()
        dft = torch.empty(n * n_seg, D, dtype=torch.float32, device=d_comp.device)
        with torch.cuda.device(d_comp.device):
            check(lib.ssnb_stpp_bwd(d_act.data_ptr(), d_comp.data_ptr() if lo else None, None if scaling is None else scaling.data_ptr(),
                                    n, n_seg, D, len(lo),
                                    _lib.int_array(lo), _lib.int_array(hi), _lib.int_array(nm), _lib.int_array(col),
                                    course[0], course[1], dft.data_ptr(), _stream()), None, "stpp_bwd")
        return dft, None, None, None, None


class LinearFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        _need_cuda(x, "x")
        x = x.contiguous().float()
        n, i = x.shape
        o = w.shape[0]
        y = torch.empty(n, o, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.ssnb_linear_fwd(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), n, i, o,
                                      y.data_ptr(), _stream()), None, "linear_fwd")
        ctx.save_for_backward(x, w)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = dy.contiguous().float()
        n, i = x.shape
        o = w.shape[0]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(w)
        db = torch.empty(o, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.ssnb_linear_bwd(x.data_ptr(), w.data_ptr(), dy.data_ptr(), n, i, o,
                                      None if dx is None else dx.data_ptr(), dw.data_ptr(), db.data_ptr(), _stream()),
                  None, "linear_bwd")
        return dx, dw, (db if ctx.has_bias else None)


def heads_loss_fused(course_ft, stpp_ft, act_fc, comp_fc, reg_fc, prop_type, target, reg_target, num_class,
                     feat_mult, fg_per_video=1, comp_group=7, props_per_video=8, ohem_ratio=0.17, comp_w=0.1,
                     reg_w=0.1, global_videos=None, loss_scale=1.0, want_grads=True):
    """One kernel: three heads + CE/OHEM/smooth-L1 + every gradient (ssn_models.py:272-289,
    ssn_train.py:210-214).  Returns dict of tensors."""
    dev = course_ft.device
    n = course_ft.shape[0]
    K, D = num_class, course_ft.shape[1]
    videos = n // props_per_video
    gv = videos if global_videos is None else global_videos
    neg = comp_group - fg_per_video
    denom_global = gv * fg_per_video + int(gv * neg * ohem_ratio)
    cfg = _lib.HeadsCfg(n, props_per_video, K, D, feat_mult, fg_per_video, comp_group, gv,
                        int(neg * ohem_ratio), float(denom_global) * videos / gv, comp_w, reg_w, loss_scale)
    f32 = dict(dtype=torch.float32, device=dev)
    out = {"raw_act": torch.empty(n, K + 1, **f32), "raw_comp": torch.empty(n, K, **f32),
           "raw_reg": torch.empty(n, 2 * K, **f32), "losses": torch.empty(4, **f32),
           "d_course": torch.empty_like(course_ft), "d_stpp": torch.empty_like(stpp_ft),
           "d_act_w": torch.empty_like(act_fc.weight), "d_act_b": torch.empty_like(act_fc.bias),
           "d_comp_w": torch.empty_like(comp_fc.weight), "d_comp_b": torch.empty_like(comp_fc.bias),
           "d_reg_w": torch.empty_like(reg_fc.weight), "d_reg_b": torch.empty_like(reg_fc.bias)}
    ws = torch.empty(lib.ssnb_heads_loss_workspace_bytes(C.byref(cfg)), dtype=torch.uint8, device=dev)
    pt = prop_type.reshape(-1).contiguous().long()
    tg = target.reshape(-1).contiguous().long()
    rt = reg_target.reshape(-1, 2).contiguous().float()
    args = [course_ft, stpp_ft, act_fc.weight, act_fc.bias, comp_fc.weight, comp_fc.bias, reg_fc.weight, reg_fc.bias,
            pt, tg, rt, out["raw_act"], out["raw_comp"], out["raw_reg"], out["losses"], out["d_course"], out["d_stpp"],
            out["d_act_w"], out["d_act_b"], out["d_comp_w"], out["d_comp_b"], out["d_reg_w"], out["d_reg_b"], ws]
    with torch.cuda.device(dev):
        check(lib.ssnb_heads_loss_fwd_bwd(C.byref(cfg), *[C.c_void_p(t.data_ptr()) for t in args], _stream()), None,
              "heads_loss_fwd_bwd")
    return out
