"""Host-side wrapper of the InceptionV3 test-time engine (ssnb_iv3_*, include/ssnb.h): plan, weights, forward and the
op-level introspection the launch-by-launch tests use."""
import ctypes as C

import torch

from . import _lib
from ._lib import lib, check
from .engine import PlannedEngine, _need_cuda, _stream

INPUT_SIZE, FEAT_DIM = 299, 2048


def conv_table(in_channels):
    """[(name, cin, cout, kh, kw, stride, pad_h, pad_w)] of the 94 convolutions, graph order, straight from the library"""
    out = []
    buf = C.create_string_buffer(128)
    v = [C.c_int() for _ in range(7)]
    for i in range(lib.ssnb_iv3_num_convs()):
        check(lib.ssnb_iv3_conv_info(i, in_channels, buf, 128, *[C.byref(x) for x in v]), None, "iv3_conv_info")
        out.append((buf.value.decode(),) + tuple(x.value for x in v))
    return out


class InceptionV3Engine(PlannedEngine):
    """One planned InceptionV3 forward for a fixed frame count (ssnb_iv3_create .. ssnb_iv3_destroy), which also runs any
    smaller frame count on the same workspace.  device=None plans without allocating (the plan needs no GPU)."""
    _set_workspace_fn, _pack_fn, _destroy_fn = "ssnb_iv3_set_workspace", "ssnb_iv3_pack_weights", "ssnb_iv3_destroy"
    _errors_on_handle = False

    def __init__(self, in_channels, frames, precision=_lib.EXACT_FP32, device=None):
        self.frames, self.in_channels, self.precision = frames, in_channels, precision
        cfg = _lib.IV3Config(in_channels, frames, precision, 0)
        self.h = C.c_void_p()
        check(lib.ssnb_iv3_create(C.byref(cfg), C.byref(self.h)), None, "ssnb_iv3_create")
        self.workspace_bytes = lib.ssnb_iv3_workspace_bytes(self.h)
        self.device = None if device is None else torch.device(device)
        self.packed_version = None
        if self.device is not None:
            self._set_workspace()

    def forward(self, x):
        """x [n, C, 299, 299] -> feat [n, 2048]; n < frames runs the first n frames of the plan"""
        _need_cuda(x, "input")
        x = x.contiguous().float()
        n = x.shape[0]
        assert 1 <= n <= self.frames and tuple(x.shape[1:]) == (self.in_channels, INPUT_SIZE, INPUT_SIZE), \
            "engine planned for [<=%d,%d,299,299], got %s" % (self.frames, self.in_channels, tuple(x.shape))
        feat = torch.empty(n, FEAT_DIM, dtype=torch.float32, device=x.device)
        with torch.cuda.device(self.device):
            if n == self.frames:
                check(lib.ssnb_iv3_forward(self.h, C.c_void_p(x.data_ptr()), C.c_void_p(feat.data_ptr()), _stream()), None, "iv3_forward")
            else:
                check(lib.ssnb_iv3_forward_frames(self.h, C.c_void_p(x.data_ptr()), n, C.c_void_p(feat.data_ptr()), _stream()), None,
                      "iv3_forward_frames")
        return feat

    # ---- introspection: the plan and the launch-by-launch tests ----
    def ops(self):
        """[(kind, in_name, out_name, conv index, k, stride, pad)] in schedule order"""
        out = []
        k, i, o = (C.create_string_buffer(64), C.create_string_buffer(128), C.create_string_buffer(128))
        v = [C.c_int() for _ in range(4)]
        for n in range(lib.ssnb_iv3_num_ops(self.h)):
            check(lib.ssnb_iv3_op_info(self.h, n, k, 64, i, 128, o, 128, *[C.byref(x) for x in v]), None, "iv3_op_info")
            out.append((k.value.decode(), i.value.decode(), o.value.decode()) + tuple(x.value for x in v))
        return out

    def value_info(self, name):
        """(C, H, W, buffer name, channel offset in the buffer)"""
        v = [C.c_int() for _ in range(4)]
        buf = C.create_string_buffer(128)
        check(lib.ssnb_iv3_value_info(self.h, name.encode(), C.byref(v[0]), C.byref(v[1]), C.byref(v[2]), buf, 128, C.byref(v[3])),
              None, "iv3_value_info")
        return v[0].value, v[1].value, v[2].value, buf.value.decode(), v[3].value

    def write(self, name, t):
        c, h, w = self.value_info(name)[:3]
        t = t.contiguous().float()
        assert tuple(t.shape) == (self.frames, c, h, w), (name, tuple(t.shape), (self.frames, c, h, w))
        with torch.cuda.device(self.device):
            check(lib.ssnb_iv3_value_write(self.h, name.encode(), C.c_void_p(t.data_ptr()), _stream()), None, "iv3_value_write")

    def read(self, name, planes=False):
        """planes=True (EXACT_TC only): hi + lo of the value's fp16 operand planes instead of the value"""
        c, h, w = self.value_info(name)[:3]
        t = torch.empty(self.frames, c, h, w, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib.ssnb_iv3_value_read(self.h, name.encode(), int(planes), C.c_void_p(t.data_ptr()), _stream()), None, "iv3_value_read")
        return t

    def run_op(self, idx, feat=None):
        with torch.cuda.device(self.device):
            check(lib.ssnb_iv3_run_op(self.h, idx, None if feat is None else C.c_void_p(feat.data_ptr()), _stream()), None, "iv3_run_op")
