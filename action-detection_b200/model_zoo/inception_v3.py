"""InceptionV3 with the reference's module surface (model_zoo/bninception/pytorch_load.py:64-67, graph
inceptionv3.yaml), executed at test time by libssn_b200's InceptionV3 engine.

The children are the reference's, in its order: per convolution `<x>_Conv2D` (nn.Conv2d with bias), `<x>_batchnorm`
(nn.BatchNorm2d) and `<x>` (nn.ReLU), the pools under their yaml ids, `top_cls_pool` and `top_cls_fc` (2048 -> 1000), so
state_dict keys and shapes match a reference checkpoint.  Their own forward() is never called.
forward(x [N, C, 299, 299]) -> top_cls_fc(8x8 average pool features [N, 2048]).

Forward only, with every BatchNorm2d frozen (eval mode), in EXACT_FP32, FAST_FP16 or EXACT_TC (set_precision).  Gradients
and training-mode BatchNorm raise NotImplementedError before any launch: training InceptionV3 is a follow-up.
"""
import torch
from torch import nn

from ssn_b200 import _lib
from ssn_b200.inception_v3 import FEAT_DIM, InceptionV3Engine, conv_table

from .backbone import EngineBackbone

_GPOOL_ID = "top_cls_pool"
FOLLOW_UP = "training InceptionV3 (backward schedule, fused_step) is a follow-up"


class InceptionV3(EngineBackbone):
    def __init__(self, model_path=None, num_classes=101, weight_url=None, in_channels=3):
        super(InceptionV3, self).__init__()
        # model_path / weight_url are accepted for signature compatibility; the graph is built into the library and there
        # is no network access for pretrained weights.
        convs = {c[0]: c for c in conv_table(in_channels)}
        plan = InceptionV3Engine(in_channels, 1)          # plans on the host only: the op order and pool geometry
        self._conv_names, self._bn_names = [], []
        for (kind, _in, out, conv, k, stride, pad) in plan.ops():
            if kind == "conv":
                name, cin, cout, kh, kw, st, ph, pw = convs[out]
                setattr(self, name + "_Conv2D", nn.Conv2d(cin, cout, (kh, kw), st, (ph, pw), bias=True))
                setattr(self, name + "_batchnorm", nn.BatchNorm2d(cout, momentum=0.1))
                setattr(self, name, nn.ReLU(inplace=True))
                self._conv_names.append(name + "_Conv2D")
                self._bn_names.append(name + "_batchnorm")
            elif kind == "maxpool":
                setattr(self, out, nn.MaxPool2d(k, stride, pad, ceil_mode=True))
            elif kind == "avgpool":
                setattr(self, out, nn.AvgPool2d(k, stride, pad, ceil_mode=True))
            else:
                setattr(self, _GPOOL_ID, nn.AvgPool2d(k, 1, 0, ceil_mode=True))
        self.top_cls_fc = nn.Linear(FEAT_DIM, 1000)
        self.last_layer_name = "top_cls_fc"
        self.precision = _lib.EXACT_FP32
        self._engines = {}

    def set_precision(self, precision, grad_scale=None):
        """ssn_b200.EXACT_FP32 (fp32 SIMT), ssn_b200.FAST_FP16 (wgmma, fp16 operands) or ssn_b200.EXACT_TC (wgmma,
        error-compensated split fp16 operands: fp32-grade results).  grad_scale is accepted for BNInception's signature and
        ignored: there is no backward."""
        if precision not in (_lib.EXACT_FP32, _lib.FAST_FP16, _lib.EXACT_TC):
            raise ValueError("unknown precision %r" % (precision,))
        self.precision = precision
        self._engines = {}

    def bn1_training(self):
        """False: every BatchNorm2d is frozen.  Raises for a training-mode BatchNorm2d (bn_mode 'partial' / 'full' in train())."""
        if any(b.training for b in self._bns()):
            raise NotImplementedError("InceptionV3 runs with frozen BatchNorm2d layers (eval mode); " + FOLLOW_UP)
        return False

    @staticmethod
    def _forward_only_key(key):
        return True

    def engine_for(self, frames, device):
        """the engine a call of `frames` frames runs on: planned for `frames`, or for the reserve_frames() count"""
        frames = self._planned_frames(frames, True)
        key = (frames, self.precision, self.in_channels(), str(device))
        return self._packed_engine(key, lambda: InceptionV3Engine(self.in_channels(), frames, self.precision, device))

    def forward(self, input):
        if not input.is_cuda:
            raise RuntimeError("InceptionV3(H100) runs on CUDA only: move the model and input to the GPU (libssn_b200 has no CPU path)")
        self.bn1_training()
        cs = self._convs()
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for c in cs for p in c.parameters())):
            raise NotImplementedError("InceptionV3 runs forward only: call it under torch.no_grad() (or with requires_grad=False "
                                      "parameters); " + FOLLOW_UP)
        feat = self.engine_for(input.shape[0], input.device).forward(input)
        return getattr(self, self.last_layer_name)(feat)
