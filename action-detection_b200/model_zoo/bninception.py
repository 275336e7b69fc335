"""BNInception with the reference's module surface (model_zoo/bninception/pytorch_load.py:8-61),
executed by libssn_b200's engine instead of an op-by-op PyTorch interpreter.

The nn.Conv2d / nn.BatchNorm2d children exist as parameter holders only: they give the module the
reference's state_dict keys (`<yaml id>.weight|bias`, `<id>_bn.weight|bias|running_mean|
running_var`, `fc.*`) and make SSN.get_optim_policies (ssn_models.py:203-251) work unchanged; their
own forward() is never called.  forward(x[N,C,224,224]) -> fc(global_pool features [N,1024]).
"""
import torch
from torch import nn

from ssn_b200 import _lib
from ssn_b200.engine import BackboneEngine, BackboneFunction, conv_table

from .backbone import EngineBackbone


class BNInception(EngineBackbone):
    def __init__(self, model_path=None, num_classes=101, weight_url=None, in_channels=3):
        super(BNInception, self).__init__()
        # model_path / weight_url are accepted for signature compatibility; the graph is built into
        # the library and there is no network access for pretrained weights.
        self._conv_names, self._bn_names = [], []
        for (name, cin, cout, k, stride, pad) in conv_table(in_channels):
            setattr(self, name, nn.Conv2d(cin, cout, k, stride, pad, bias=True))
            setattr(self, name + "_bn", nn.BatchNorm2d(cout, momentum=0.1))
            self._conv_names.append(name)
            self._bn_names.append(name + "_bn")
        self.fc = nn.Linear(1024, 1000)
        self.last_layer_name = "fc"
        self.precision = _lib.EXACT_FP32
        self.grad_scale = 1.0
        self._engines = {}

    # ---- engine management --------------------------------------------------------------------
    def set_precision(self, precision, grad_scale=None):
        """precision: ssn_b200.EXACT_FP32 (fp32 SIMT), ssn_b200.FAST_FP16 (wgmma, fp16 operands) or
        ssn_b200.EXACT_TC (wgmma, error-compensated split fp16 operands: fp32-grade results)."""
        if precision == _lib.FAST_FP16 and grad_scale is None and self.grad_scale == 1.0:
            raise ValueError("FAST_FP16 stores gradients in fp16: pass an explicit power-of-two grad_scale (e.g. 4096) so small "
                             "gradients do not underflow, and poll engine.grad_overflow() to catch overflow")
        self.precision = precision
        if grad_scale is not None:
            self.grad_scale = float(grad_scale)
        self._engines = {}

    def grad_overflow(self, clear=True):
        """True when a gradient left the fp16 range under grad_scale in any engine since the last call (device sync)."""
        return any([e.grad_overflow(clear) for e in self._engines.values()])

    def bn1_training(self):
        """bn_mode='partial' (ssn_models.py:95-105): the first BatchNorm2d stays in training mode, every other one is frozen.
        Returns True for that pattern, False when all are frozen, raises for anything else ('full')."""
        bns = self._bns()
        if any(b.training for b in bns[1:]):
            raise NotImplementedError("only bn_mode='frozen' and 'partial' are accelerated: BatchNorm2d layers after the first must be in "
                                      "eval mode ('full' is listed as a next step in DESIGN.md)")
        return bool(bns[0].training)

    @staticmethod
    def _forward_only_key(key):
        return not key[1] and not key[5]

    def engine_for(self, frames, training, device, bn1_train=False):
        """the engine a call of `frames` frames runs on: planned for `frames`, or for the reserve_frames() count when it is a
        forward-only (training=False, bn1_train=False) call"""
        if bn1_train and self.precision == _lib.FAST_FP16:
            raise NotImplementedError("bn_mode='partial' runs in EXACT_FP32 / EXACT_TC precision (fp32 activations), not FAST_FP16")
        frames = self._planned_frames(frames, not training and not bn1_train)
        key = (frames, bool(training), self.precision, self.in_channels(), str(device), bool(bn1_train))
        return self._packed_engine(key, lambda: BackboneEngine(self.in_channels(), frames, self.precision, training, self.grad_scale,
                                                               device, bn1_train=bn1_train))

    def forward(self, input):
        if not input.is_cuda:
            raise RuntimeError("BNInception(H100) runs on CUDA only: move the model and input to the GPU "
                               "(libssn_b200 has no CPU path)")
        bn1_train = self.bn1_training()
        cs = self._convs()
        params = [c.weight for c in cs] + [c.bias for c in cs]
        bn1 = self._bns()[0]
        if bn1_train:
            params += [bn1.weight, bn1.bias]
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        eng = self.engine_for(input.shape[0], need_grad, input.device, bn1_train)
        if bn1_train:
            eng.set_bn1(bn1)                         # batch statistics + running-stat update happen inside the forward
            if bn1.num_batches_tracked is not None:
                bn1.num_batches_tracked.add_(1)
        if need_grad:
            feat = BackboneFunction.apply(input, eng, len(cs), bn1 if bn1_train else None, *params)
        else:
            feat = eng.forward(input)
        return self.fc(feat)
