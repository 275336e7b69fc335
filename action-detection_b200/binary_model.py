"""Drop-in for the reference's binary_model.py (BinaryClassifier :7-307, the TAG actionness classifier): same constructor,
forward(inputdata, target) semantics, attributes and state_dict keys, so binary_train.py:114-183 and binary_test.py:63-94
run against it unchanged.  The BNInception backbone, the segment mean and classifier_fc execute in libssn_b200.so; the
loss stays the caller's torch.nn.CrossEntropyLoss (binary_train.py:135), or BinaryClassifier.fused_step does the whole
training step in the library.

base_model='BNInception' with RGB / Flow input is accelerated, and base_model='InceptionV3' at test time (scoring only);
other backbones and modalities raise ValueError like
the SSN drop-in does.  Construction, Flow conv1 expansion, bn_mode handling and the optimiser policies are SSN's
(ssn_models._BNInceptionModel): the reference's two files repeat the same code.

Deliberate differences from the reference:
  * binary_model.py:214 sets `m.weight_requires_grad` (a typo), so the reference leaves every frozen BatchNorm2d weight
    with requires_grad=True: autograd fills its .grad, but no optimiser group holds it (:289-291).  Here frozen BatchNorm2d
    weights and biases both stop requiring gradients, as in SSN.train.  Training is identical.
  * train() returns self (nn.Module.train's contract); the reference returns None.
  * modality 'RGBDiff' raises ValueError.  It cannot run in the reference on Python 3 (filter(...)[0] at :88, conv.layer at
    :104).
"""
import torch

from ssn_models import _BNInceptionModel, _HeadLinear
from ssn_b200 import _lib
from ssn_b200._lib import lib, check
from ssn_b200.engine import STPPFunction, _stream


class BinaryClassifier(_BNInceptionModel):
    def __init__(self, num_class, course_segment, modality,
                 base_model='resnet101', new_length=None,
                 dropout=0.8,
                 crop_num=1, test_mode=False, bn_mode='frozen', verbose=False):
        super(BinaryClassifier, self).__init__()
        self.modality = modality
        self.num_segments = course_segment
        self.course_segment = course_segment
        self.reshape = True
        self.dropout = dropout
        self.crop_num = crop_num
        self.test_mode = test_mode
        self.bn_mode = bn_mode
        if new_length is None:
            self.new_length = 1 if modality == "RGB" else 5
        else:
            self.new_length = new_length
        if verbose:
            print("Initializing BinaryClassifier (H100) base model {} modality {} course_segment {} new_length {} dropout {} bn {}".format(
                base_model, modality, course_segment, self.new_length, dropout, bn_mode))
        self._prepare_base_model(base_model)
        self._prepare_binary_classifier(num_class)
        self.prepare_bn()

    # ---- construction (binary_model.py:117-132) ----------------------------------------------------
    def _prepare_binary_classifier(self, num_class):
        feature_dim = self._replace_last_layer()
        self.classifier_fc = _HeadLinear(feature_dim, num_class)
        torch.nn.init.normal_(self.classifier_fc.weight.data, 0, 0.001)
        torch.nn.init.constant_(self.classifier_fc.bias.data, 0)
        self.test_fc = None
        self.feature_dim = feature_dim
        return feature_dim

    # ---- test-time FC (binary_model.py:245-254): test_fc shares classifier_fc's tensors -------------
    def prepare_test_fc(self):
        self.test_fc = _HeadLinear(self.classifier_fc.in_features, self.classifier_fc.out_features)
        self.test_fc.weight.data = self.classifier_fc.weight.data
        self.test_fc.bias.data = self.classifier_fc.bias.data

    # ---- forward (binary_model.py:218-240) -----------------------------------------------------------
    def forward(self, inputdata, target):
        if not self.test_mode:
            return self.train_forward(inputdata, target)
        return self.test_forward(inputdata)

    def train_forward(self, inputdata, target):
        """base_out.view(-1, course_segment, 1024).mean(1) -> classifier_fc; returns (raw scores [n, K], target.view(-1))"""
        base_out = self.base_model(self._frames(inputdata))
        # the STPP bridge with an empty part table: the course mean over all course_segment snippets, nothing else
        course_ft, _ = STPPFunction.apply(base_out, None, ([], [], [], []), self.course_segment, (0, self.course_segment))
        return self.classifier_fc(course_ft), target.view(-1)

    def test_forward(self, input):
        base_out = self.base_model(self._frames(input))
        return self.test_fc(base_out), base_out

    # ---- fused training step: backbone fwd -> pool + mask + segment mean -> classifier + CE (+grads) -> backbone bwd ------
    def fused_step(self, input, target, loss_scale=1.0, grad_sync=None, meters=None):
        """Same arithmetic as train_forward + torch.nn.CrossEntropyLoss() + loss.backward() (binary_train.py:153-169) in
        five library calls.  Accumulates into .grad like autograd and returns the mean loss as a device tensor [1].  Every
        gradient is multiplied by loss_scale (1/world for data parallel with equal rows per rank).  grad_sync
        (ssn_b200.dp.GradSync): exchange the gradients bucket by bucket while the backward of the lower layers is running.
        meters (ssn_b200.meters.StepMeters('binary')): add this step's loss and accuracies to it, on the device.
        Keeps feat, course, logits and the dropout mask (None without dropout) of the step in self.last_fused."""
        self._require_trainable_backbone()
        if not input.is_cuda:
            raise RuntimeError("BinaryClassifier(H100).fused_step needs CUDA tensors (libssn_b200 has no CPU path)")
        if self.base_model.bn1_training():
            raise NotImplementedError("fused_step implements bn_mode='frozen'; with bn_mode='partial' use the module path "
                                      "(model(input, target), CrossEntropyLoss, loss.backward())")
        frames = self._frames(input)
        eng = self.base_model.engine_for(frames.shape[0], True, frames.device)
        x = frames.contiguous().float()
        mask = None
        if self.dropout != 0 and self.training:
            keep = 1.0 - self.dropout
            mask = torch.bernoulli(torch.full((x.shape[0], self.feature_dim), keep, device=x.device)) / keep
        r = self._fused_forward(eng, x, target, mask, loss_scale)
        if meters is not None:
            meters.update_binary(r["loss"], r["logits"], r["target"], input.size(0))
        n, S = r["course"].shape[0], self.course_segment
        w, b = self.classifier_fc.weight, self.classifier_fc.bias
        dft = torch.empty(x.shape[0], self.feature_dim, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.ssnb_stpp_bwd(r["d_course"].data_ptr(), None, None, n, S, self.feature_dim, 0, None, None, None, None, 0, S,
                                    dft.data_ptr(), _stream()), None, "stpp_bwd")
        if mask is not None:
            dft = dft * mask
        if w.requires_grad:
            self._accumulate_grad(w, r["dw"])
        if b.requires_grad:
            self._accumulate_grad(b, r["db"])
        self._fused_backbone_backward(eng, dft, grad_sync)
        self.last_fused = dict(feat=r["feat"], course=r["course"], logits=r["logits"], mask=mask)
        return r["loss"]

    def _fused_forward(self, eng, x, target, mask, loss_scale):
        """backbone forward -> global pool (+ dropout mask) + segment mean -> classifier + cross-entropy (+ its gradients):
        the forward half that fused_step and fused_eval share"""
        dev = x.device
        F_, S, D = x.shape[0], self.course_segment, self.feature_dim
        if F_ % S:
            raise ValueError("%d frames are not a whole number of %d-segment proposals" % (F_, S))
        n, K = F_ // S, self.classifier_fc.out_features
        tg = target.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()
        if tg.numel() != n:
            raise ValueError("%d targets for %d proposals" % (tg.numel(), n))
        f32 = dict(dtype=torch.float32, device=dev)
        feat, course = torch.empty(F_, D, **f32), torch.empty(n, D, **f32)
        w, b = self.classifier_fc.weight, self.classifier_fc.bias
        logits, loss = torch.empty(n, K, **f32), torch.empty(1, **f32)
        d_course, dw, db = torch.empty(n, D, **f32), torch.empty_like(w), torch.empty_like(b)
        ws = torch.empty(lib.ssnb_classifier_ce_workspace_bytes(n, K), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(lib.ssnb_backbone_fwd(eng.h, x.data_ptr(), feat.data_ptr(), _stream()), eng.h, "backbone_fwd")
            # zero STPP parts: global pool (+ mask) into feat and the course mean over the S snippets of each proposal
            check(lib.ssnb_gpool_stpp_fwd(eng.h, None if mask is None else mask.data_ptr(), None, S, 0, None, None, None, None,
                                          0, S, feat.data_ptr(), course.data_ptr(), None, _stream()), eng.h, "gpool_stpp_fwd")
            check(lib.ssnb_classifier_ce_fwd_bwd(course.data_ptr(), w.data_ptr(), b.data_ptr(), tg.data_ptr(), n, D, K,
                                                 float(loss_scale), logits.data_ptr(), loss.data_ptr(), d_course.data_ptr(),
                                                 dw.data_ptr(), db.data_ptr(), ws.data_ptr(), _stream()), None, "classifier_ce_fwd_bwd")
        return dict(feat=feat, course=course, logits=logits, loss=loss, target=tg, d_course=d_course, dw=dw, db=db)

    def fused_eval(self, input, target, meters=None):
        """The body of validate() (binary_train.py:219-243): the forward of a forward-only engine, global pool + segment mean,
        classifier_fc and CrossEntropyLoss, without a backward.  The model must be in eval() (binary_train.py:225): no
        dropout, no running-statistic update; no .grad changes.  Returns the mean loss [1] on the device, what fused_step's
        forward half computes from the same features; meters (StepMeters('binary')) gets the loss and accuracies.  Keeps
        feat, course and logits in self.last_eval."""
        self._require_trainable_backbone()
        if self.training:
            raise RuntimeError("fused_eval runs validate()'s forward: call model.eval() first (binary_train.py:225)")
        if not input.is_cuda:
            raise RuntimeError("BinaryClassifier(H100).fused_eval needs CUDA tensors (libssn_b200 has no CPU path)")
        frames = self._frames(input)
        eng = self.base_model.engine_for(frames.shape[0], False, frames.device)
        if eng.frames != frames.shape[0]:
            raise ValueError("fused_eval pools the engine's whole plan: %d frames with %d reserved by reserve_frames(); "
                             "call reserve_frames(None) or pass the reserved count" % (frames.shape[0], eng.frames))
        r = self._fused_forward(eng, frames.contiguous().float(), target, None, 1.0)
        if meters is not None:
            meters.update_binary(r["loss"], r["logits"], r["target"], input.size(0))
        self.last_eval = dict(feat=r["feat"], course=r["course"], logits=r["logits"])
        return r["loss"]
