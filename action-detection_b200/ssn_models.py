"""Drop-in for the reference's ssn_models.py (SSN :10-395): same constructor, forward signature,
attributes and state_dict keys, so the loops in ssn_train.py:191-253 / ssn_test.py:68-96 run
against it unchanged.  The BNInception backbone, STPP and the heads execute in libssn_b200.so.

base_model='BNInception' with RGB / Flow input is accelerated (the hot path this repo covers), and
base_model='InceptionV3' at test time (forward only); other backbones raise ValueError like an unknown name does in the
reference (:153-154).
"""
import torch
from torch import nn

from ops.ssn_ops import Identity, StructuredTemporalPyramidPooling
from ssn_b200.engine import LinearFunction, heads_loss_fused
from ssn_b200 import _lib
from ssn_b200._lib import lib, check


class _HeadLinear(nn.Linear):
    """nn.Linear (so optimiser policies / state_dict are unchanged) computed by ssnb_linear_*."""

    def forward(self, input):
        return LinearFunction.apply(input, self.weight, self.bias)


class _BNInceptionModel(torch.nn.Module):
    """What SSN and BinaryClassifier share (ssn_models.py:69-174,203-251,318-343 and binary_model.py:55-80,117-145,
    165-215,260-307 of the reference are the same code): the BNInception backbone for RGB or Flow input with its last
    layer replaced by Dropout / Identity, bn_mode handling, optimiser policies and the data-side attributes.  Subclasses
    set modality, new_length and dropout before calling _prepare_base_model."""

    # ---- construction (ssn_models.py:69-154) ------------------------------------------------------
    def _prepare_base_model(self, base_model):
        if base_model not in ('BNInception', 'InceptionV3'):
            raise ValueError('Unknown base model: {} (the H100 hot path implements BNInception and, at test time, '
                             'InceptionV3)'.format(base_model))
        if self.modality == 'RGB':
            in_ch = 3 * self.new_length
        elif self.modality == 'Flow':
            in_ch = 2 * self.new_length
        else:
            raise ValueError('modality {} is outside the accelerated path (RGB, Flow)'.format(self.modality))
        import model_zoo
        net = getattr(model_zoo, base_model)
        if self.modality == 'Flow':
            # like the reference: build the 3-channel network (this is where pretrained RGB weights would be loaded) and swap
            # the first convolution for the mean-expanded 2*new_length-channel kernel (_construct_flow_model, ssn_models.py:318-343)
            self.base_model = self._construct_flow_model(net(in_channels=3))
            assert self.base_model.in_channels() == in_ch
        else:
            self.base_model = net(in_channels=in_ch)
        # BNInception (ssn_models.py:121-132) and InceptionV3 (:133-144) differ in the last layer's name and the input size only
        self.base_model.last_layer_name = 'fc' if base_model == 'BNInception' else 'top_cls_fc'
        self.input_size = 224 if base_model == 'BNInception' else 299
        self.input_mean = [104, 117, 128]
        self.input_std = [1]
        if self.modality == 'Flow':
            self.input_mean = [128]

    def _construct_flow_model(self, base_model):
        """replace the first convolution by one with 2*new_length input channels whose kernels are the mean of the RGB kernels
        over the input-channel axis, bias kept (ssn_models.py:318-343)"""
        name = base_model._conv_names[0]
        conv_layer = getattr(base_model, name)
        params = [x.clone() for x in conv_layer.parameters()]
        kernel_size = params[0].size()
        new_kernel_size = kernel_size[:1] + (2 * self.new_length,) + kernel_size[2:]
        new_kernels = params[0].data.mean(dim=1, keepdim=True).expand(new_kernel_size).contiguous()
        new_conv = nn.Conv2d(2 * self.new_length, conv_layer.out_channels, conv_layer.kernel_size, conv_layer.stride, conv_layer.padding,
                             bias=True if len(params) == 2 else False)
        new_conv.weight.data = new_kernels
        if len(params) == 2:
            new_conv.bias.data = params[1].data
        setattr(base_model, name, new_conv)
        base_model._engines = {}               # engines are planned per input-channel count
        return base_model

    def _replace_last_layer(self):
        """fc -> Dropout(p=dropout), or Identity for dropout 0 (ssn_models.py:71-75); returns the feature dimension"""
        feature_dim = getattr(self.base_model, self.base_model.last_layer_name).in_features
        if self.dropout == 0:
            setattr(self.base_model, self.base_model.last_layer_name, Identity())
        else:
            setattr(self.base_model, self.base_model.last_layer_name, nn.Dropout(p=self.dropout))
        return feature_dim

    # bn_mode -> 1-based index of the first BatchNorm2d that stays in eval mode with frozen affine parameters
    # ('partial': the first one trains, 'full': none frozen), ssn_models.py:95-105
    _FIRST_FROZEN_BN = {'frozen': 1, 'partial': 2, 'full': None}

    def prepare_bn(self):
        if self.bn_mode not in self._FIRST_FROZEN_BN:
            raise ValueError("unknown bn mode")
        self.freeze_count = self._FIRST_FROZEN_BN[self.bn_mode]

    def train(self, mode=True):
        """nn.Module.train, then the BatchNorm2d layers from `freeze_count` on go back to eval mode and stop training
        their affine parameters (ssn_models.py:156-174)"""
        super().train(mode)
        if self.freeze_count is not None:
            bns = [m for m in self.base_model.modules() if isinstance(m, nn.BatchNorm2d)]
            for bn in bns[self.freeze_count - 1:]:
                bn.eval()
                bn.weight.requires_grad = False
                bn.bias.requires_grad = False
        return self

    def set_precision(self, precision, grad_scale=None):
        self.base_model.set_precision(precision, grad_scale)

    # ---- optimiser groups (ssn_models.py:203-251) ---------------------------------------------------
    def get_optim_policies(self):
        first_conv_weight, first_conv_bias, normal_weight, normal_bias, bn = [], [], [], [], []
        conv_cnt = 0
        for m in self.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Conv1d)):
                ps = list(m.parameters())
                conv_cnt += 1
                (first_conv_weight if conv_cnt == 1 else normal_weight).append(ps[0])
                if len(ps) == 2:
                    (first_conv_bias if conv_cnt == 1 else normal_bias).append(ps[1])
            elif isinstance(m, torch.nn.Linear):
                ps = list(m.parameters())
                normal_weight.append(ps[0])
                if len(ps) == 2:
                    normal_bias.append(ps[1])
            elif isinstance(m, torch.nn.BatchNorm1d):
                bn.extend(list(m.parameters()))
            elif isinstance(m, torch.nn.BatchNorm2d):
                pass  # frozen (train())
            elif len(m._modules) == 0:
                if len(list(m.parameters())) > 0:
                    raise ValueError("New atomic module type: {}. Need to give it a learning policy".format(type(m)))
        return [
            {'params': first_conv_weight, 'lr_mult': 1, 'decay_mult': 1, 'name': "first_conv_weight"},
            {'params': first_conv_bias, 'lr_mult': 2, 'decay_mult': 0, 'name': "first_conv_bias"},
            {'params': normal_weight, 'lr_mult': 1, 'decay_mult': 1, 'name': "normal_weight"},
            {'params': normal_bias, 'lr_mult': 2, 'decay_mult': 0, 'name': "normal_bias"},
            {'params': bn, 'lr_mult': 1, 'decay_mult': 0, 'name': "BN scale/shift"},
        ]

    def _require_trainable_backbone(self):
        from model_zoo import InceptionV3
        if isinstance(self.base_model, InceptionV3):
            raise NotImplementedError("fused_step trains the BNInception backbone; InceptionV3 runs at test time only: "
                                      "training InceptionV3 (backward schedule, fused_step) is a follow-up")

    def _frames(self, input):
        sample_len = (3 if self.modality == "RGB" else 2) * self.new_length
        return input.view((-1, sample_len) + input.size()[-2:])

    @staticmethod
    def _accumulate_grad(p, g):
        if p.grad is None:
            p.grad = g
        else:
            p.grad.add_(g)

    def _fused_backbone_backward(self, eng, dft, grad_sync):
        """the tail of fused_step once the head gradients are in .grad: start the head bucket's exchange, then the engine
        backward from dfeat straight into the convolutions' .grad, bucket by bucket when grad_sync is given"""
        if grad_sync is not None:
            grad_sync.begin()
            grad_sync.heads_done()
        cs = self.base_model._convs()
        params = [c.weight for c in cs] + [c.bias for c in cs]
        for p in params:
            if p.requires_grad and p.grad is None:
                p.grad = torch.zeros_like(p)
        # straight into .grad; parameters with requires_grad=False get no gradient (None -> the kernels skip them)
        buckets = grad_sync.engine_buckets(eng)[0] if grad_sync is not None else None
        eng.backward(dft, [c.weight.grad if c.weight.requires_grad else None for c in cs],
                     [c.bias.grad if c.bias.requires_grad else None for c in cs], accumulate=True, buckets=buckets,
                     on_bucket=(lambda i: grad_sync.bucket_done(eng, i)) if grad_sync is not None else None)

    # ---- data-side attributes the drivers read (ssn_train.py:60-65, ssn_test.py:109-142) -------------
    @property
    def crop_size(self):
        return self.input_size

    @property
    def scale_size(self):
        return self.input_size * 256 // 224

    def get_augmentation(self):
        # PIL group transforms are CPU data-pipeline code outside this hot path (SURVEY.md §2.1);
        # if the reference's transforms.py is importable, use it.
        try:
            import torchvision
            from transforms import GroupMultiScaleCrop, GroupRandomHorizontalFlip
        except ImportError as e:
            raise NotImplementedError("get_augmentation needs the reference's transforms.py on sys.path "
                                      "(data pipeline is out of scope for the H100 hot path)") from e
        scales = [1, .875, .75, .66] if self.modality == 'RGB' else [1, .875, .75]
        return torchvision.transforms.Compose([GroupMultiScaleCrop(self.input_size, scales),
                                               GroupRandomHorizontalFlip(is_flow=(self.modality == 'Flow'))])

    def frame_transforms(self):
        """The data-side transforms of the drivers on the GPU (ops/frame_transforms.py), with this model's scales, input_mean,
        input_std and modality filled in.  Each transform takes uint8 frames (GroupToUint8 on the dataset side) and returns
        the CUDA fp32 [frames, C, 224, 224] input that get_augmentation / GroupOverSample / GroupScale + GroupCenterCrop
        followed by Stack, ToTorchFormatTensor(div=False) and GroupNormalize produce:
          sample_train_params(sizes)     the crop and flip draws of get_augmentation(), one per group
          train(frames, params)          get_augmentation() (training)
          oversample(frames)             GroupOverSample(crop_size, scale_size) (10-crop test)
          center_crop(frames)            GroupScale(scale_size) + GroupCenterCrop(crop_size) (1-crop test, validation)
          to_uint8                       the dataset-side transform"""
        import functools
        import types
        from ops import frame_transforms as T
        is_flow = self.modality == 'Flow'
        scales = [1, .875, .75] if is_flow else [1, .875, .75, .66]
        fc = (2 if is_flow else 3) * self.new_length
        common = dict(mean=self.input_mean, std=self.input_std, frame_channels=fc)
        return types.SimpleNamespace(
            sample_train_params=functools.partial(T.sample_train_params, scales=scales, input_size=self.input_size),
            train=functools.partial(T.train_frames, input_size=self.input_size, is_flow=is_flow, **common),
            oversample=functools.partial(T.oversample_frames, crop_size=self.crop_size, scale_size=self.scale_size, **common),
            center_crop=functools.partial(T.center_crop_frames, crop_size=self.crop_size, scale_size=self.scale_size, **common),
            to_uint8=T.GroupToUint8())


class SSN(_BNInceptionModel):
    def __init__(self, num_class,
                 starting_segment, course_segment, ending_segment, modality,
                 base_model='resnet101', new_length=None,
                 dropout=0.8,
                 crop_num=1, no_regression=False, test_mode=False,
                 stpp_cfg=(1, (1, 2), 1), bn_mode='frozen', verbose=False):
        super(SSN, self).__init__()
        self.modality = modality
        self.num_segments = starting_segment + course_segment + ending_segment
        self.starting_segment = starting_segment
        self.course_segment = course_segment
        self.ending_segment = ending_segment
        self.reshape = True
        self.dropout = dropout
        self.crop_num = crop_num
        self.with_regression = not no_regression
        self.test_mode = test_mode
        self.bn_mode = bn_mode
        self.num_class = num_class
        if new_length is None:
            self.new_length = 1 if modality == "RGB" else 5
        else:
            self.new_length = new_length
        if verbose:
            print("Initializing SSN (H100) base model {} modality {} segments {}+{}+{} dropout {} stpp {} bn {}".format(
                base_model, modality, starting_segment, course_segment, ending_segment, dropout, stpp_cfg, bn_mode))
        self._prepare_base_model(base_model)
        self._prepare_ssn(num_class, stpp_cfg)
        self.prepare_bn()

    def _prepare_ssn(self, num_class, stpp_cfg):
        feature_dim = self._replace_last_layer()
        self.stpp = StructuredTemporalPyramidPooling(feature_dim, True, configs=stpp_cfg)
        self.activity_fc = _HeadLinear(self.stpp.activity_feat_dim(), num_class + 1)
        self.completeness_fc = _HeadLinear(self.stpp.completeness_feat_dim(), num_class)
        nn.init.normal_(self.activity_fc.weight.data, 0, 0.001)
        nn.init.constant_(self.activity_fc.bias.data, 0)
        nn.init.normal_(self.completeness_fc.weight.data, 0, 0.001)
        nn.init.constant_(self.completeness_fc.bias.data, 0)
        self.test_fc = None
        if self.with_regression:
            self.regressor_fc = _HeadLinear(self.stpp.completeness_feat_dim(), 2 * num_class)
            nn.init.normal_(self.regressor_fc.weight.data, 0, 0.001)
            nn.init.constant_(self.regressor_fc.bias.data, 0)
        else:
            self.regressor_fc = None
        return feature_dim

    # ---- test-time FC folding (ssn_models.py:176-201) ----------------------------------------------
    def prepare_test_fc(self):
        M = self.stpp.feat_multiplier
        D = self.activity_fc.in_features
        self.test_fc = _HeadLinear(D, self.activity_fc.out_features + self.completeness_fc.out_features * M
                                   + (self.regressor_fc.out_features * M if self.with_regression else 0))

        def reorg(fc):
            o = fc.out_features
            w = fc.weight.data.view(o, M, D).transpose(0, 1).contiguous().view(-1, D)
            b = fc.bias.data.view(1, -1).expand(M, o).contiguous().view(-1) / M
            return w, b

        cw, cb = reorg(self.completeness_fc)
        weight = torch.cat((self.activity_fc.weight.data, cw))
        bias = torch.cat((self.activity_fc.bias.data, cb))
        if self.with_regression:
            rw, rb = reorg(self.regressor_fc)
            weight = torch.cat((weight, rw))
            bias = torch.cat((bias, rb))
        self.test_fc.weight.data = weight
        self.test_fc.bias.data = bias

    # ---- forward (ssn_models.py:253-300) -------------------------------------------------------------
    def forward(self, input, aug_scaling, target, reg_target, prop_type):
        if not self.test_mode:
            return self.train_forward(input, aug_scaling, target, reg_target, prop_type)
        return self.test_forward(input)

    def _seg_split(self):
        return [self.starting_segment, self.starting_segment + self.course_segment, self.num_segments]

    def train_forward(self, input, aug_scaling, target, reg_target, prop_type):
        # The row selections depend on prop_type only.  nonzero() synchronises host and device (its result size is
        # data dependent), so it runs BEFORE the backbone is enqueued: the host then stays ahead of the GPU for the
        # whole step instead of stalling behind the backbone forward and leaving the GPU idle while it catches up.
        type_data = prop_type.view(-1).data
        # .view(-1) instead of the reference's .squeeze(): identical for >1 selected row and keeps
        # the row dimension when exactly one row matches (SURVEY.md §7.2-6).
        act_indexer = ((type_data == 0) | (type_data == 2)).nonzero().view(-1)
        comp_indexer = ((type_data == 0) | (type_data == 1)).nonzero().view(-1)
        reg_indexer = (type_data == 0).nonzero().view(-1) if self.with_regression else None
        base_out = self.base_model(self._frames(input))
        activity_ft, completeness_ft = self.stpp(base_out, aug_scaling, self._seg_split())
        raw_act_fc = self.activity_fc(activity_ft)
        raw_comp_fc = self.completeness_fc(completeness_ft)
        target = target.view(-1)
        if self.with_regression:
            reg_target = reg_target.view(-1, 2)
            raw_regress_fc = self.regressor_fc(completeness_ft).view(-1, self.completeness_fc.out_features, 2)
            return raw_act_fc[act_indexer, :], target[act_indexer], \
                raw_comp_fc[comp_indexer, :], target[comp_indexer], \
                raw_regress_fc[reg_indexer, :, :], target[reg_indexer], reg_target[reg_indexer, :]
        return raw_act_fc[act_indexer, :], target[act_indexer], raw_comp_fc[comp_indexer, :], target[comp_indexer]

    def test_forward(self, input):
        base_out = self.base_model(self._frames(input))
        return self.test_fc(base_out), base_out

    def test_scores(self, input, num_crop=10):
        """One chunk of a test video, crop-major [num_crop * ticks, C, H, W] -> per-tick scores [ticks, D]: what the reference's
        loop body computes as `rst, _ = net(frames, None, None, None, None); rst.view(num_crop, -1, D).mean(dim=0)`
        (ssn_test.py:80-84), with the crop mean folded into the folded FC (one kernel, 1/num_crop of the FC work).  Unlike
        the reference's data loader (gen_batchsize = 4 ticks -> 40-image calls, ssn_dataset.py:393) the chunk size is the
        caller's: >= 256 frames per call keep the tensor cores busy."""
        if self.test_fc is None:
            raise RuntimeError("call prepare_test_fc() first (ssn_test.py:62)")
        frames = self._frames(input)
        F_ = frames.shape[0]
        assert F_ % num_crop == 0, "frame count must be a multiple of the crop count"
        nt = F_ // num_crop
        with torch.no_grad():
            base_out = self.base_model(frames).contiguous()          # [F, 1024 | 2048]: fc is Identity / eval-mode Dropout at test time
        out = torch.empty(nt, self.test_fc.out_features, dtype=torch.float32, device=base_out.device)
        from ssn_b200.engine import _stream
        with torch.cuda.device(base_out.device):
            check(lib.ssnb_test_fc_cropmean(base_out.data_ptr(), self.test_fc.weight.data_ptr(), self.test_fc.bias.data_ptr(), num_crop, nt,
                                            base_out.shape[1], self.test_fc.out_features, out.data_ptr(), _stream()), None, "test_fc_cropmean")
        return out

    # ---- fused training step: backbone fwd -> pool+STPP -> heads+loss(+grads) -> backbone bwd ---------
    def fused_step(self, input, aug_scaling, target, reg_target, prop_type, fg_per_video=1, comp_group=7,
                   props_per_video=8, ohem_ratio=0.17, comp_w=0.1, reg_w=0.1, global_videos=None, loss_scale=1.0, grad_sync=None):
        """Same arithmetic as train_forward + the three criteria + loss.backward() of
        ssn_train.py:207-236, issued as ~4 library calls.  Accumulates into .grad like autograd and
        returns losses[4] = (act, comp, reg, total) as a device tensor.  grad_sync (ssn_b200.dp.GradSync): exchange the
        gradients bucket by bucket while the backward of the lower layers is still running."""
        import ctypes as C
        from ssn_b200.engine import _stream
        self._require_trainable_backbone()
        assert self.with_regression, "fused_step implements the regression configuration"
        if not input.is_cuda:
            raise RuntimeError("SSN(H100).fused_step needs CUDA tensors (libssn_b200 has no CPU path)")
        if self.base_model.bn1_training():
            raise NotImplementedError("fused_step implements bn_mode='frozen'; with bn_mode='partial' use the module path "
                                      "(model(...), criteria, loss.backward()), which runs the first BatchNorm2d in training mode")
        frames = self._frames(input)
        bm = self.base_model
        eng = bm.engine_for(frames.shape[0], True, frames.device)
        x = frames.contiguous().float()
        dev = x.device
        F_ = x.shape[0]
        n = F_ // self.num_segments
        feat = torch.empty(F_, 1024, dtype=torch.float32, device=dev)
        mask = None
        if self.dropout != 0 and self.training:
            keep = 1.0 - self.dropout
            mask = torch.bernoulli(torch.full((F_, 1024), keep, device=dev)) / keep
        with torch.cuda.device(dev):
            check(lib.ssnb_backbone_fwd(eng.h, x.data_ptr(), feat.data_ptr(), _stream()), eng.h, "backbone_fwd")
            lo, hi, nm, col = self.stpp.part_table(self._seg_split())
            D = 1024
            course = torch.empty(n, D, dtype=torch.float32, device=dev)
            stpp = torch.empty(n, len(lo) * D, dtype=torch.float32, device=dev)
            sc = aug_scaling.contiguous().float().view(-1, 2)
            check(lib.ssnb_gpool_stpp_fwd(eng.h, None if mask is None else mask.data_ptr(), sc.data_ptr(),
                                          self.num_segments, len(lo), _lib.int_array(lo), _lib.int_array(hi),
                                          _lib.int_array(nm), _lib.int_array(col), self.starting_segment,
                                          self.starting_segment + self.course_segment, feat.data_ptr(),
                                          course.data_ptr(), stpp.data_ptr(), _stream()), eng.h, "gpool_stpp_fwd")
        out = heads_loss_fused(course, stpp, self.activity_fc, self.completeness_fc, self.regressor_fc, prop_type,
                               target, reg_target, self.num_class, self.stpp.feat_multiplier, fg_per_video, comp_group,
                               props_per_video, ohem_ratio, comp_w, reg_w, global_videos, loss_scale)
        dft = torch.empty(F_, D, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib.ssnb_stpp_bwd(out["d_course"].data_ptr(), out["d_stpp"].data_ptr(), sc.data_ptr(), n,
                                    self.num_segments, D, len(lo), _lib.int_array(lo), _lib.int_array(hi),
                                    _lib.int_array(nm), _lib.int_array(col), self.starting_segment,
                                    self.starting_segment + self.course_segment, dft.data_ptr(), _stream()), None, "stpp_bwd")
        if mask is not None:
            dft = dft * mask
        for fc, k in ((self.activity_fc, "act"), (self.completeness_fc, "comp"), (self.regressor_fc, "reg")):
            if fc.weight.requires_grad:
                self._accumulate_grad(fc.weight, out["d_%s_w" % k])
            if fc.bias.requires_grad:
                self._accumulate_grad(fc.bias, out["d_%s_b" % k])
        self._fused_backbone_backward(eng, dft, grad_sync)
        self.last_fused = dict(out, feat=feat, course=course, stpp=stpp, mask=mask)
        return out["losses"]
