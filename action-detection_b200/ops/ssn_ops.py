"""Drop-in for the reference's ops/ssn_ops.py: same class names, constructor arguments, call
conventions and error behaviour; the arithmetic runs in libssn_b200.so (CUDA, sm_90a).

Reference: ops/ssn_ops.py — Identity :8-10, parse_stage_config :13-19,
StructuredTemporalPyramidPooling :22-79, STPPReorgainzed :82-170, OHEMHingeLoss :173-213,
CompletenessLoss :216-239, ClassWiseRegressionLoss :242-258.
"""
import ctypes as C

import torch

from ssn_b200 import _lib
from ssn_b200._lib import lib, check
from ssn_b200.engine import STPPFunction, parse_stage_config, stpp_part_table, _stream, _need_cuda


class Identity(torch.nn.Module):
    def forward(self, input):
        return input


class StructuredTemporalPyramidPooling(torch.nn.Module):
    """STPP for training: forward(ft [n*n_seg, D], scaling [n,2], seg_split [x1,x2,n_seg])
    -> (course_ft, stpp_ft) with standalong_classifier, else (stpp_ft, stpp_ft)."""

    def __init__(self, feat_dim, standalong_classifier=False, configs=(1, (1, 2), 1)):
        super(StructuredTemporalPyramidPooling, self).__init__()
        self.sc = standalong_classifier
        self.feat_dim = feat_dim
        # (starting, course, ending) stage -> (pyramid part counts, number of pooled vectors), ops/ssn_ops.py:30-36
        stages = [parse_stage_config(c) for c in configs[:3]]
        self.parts = tuple(parts for parts, _ in stages)
        self.norm_num = tuple(mult for _, mult in stages)
        self.feat_multiplier = sum(self.norm_num)

    def part_table(self, seg_split):
        return stpp_part_table(self.parts, self.norm_num, seg_split)

    def forward(self, ft, scaling, seg_split):
        x1, x2, n_seg = seg_split
        course_ft, stpp_ft = STPPFunction.apply(ft, scaling, self.part_table(seg_split), n_seg, (x1, x2))
        if not self.sc:
            return stpp_ft, stpp_ft
        return course_ft, stpp_ft

    def activity_feat_dim(self):
        return self.feat_dim if self.sc else self.feat_dim * self.feat_multiplier

    def completeness_feat_dim(self):
        return self.feat_dim * self.feat_multiplier


class STPPReorgainzed:
    """Re-organised testing (pool the per-frame scores instead of the features)."""

    def __init__(self, feat_dim, act_score_len, comp_score_len, reg_score_len,
                 standalong_classifier=False, with_regression=True, stpp_cfg=(1, 1, 1)):
        self.sc = standalong_classifier
        self.act_len = act_score_len
        self.comp_len = comp_score_len
        self.reg_len = reg_score_len
        self.with_regression = with_regression
        self.feat_dim = feat_dim
        parts = [parse_stage_config(c)[0] for c in stpp_cfg]
        self.stpp_cfg = tuple(parts)
        mult = sum(sum(p) for p in parts)
        self.act_slice = slice(0, self.act_len if self.sc else (self.act_len * mult))
        self.comp_slice = slice(self.act_slice.stop, self.act_slice.stop + self.comp_len * mult)
        self.reg_slice = slice(self.comp_slice.stop, self.comp_slice.stop + self.reg_len * mult)
        if not (self.sc and self.with_regression):
            raise NotImplementedError("the CUDA re-organised pooling covers the configuration SSN uses at test time "
                                      "(standalong_classifier=True, with_regression=True; ssn_test.py:64-66)")

    def forward(self, scores, proposal_ticks, scaling):
        assert scores.size(1) == self.feat_dim
        _need_cuda(scores, "scores")
        dev = scores.device
        scores = scores.contiguous().float()
        ticks = proposal_ticks.to(device=dev, dtype=torch.int32).contiguous()
        sc = scaling.to(device=dev, dtype=torch.float32).contiguous()
        n = ticks.size(0)
        out_act = torch.empty(n, self.act_len, dtype=torch.float32, device=dev)
        out_comp = torch.empty(n, self.comp_len, dtype=torch.float32, device=dev)
        out_reg = torch.empty(n, self.reg_len, dtype=torch.float32, device=dev)
        counts = [len(p) for p in self.stpp_cfg]
        levels = [v for p in self.stpp_cfg for v in p]
        with torch.cuda.device(dev):
            # one fp64 column scan of the score table + a two-load gather per pooled part
            ws = torch.empty(lib.ssnb_stpp_reorg_workspace_bytes(scores.size(0), scores.size(1)), dtype=torch.uint8, device=dev)
            check(lib.ssnb_stpp_reorg_prefix(scores.data_ptr(), scores.size(0), scores.size(1), ticks.data_ptr(), sc.data_ptr(),
                                             n, self.act_len, self.comp_len, self.reg_len, _lib.int_array(counts),
                                             _lib.int_array(levels), out_act.data_ptr(), out_comp.data_ptr(),
                                             out_reg.data_ptr(), ws.data_ptr(), _stream()), None, "stpp_reorg_prefix")
        return out_act, out_comp, out_reg


def _host_offsets(offsets, what):
    o = [int(x) for x in offsets]
    if not o or o[0] != 0 or any(b < a for a, b in zip(o, o[1:])):
        raise ValueError("%s must be V + 1 non-decreasing ints starting at 0" % what)
    return o


def reorg_packed(scores, tick_offsets, ticks32, scaling32, offsets, stpp_cfg, act_len, comp_len, reg_len, reg_stats=None):
    """The tail of ssn_test.py's worker loop (:87-92) for V videos in one library call (ssnb_stpp_reorg_batch):
    STPPReorgainzed.forward of every video (standalong_classifier, with_regression), then, with reg_stats, the regression
    de-normalisation.  scores [sum T, D] CUDA fp32, video v's ticks at rows tick_offsets[v] .. tick_offsets[v+1]-1; ticks32
    [sum N, 4] / scaling32 [sum N, 2] and offsets (V + 1 row offsets) as ops.proposal_lists.test_proposals returns them;
    stpp_cfg e.g. (1, (1, 2), 1); reg_stats: the checkpoint's [2, 2] (means, then stds), or None.
    -> device tensors (act [sum N, act_len], comp [sum N, comp_len], reg) ready for ops.detection.detections_packed, reg
    [sum N, reg_len // 2, 2] de-normalised when reg_stats is given, else the raw [sum N, reg_len].  Each video's rows are
    bitwise STPPReorgainzed.forward's for that video alone followed by the reference's two torch lines.
    Memory: the call holds (sum T + V) * D doubles of prefix tables beside the sum T * D fp32 scores, 12.8 KB + 6.4 KB per
    tick at K = 100 with (1, (1, 2), 1) (D = 1601): batch the videos so that a call fits (INTEGRATION.md)."""
    toff, off = _host_offsets(tick_offsets, "tick_offsets"), _host_offsets(offsets, "offsets")
    if len(toff) != len(off):
        raise ValueError("tick_offsets and offsets describe %d and %d videos" % (len(toff) - 1, len(off) - 1))
    V, T, N = len(off) - 1, toff[-1], off[-1]
    parts = [parse_stage_config(c)[0] for c in stpp_cfg]
    if len(parts) != 3:
        raise ValueError("stpp_cfg has three stages (starting, course, ending)")
    mult = sum(sum(p) for p in parts)
    if scores.dim() != 2 or scores.shape[0] != T:
        raise ValueError("scores must be [tick_offsets[-1] = %d, D], got %s" % (T, tuple(scores.shape)))
    D = scores.shape[1]
    if D != act_len + mult * (comp_len + reg_len):
        raise ValueError("D = %d does not match act_len + M * (comp_len + reg_len) with M = %d" % (D, mult))
    if tuple(ticks32.shape) != (N, 4) or tuple(scaling32.shape) != (N, 2):
        raise ValueError("ticks32 must be [offsets[-1] = %d, 4] and scaling32 [%d, 2]" % (N, N))
    stats = None
    if reg_stats is not None:
        stats = torch.as_tensor(reg_stats, dtype=torch.float64).cpu()
        if tuple(stats.shape) != (2, 2) or reg_len % 2:
            raise ValueError("reg_stats must be [2, 2] (means, then stds) and reg_len even")
        stats = (C.c_double * 4)(*stats.reshape(-1).tolist())
    for t, nm in ((scores, "scores"), (ticks32, "ticks32"), (scaling32, "scaling32")):
        _need_cuda(t, nm)
    dev = scores.device
    scores = scores.contiguous().float()
    ticks = ticks32.to(device=dev, dtype=torch.int32).contiguous()
    sc = scaling32.to(device=dev, dtype=torch.float32).contiguous()
    outs = [torch.empty(max(N, 1), L, dtype=torch.float32, device=dev) for L in (act_len, comp_len, reg_len)]
    c_toff, c_off = (C.c_int64 * (V + 1))(*toff), (C.c_int64 * (V + 1))(*off)
    ws_bytes = lib.ssnb_stpp_reorg_batch_workspace_bytes(c_toff, V, D)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    toff_dev = torch.tensor(toff, dtype=torch.int64, device=dev)
    off_dev = torch.tensor(off, dtype=torch.int64, device=dev)
    counts = [len(p) for p in parts]
    levels = [v for p in parts for v in p]
    with torch.cuda.device(dev):
        check(lib.ssnb_stpp_reorg_batch(scores.data_ptr(), D, c_toff, toff_dev.data_ptr(), ticks.data_ptr(), sc.data_ptr(), c_off,
                                        off_dev.data_ptr(), V, act_len, comp_len, reg_len, _lib.int_array(counts), _lib.int_array(levels),
                                        stats, *[o.data_ptr() for o in outs], ws.data_ptr(), ws_bytes, _stream()), None, "stpp_reorg_batch")
    act, comp, reg = (o[:N] for o in outs)
    return act, comp, (reg if stats is None else reg.view(N, reg_len // 2, 2))


class OHEMHingeLoss(torch.autograd.Function):
    """Class-wise hinge loss with online hard example mining; apply(pred, labels, is_positive,
    ohem_ratio, group_size) -> tensor of shape [1]; gradient only w.r.t. pred."""

    @staticmethod
    def forward(ctx, pred, labels, is_positive, ohem_ratio, group_size):
        n_sample = pred.size()[0]
        assert n_sample == len(labels), "mismatch between sample size and label size"
        _need_cuda(pred, "pred")
        dev = pred.device
        pred = pred.contiguous().float()
        labels = labels.to(device=dev, dtype=torch.int64).contiguous()
        K = pred.size(1)
        keep_num = int(group_size * ohem_ratio)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        kept = torch.empty(n_sample, dtype=torch.uint8, device=dev)
        slopes = torch.empty(2 * n_sample, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib.ssnb_ohem_hinge_fwd(pred.data_ptr(), labels.data_ptr(), n_sample, K, int(is_positive),
                                          int(group_size), keep_num, loss.data_ptr(), kept.data_ptr(),
                                          slopes.data_ptr(), _stream()), None, "ohem_hinge_fwd")
        ctx.save_for_backward(labels, kept, slopes)
        ctx.shape = (n_sample, K)
        return loss

    @staticmethod
    def backward(ctx, grad_output):
        labels, kept, slopes = ctx.saved_tensors
        m, K = ctx.shape
        g = grad_output.contiguous().float().view(-1)
        grad_in = torch.empty(m, K, dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            check(lib.ssnb_ohem_hinge_bwd(labels.data_ptr(), kept.data_ptr(), slopes.data_ptr(), g.data_ptr(), m, K,
                                          grad_in.data_ptr(), _stream()), None, "ohem_hinge_bwd")
        return grad_in, None, None, None, None


class CompletenessLoss(torch.nn.Module):
    def __init__(self, ohem_ratio=0.17):
        super(CompletenessLoss, self).__init__()
        self.ohem_ratio = ohem_ratio
        self.sigmoid = torch.nn.Sigmoid()

    def forward(self, pred, labels, sample_split, sample_group_size):
        """Per video the first `sample_split` rows are positives (all kept), the rest incomplete proposals (hardest
        `ohem_ratio` kept); both hinge sums are divided by the number of kept rows (ops/ssn_ops.py:223-239)."""
        n_pos, n_neg = sample_split, sample_group_size - sample_split

        def rows(t):                      # [videos, rows, ...] -> [videos * rows, ...]
            return t.contiguous().view(-1, *t.shape[2:])

        by_video = pred.view(-1, sample_group_size, pred.size(1))
        lab = labels.view(-1, sample_group_size)
        pos_pred, neg_pred = rows(by_video[:, :n_pos]), rows(by_video[:, n_pos:])
        pos_loss = OHEMHingeLoss.apply(pos_pred, rows(lab[:, :n_pos]), 1, 1.0, n_pos)
        neg_loss = OHEMHingeLoss.apply(neg_pred, rows(lab[:, n_pos:]), -1, self.ohem_ratio, n_neg)
        kept = float(pos_pred.size(0) + int(neg_pred.size(0) * self.ohem_ratio))
        return pos_loss / kept + neg_loss / kept


class _ClassWiseRegFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, labels, targets):
        _need_cuda(pred, "pred")
        dev = pred.device
        pred = pred.contiguous().float()
        labels = labels.to(device=dev, dtype=torch.int64).contiguous()
        targets = targets.to(device=dev, dtype=torch.float32).contiguous()
        n, K = pred.size(0), pred.size(1)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib.ssnb_classwise_reg_fwd(pred.data_ptr(), labels.data_ptr(), targets.data_ptr(), n, K,
                                             loss.data_ptr(), _stream()), None, "classwise_reg_fwd")
        ctx.save_for_backward(pred, labels, targets)
        return loss.view(())

    @staticmethod
    def backward(ctx, grad_output):
        pred, labels, targets = ctx.saved_tensors
        n, K = pred.size(0), pred.size(1)
        g = grad_output.contiguous().float().view(-1)
        gp = torch.empty_like(pred)
        with torch.cuda.device(pred.device):
            check(lib.ssnb_classwise_reg_bwd(pred.data_ptr(), labels.data_ptr(), targets.data_ptr(), g.data_ptr(), n, K,
                                             gp.data_ptr(), _stream()), None, "classwise_reg_bwd")
        return gp, None, None


class ClassWiseRegressionLoss(torch.nn.Module):
    """Location regression loss on the ground-truth class: SmoothL1(pred[i, label_i-1, :], target_i) * 2."""

    def __init__(self):
        super(ClassWiseRegressionLoss, self).__init__()

    def forward(self, pred, labels, targets):
        return _ClassWiseRegFn.apply(pred, labels, targets)
