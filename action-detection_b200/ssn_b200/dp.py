"""Data-parallel host logic: one process per GPU, videos sharded over ranks, gradients exchanged with NCCL over one flat
fp32 buffer (replaces nn.DataParallel, ssn_train.py:67).

Loss normalisation stays exact under sharding (SURVEY section 8e): cross-entropy and regression are means over per-video
fixed row counts, so rank means average to the global mean; the completeness loss divides by pos_cnt + int(neg_cnt *
ohem_ratio) of the GLOBAL batch (ops/ssn_ops.py:236-239), which is NOT world * the per-rank value in general (B=64:
int(65.28)=65 vs 8*int(8.16)=64).

GradSync exchanges the flat gradient buffer in BUCKETS (heads -> inception_5b..4e -> 4d..4a -> 3c..conv1; "heads" is every
parameter outside base_model) on a communication stream while the backward of the layers below is still running (ssnb_backbone_bwd_range finalises a
bucket's weight gradients before returning); the whole pattern is capturable in a CUDA graph.
"""
import torch
import torch.distributed as dist


def completeness_denominator(global_videos, fg_per_video=1, comp_group=7, ohem_ratio=0.17):
    """pos_cnt + int(neg_cnt * ratio) of the global batch, Python int() semantics."""
    neg = comp_group - fg_per_video
    return global_videos * fg_per_video + int(global_videos * neg * ohem_ratio)


def shard_loss_config(global_videos, world, fg_per_video=1, comp_group=7, ohem_ratio=0.17):
    """(comp_denom, loss_scale) for one rank such that SUMMING the per-rank gradients over ranks
    reproduces the global-batch gradient."""
    assert global_videos % world == 0, "equal videos per rank"
    denom = completeness_denominator(global_videos, fg_per_video, comp_group, ohem_ratio)
    return float(denom) / world, 1.0 / world


class FlatGrads:
    """Views every parameter's .grad into one flat fp32 buffer so the gradient exchange is a single
    collective (42.3 MB for K=20 RGB).  (ssn_b200.optim.FusedSGD owns such a buffer itself.)"""

    def __init__(self, params, device):
        self.params = [p for p in params if p.requires_grad]
        self.flat = torch.zeros(sum(p.numel() for p in self.params), dtype=torch.float32, device=device)
        self.offsets = []
        off = 0
        for p in self.params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            self.offsets.append(off)
            off += p.numel()

    def rebind(self):
        """optimizer.zero_grad(set_to_none=True) (the default, and what the reference loop calls) drops the views: re-attach,
        keeping whatever gradient a parameter holds"""
        for p, off in zip(self.params, self.offsets):
            view = self.flat[off:off + p.numel()].view_as(p)
            if p.grad is None:
                view.zero_()
                p.grad = view
            elif p.grad.data_ptr() != view.data_ptr():
                view.copy_(p.grad)
                p.grad = view

    def zero(self):
        self.flat.zero_()
        self.rebind()

    def all_reduce(self):
        self.rebind()
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat)


BUCKET_STARTS = ("inception_4e_3x3_reduce", "inception_4a_1x1", "conv1_7x7_s2")     # first convolution (graph order) of each backbone bucket


class GradSync:
    """Bucketed all-reduce of a flat gradient buffer laid out in model.parameters() order, overlapped with the backward.

    sync = GradSync(flat_grad, params_in_flat_order, model)      # once
    losses = model.fused_step(..., grad_sync=sync)               # issues the bucket all-reduces as gradients become final
    sync.finish()                                                # the compute stream waits for the exchange; then optimizer.step()
    """

    def __init__(self, flat_grad, params, model, starts=BUCKET_STARTS):
        self.flat = flat_grad
        self.enabled = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        self.comm = torch.cuda.Stream(device=flat_grad.device) if self.enabled else None
        self.starts = tuple(starts)
        off, self.offset_of = 0, {}
        for p in params:
            self.offset_of[id(p)] = off
            off += p.numel()
        self.total = off
        bm = model.base_model
        convs = bm._convs()
        self.conv_offsets = [self.offset_of[id(c.weight)] for c in convs]
        # the head bucket: every parameter of the flat buffer outside base_model (SSN's three heads, BinaryClassifier's classifier_fc)
        in_backbone = {id(p) for p in bm.parameters()}
        self.heads_lo = min(self.offset_of[id(p)] for p in params if id(p) not in in_backbone)
        assert self.heads_lo >= max(self.conv_offsets), "flat buffer must hold the backbone parameters before the heads"
        self._ranges = {}
        self.launched = []

    def engine_buckets(self, eng):
        key = id(eng)
        if key not in self._ranges:
            ranges, first_convs = eng.bucket_ranges(list(self.starts))
            hi_off = self.heads_lo
            slices = []
            for ci in first_convs:
                lo_off = self.conv_offsets[ci]
                slices.append((lo_off, hi_off))
                hi_off = lo_off
            self._ranges[key] = (ranges, slices)
        return self._ranges[key]

    def _reduce(self, lo, hi):
        self.launched.append((lo, hi))
        if not self.enabled or hi <= lo:
            return
        self.comm.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.comm):
            dist.all_reduce(self.flat[lo:hi])

    def begin(self):
        self.launched = []

    def heads_done(self):
        self._reduce(self.heads_lo, self.total)

    def bucket_done(self, eng, i):
        lo, hi = self.engine_buckets(eng)[1][i]
        self._reduce(lo, hi)

    def finish(self):
        if self.enabled:
            torch.cuda.current_stream().wait_stream(self.comm)
