"""Float64 restatement of the tail of the SSN training step.  TEST INFRASTRUCTURE ONLY.

What bench.py's training step runs around the backbone, op by op:
  fused global pool + dropout + STPP   (ssnb_gpool_stpp_fwd: gpool_stpp_v2_kernel / gpool_stpp_kernel)
  heads + multi-task loss + gradients  (ssnb_heads_loss_fwd_bwd: heads_loss_kernel)
  STPP backward                        (ssnb_stpp_bwd)
  momentum SGD, per-segment lr / wd    (ssnb_sgd_step_groups)
Each function below follows the reference lines the kernels cite and takes what the kernel consumed, so one op's rounding
never reaches the next (the pooled STPP is formed from the feat the kernel wrote; the heads are fed the kernel's course /
stpp).  Device-agnostic torch, float64.

`Checker` compares a kernel's outputs with these: the error of a quantity is max |got - ref| over the tensor, divided by
max |ref| of the tensor or, for per-row quantities (one row per proposal or frame), of the row; a record holds the worst
value and where it sits.  A NaN in got is an error unless ref has a NaN in the same place.

`ssn_step_dfeat` is the gradient such a step hands the backbone's backward, at the magnitude training produces.
"""
import math

import torch
import torch.nn.functional as F

from . import ssn_oracle as O
from . import synth

HEAD_KEYS = ("activity_fc.weight", "activity_fc.bias", "completeness_fc.weight", "completeness_fc.bias",
             "regressor_fc.weight", "regressor_fc.bias")
OHEM_GAP = 1e-4          # heads inputs: least gap between the last kept and the first dropped negative hinge loss of a group


def _d(t, device=None):
    return t.detach().to(device=device if device is not None else t.device, dtype=torch.float64)


# ---- pooling + STPP (ops/ssn_ops.py:39-70) -------------------------------------------------------------------------------
def part_table(stpp_cfg, seg_split):
    """(lo, hi, norm, scale_col) lists of the pyramid's parts over segment indices (ops/ssn_ops.py:49-53)"""
    parts = O.stpp_parts(stpp_cfg, seg_split)
    return tuple([p[i] for p in parts] for i in range(4))


def stpp64(feat, scaling, table, n_seg, course):
    """StructuredTemporalPyramidPooling.forward on per-frame features [F, D] -> (course [n, D], stpp [n, P * D]): per part
    the segment mean / norm, then * scaling[:, col] (ops/ssn_ops.py:49-64); course = mean over segments [course[0], course[1])"""
    src = _d(feat).view(-1, n_seg, feat.shape[-1])
    sc = _d(scaling, src.device).reshape(-1, 2) if scaling is not None else None
    parts = []
    for lo, hi, nm, col in zip(*table):
        p = src[:, lo:hi].mean(1) / nm
        if col >= 0:
            p = p * sc[:, col:col + 1]
        parts.append(p)
    stpp = torch.cat(parts, 1) if parts else src.new_zeros(src.shape[0], 0)
    return src[:, course[0]:course[1]].mean(1), stpp


def pool_stpp64(y5b, mask, table, scaling, n_seg, course):
    """the fused global pool + dropout + STPP: y5b [F, C, 7, 7] as the engine stored it (eng.read('inception_5b_output'));
    feat = pixel mean * mask (ssn_models.py:71-75 Dropout, after BNInception's global_pool), then course / stpp of feat"""
    feat = _d(y5b).mean((2, 3))
    if mask is not None:
        feat = feat * _d(mask, feat.device)
    return (feat,) + stpp64(feat, scaling, table, n_seg, course)


def stpp_vjp64(d_course, d_stpp, scaling, table, n_seg, course):
    """vjp of stpp64 with respect to the per-frame features: [n * n_seg, D]"""
    dc = _d(d_course)
    n, D = dc.shape
    g = dc.new_zeros(n, n_seg, D)
    g[:, course[0]:course[1]] += (dc / (course[1] - course[0])).unsqueeze(1)
    if table[0]:
        ds = _d(d_stpp, dc.device).view(n, -1, D)
        sc = _d(scaling, dc.device).reshape(-1, 2)
        for q, (lo, hi, nm, col) in enumerate(zip(*table)):
            v = ds[:, q] / nm
            if col >= 0:
                v = v * sc[:, col:col + 1]
            g[:, lo:hi] += (v / (hi - lo)).unsqueeze(1)
    return g.view(n * n_seg, D)


# ---- heads + multi-task loss (ssn_models.py:272-289, ops/ssn_ops.py:173-258, ssn_train.py:210-214) ----------------------
def heads_cfg(n, props_per_video, num_class, feat_mult, fg_per_video=1, comp_group=7, ohem_ratio=0.17, comp_w=0.1,
              reg_w=0.1, global_videos=None, loss_scale=1.0, feat_dim=1024):
    """the ssnb_heads_cfg fields as SSN.fused_step sets them (ssn_b200.dp.shard_loss_config): the completeness denominator of the
    GLOBAL batch, pos_cnt + int(neg_cnt * ratio) (ops/ssn_ops.py:236-239), times this call's share of the videos"""
    videos = n // props_per_video
    gv = videos if global_videos is None else global_videos
    neg = comp_group - fg_per_video
    denom = gv * fg_per_video + int(gv * neg * ohem_ratio)
    return dict(n=n, props_per_video=props_per_video, num_class=num_class, feat_dim=feat_dim, feat_mult=feat_mult,
                fg_per_video=fg_per_video, comp_group=comp_group, global_videos=gv, keep_neg=int(neg * ohem_ratio),
                comp_denom=float(denom) * videos / gv, comp_w=comp_w, reg_w=reg_w, loss_scale=loss_scale)


def _rows(prop_type):
    t = prop_type.reshape(-1)
    return (((t == 0) | (t == 2)).nonzero().view(-1), ((t == 0) | (t == 1)).nonzero().view(-1), (t == 0).nonzero().view(-1))


def _comp_hinge(raw_comp, comp_rows, target, cfg):
    """per group of comp_group completeness rows: (column picked, positive hinge losses [g, P], negative ones [g, Ng])"""
    K, G, P = cfg["num_class"], cfg["comp_group"], cfg["fg_per_video"]
    col = (target[comp_rows] - 1) % K                    # labels - 1 with Python's negative wrap (ops/ssn_ops.py:186)
    z = raw_comp[comp_rows, col].view(-1, G)
    return col, (1 - z[:, :P]).clamp_min(0), (1 + z[:, P:]).clamp_min(0)


def ohem_gap(raw_comp, prop_type, target, cfg):
    """least gap, over the groups, between the last kept and the first dropped negative hinge loss (inf if nothing is
    dropped; groups where both are 0 do not count, their choice changes neither loss nor gradient)"""
    _a, ci, _r = _rows(prop_type)
    _col, _lp, ln = _comp_hinge(_d(raw_comp), ci, target.reshape(-1).long(), cfg)
    k = cfg["keep_neg"]
    if k <= 0 or k >= ln.shape[1]:
        return math.inf
    s = ln.sort(1, descending=True).values
    gap = s[:, k - 1] - s[:, k]
    gap = torch.where((s[:, k - 1] == 0) & (s[:, k] == 0), torch.full_like(gap, math.inf), gap)
    return float(gap.min())


def heads_case(videos, num_class, feat_mult, fg_per_video=1, comp_group=7, props_per_video=8, seed=0, **cfg_kw):
    """seeded inputs of one heads + loss call: course, stpp, heads (synth_heads keys), prop_type, target, reg_target and the
    cfg (heads_cfg(**cfg_kw)).  Per video: fg_per_video proposals of type 0, then comp_group - fg_per_video incomplete ones
    (type 1), then background (type 2).  Re-seeded until every OHEM choice is at least OHEM_GAP away from a tie, so that
    the fp32 rounding of a logit cannot swap a kept negative."""
    from . import synth
    K, n = num_class, videos * props_per_video
    ptype = torch.tensor([0] * fg_per_video + [1] * (comp_group - fg_per_video) + [2] * (props_per_video - comp_group)).repeat(videos)
    cfg = heads_cfg(n, props_per_video, K, feat_mult, fg_per_video, comp_group, **cfg_kw)
    for attempt in range(100):
        s = seed * 100 + attempt
        g = torch.Generator().manual_seed(s)
        course, stpp = torch.randn(n, 1024, generator=g), torch.randn(n, 1024 * feat_mult, generator=g)
        heads = synth.synth_heads(K, feat_mult, seed=s, std=0.02, bias_std=0.1)
        target = torch.randint(1, K + 1, (n,), generator=g)
        target[ptype == 2] = 0
        reg_target = torch.randn(n, 2, generator=g)
        raw_comp = stpp.double() @ heads["completeness_fc.weight"].double().T + heads["completeness_fc.bias"].double()
        if ohem_gap(raw_comp, ptype, target, cfg) >= OHEM_GAP:
            return dict(course=course, stpp=stpp, heads=heads, prop_type=ptype, target=target, reg_target=reg_target, cfg=cfg)
    raise RuntimeError("no seed keeps the OHEM choices away from ties")


def heads_loss64(course, stpp, heads, prop_type, target, reg_target, cfg):
    """every output of ssnb_heads_loss_fwd_bwd in float64: raw logits (all rows), losses [act, comp, reg, total], d_course,
    d_stpp, and dW / db of the three heads.  cfg: the ssnb_heads_cfg fields (heads_cfg).
      activity      cross entropy, mean over the rows of type 0 / 2;
      completeness  per group of comp_group rows of type 0 / 1: the fg_per_video positives' hinge losses all kept, of the
                    negatives the keep_neg largest (ties: the lower index first), summed / comp_denom;
      regression    class-wise smooth L1 of the type-0 rows, mean over 2 * rows, * 2;
      total         act + comp_w * comp + reg_w * reg.
    Every gradient is multiplied by loss_scale, the losses are not.  A completeness row count that is not a multiple of
    comp_group gives a NaN completeness and total loss."""
    dev = course.device
    xc, xs = _d(course), _d(stpp, dev)
    aw, ab, cw, cb, rw, rb = (_d(heads[k], dev) for k in HEAD_KEYS)
    K, n, s = cfg["num_class"], xc.shape[0], float(cfg["loss_scale"])
    pt = prop_type.reshape(-1).to(dev).long()
    tg = target.reshape(-1).to(dev).long()
    rt = _d(reg_target, dev).reshape(-1, 2)
    raw_act, raw_comp, raw_reg = xc @ aw.T + ab, xs @ cw.T + cb, xs @ rw.T + rb
    da, dc, dr = torch.zeros_like(raw_act), torch.zeros_like(raw_comp), torch.zeros_like(raw_reg)
    ai, ci, ri = _rows(pt)
    la = lr = xc.new_zeros(())
    if len(ai):
        z = raw_act[ai]
        lse = torch.logsumexp(z, 1)
        la = (lse - z[torch.arange(len(ai), device=dev), tg[ai]]).mean()
        oh = torch.nn.functional.one_hot(tg[ai], K + 1).double()
        da[ai] = (torch.softmax(z, 1) - oh) / len(ai) * s
    G, keep, denom, cwt = cfg["comp_group"], cfg["keep_neg"], float(cfg["comp_denom"]), float(cfg["comp_w"])
    if len(ci) % G:
        lc = xc.new_tensor(math.nan)
    else:
        col, lp, ln = _comp_hinge(raw_comp, ci, tg, cfg)
        order = ln.sort(dim=1, descending=True, stable=True).indices
        kept = torch.zeros_like(ln, dtype=torch.bool).scatter_(1, order[:, :keep], True)
        lc = (lp.sum() + (ln * kept).sum()) / denom
        gz = torch.cat([torch.where(lp != 0, -1.0, 0.0), torch.where(kept & (ln != 0), 1.0, 0.0)], 1)
        dc[ci, col] = gz.reshape(-1).double() / denom * cwt * s
    if len(ri):
        col = (tg[ri] - 1) % K
        d = raw_reg.view(n, K, 2)[ri, col] - rt[ri]
        a = d.abs()
        lr = torch.where(a < 1, 0.5 * d * d, a - 0.5).sum() / (2 * len(ri)) * 2
        dr.view(n, K, 2)[ri, col] = d.clamp(-1, 1) / (2 * len(ri)) * 2 * float(cfg["reg_w"]) * s
    total = la + lc * cwt + lr * float(cfg["reg_w"])
    return {"raw_act": raw_act, "raw_comp": raw_comp, "raw_reg": raw_reg, "losses": torch.stack([la, lc, lr, total]),
            "d_course": da @ aw, "d_stpp": dc @ cw + dr @ rw,
            "d_act_w": da.T @ xc, "d_act_b": da.sum(0), "d_comp_w": dc.T @ xs, "d_comp_b": dc.sum(0),
            "d_reg_w": dr.T @ xs, "d_reg_b": dr.sum(0)}


# ---- momentum SGD (torch.optim.SGD, dampening 0, no Nesterov; per-parameter lr_mult / decay_mult, ssn_train.py:391-398) --
def sgd64(param, grad, mom_buf, seg_end, seg_lr, seg_wd, momentum, grad_mult=1.0):
    """one step over flat buffers cut into segments ending at seg_end: g' = g * grad_mult + wd * p, buf = momentum * buf + g',
    p -= lr * buf.  Returns (param, buf) in float64."""
    p, g, b = _d(param), _d(grad), _d(mom_buf)
    ends = seg_end.detach().to(device=p.device, dtype=torch.int64)
    seg = torch.bucketize(torch.arange(p.numel(), device=p.device), ends, right=True)
    lr, wd = _d(seg_lr, p.device)[seg], _d(seg_wd, p.device)[seg]
    b = momentum * b + (g * grad_mult + wd * p)
    return p - lr * b, b


# ---- comparator ----------------------------------------------------------------------------------------------------------
class Record:
    """one check: op, quantity, worst normalised error, bar, and where the worst error sits (row index, or element index
    for a tensor-wide normaliser)"""

    def __init__(self, op, quantity, err, bar, where):
        self.op, self.quantity, self.err, self.bar, self.where = op, quantity, err, bar, where

    @property
    def ok(self):
        return self.err <= self.bar

    @property
    def key(self):
        return (self.op, self.quantity)

    def __repr__(self):
        return "%s %s: %.3e (bar %.1e) at %s" % (self.op, self.quantity, self.err, self.bar, self.where)


class Checker:
    def __init__(self):
        self.records = []

    def add(self, op, quantity, got, ref, bar, rows=False):
        """rows: normalise each row (the first dimension) by its own max |ref|; else the whole tensor by max |ref|"""
        ref = _d(ref)
        got = _d(got, ref.device).reshape(ref.shape)
        both_nan = torch.isnan(got) & torch.isnan(ref)
        diff = torch.where(both_nan, torch.zeros_like(ref), (got - ref).abs())
        diff = torch.where(torch.isnan(diff), torch.full_like(diff, math.inf), diff)
        scale = torch.where(torch.isnan(ref), torch.zeros_like(ref), ref.abs())
        if rows:
            diff, scale = diff.reshape(ref.shape[0], -1), scale.reshape(ref.shape[0], -1)
            num, den = diff.amax(1), scale.amax(1)
        else:
            num, den = diff.reshape(1, -1), scale.reshape(-1).amax().expand(1, diff.numel())
        e = torch.where(den > 0, num / den.clamp_min(1e-300), torch.where(num > 0, torch.full_like(num, math.inf),
                                                                          torch.zeros_like(num))).reshape(-1)
        k = int(e.argmax()) if e.numel() else 0
        err = float(e[k]) if e.numel() else 0.0
        rec = Record(op, quantity, err, bar, ("row %d" % k) if rows else ("element %d" % k))
        self.records.append(rec)
        return rec

    def failures(self):
        return [r for r in self.records if not r.ok]

    def failed(self):
        return {r.key for r in self.failures()}

    def report(self):
        return "\n".join(map(repr, self.records))

    def assert_ok(self):
        bad = self.failures()
        assert not bad, "step check failed at:\n" + "\n".join(map(repr, bad))


# ---- per-op checks --------------------------------------------------------------------------------------------------------
# Bars, about 4x the worst value measured on an H100 80GB HBM3 (400 W) by tests/test_gpu_step_tail.py:
#   pooling: feat / course / stpp, fp32 sums of 49 pixels and of at most 16 segments.  EXACT_TC 2.8e-7 (first-generation
#            kernel, feat), FAST 1.1e-7 (gpool_stpp_v2_kernel<__half>, feat / course); the EXACT_TC bar stays at 1e-6;
#   STPP backward 1.3e-7; heads logits and gradients 9.2e-7 (d_course at K = 200); losses 2.3e-7; SGD 8.2e-8.
POOL_BARS = {"exact_tc": 1e-6, "fast": 5e-7}
POOL_BAR = POOL_BARS["exact_tc"]
STPP_BWD_BAR = 5e-7
LOGIT_BAR = 4e-6         # raw logits and every gradient of the heads kernel
LOSS_BAR = 1e-6          # each of the four losses, relative
SGD_BAR = 3e-7           # parameters and momentum after one step, per parameter tensor
LOSS_NAMES = ("loss_act", "loss_comp", "loss_reg", "loss_total")
ROW_KEYS = ("raw_act", "raw_comp", "raw_reg", "d_course", "d_stpp")
PARAM_KEYS = ("d_act_w", "d_act_b", "d_comp_w", "d_comp_b", "d_reg_w", "d_reg_b")


def check_pool_stpp(chk, op, y5b, mask, scaling, table, n_seg, course, feat, course_ft, stpp_ft, bar=POOL_BAR):
    """feat against the pixel mean (x mask) of y5b; course / stpp against STPP of the feat the kernel wrote"""
    ref_feat = _d(y5b).mean((2, 3))
    if mask is not None:
        ref_feat = ref_feat * _d(mask, ref_feat.device)
    chk.add(op, "feat", feat, ref_feat, bar, rows=True)
    rc, rs = stpp64(feat, scaling, table, n_seg, course)
    chk.add(op, "course", course_ft, rc, bar, rows=True)
    chk.add(op, "stpp", stpp_ft, rs, bar, rows=True)


def check_heads(chk, op, out, ref, bar=LOGIT_BAR, loss_bar=LOSS_BAR):
    """every output of one heads + loss call (out) against heads_loss64 (ref)"""
    for k in ROW_KEYS:
        chk.add(op, k, out[k], ref[k], bar, rows=True)
    for k in PARAM_KEYS:
        chk.add(op, k, out[k], ref[k], bar)
    for i, name in enumerate(LOSS_NAMES):
        chk.add(op, name, out["losses"][i:i + 1], ref["losses"][i:i + 1], loss_bar, rows=True)


def check_sgd(chk, op, seg_end, param, mom, ref_param, ref_mom, bar=SGD_BAR):
    """parameters and momentum after a step against sgd64, each parameter tensor (segment) normalised by itself"""
    lo = 0
    worst = {}
    for i, hi in enumerate(seg_end.tolist()):
        for q, got, ref in (("param", param, ref_param), ("momentum", mom, ref_mom)):
            c = Checker()
            r = c.add(op, q, got[lo:hi], ref[lo:hi], bar)
            if q not in worst or r.err > worst[q].err:
                worst[q] = Record(op, q, r.err, bar, "segment %d, %s" % (i, r.where))
        lo = hi
    chk.records.extend(worst.values())


# bench.py's training step: 4 videos x 8 proposals x 9 segments (F = 288), K = 20
STEP_VIDEOS, STEP_PROPS, STEP_SEG, STEP_K = 4, 8, 9, 20


def ssn_step_dfeat(feat, seed=0):
    """dL/dfeat of one SSN training step in float64, rounded to fp32: bench-shaped proposals (4 videos x 8 proposals x 9
    segments, K = 20), heads as ssn_models initialises them (N(0, 0.001), zero bias), a seeded dropout 0.8 mask on feat
    (ssn_models.fused_step), STPP (1, (1, 2), 1) and SSN's loss (oracle total_loss).  feat: [F, 1024]; F below 288 frames
    is tiled up to 288 and the first F rows of the gradient are returned."""
    F_ = feat.shape[0]
    n = STEP_VIDEOS * STEP_PROPS * STEP_SEG
    f64 = feat.detach().double().cpu().repeat((n + F_ - 1) // F_, 1)[:n].clone().requires_grad_(True)
    _x, scaling, target, reg_target, prop_type = synth.synth_batch(STEP_VIDEOS, STEP_K, 3, seed=seed, size=8)
    heads = {k: v.double() for k, v in synth.synth_heads(STEP_K, 5, std=0.001).items()}
    g = torch.Generator().manual_seed(500 + seed)
    keep = 0.2
    mask = (torch.rand(n, 1024, generator=g, dtype=torch.float64) < keep).double() / keep
    with torch.enable_grad():
        course, stpp = O.stpp_forward(f64 * mask, scaling.double(), [2, 7, STEP_SEG])
        raw_act = F.linear(course, heads["activity_fc.weight"], heads["activity_fc.bias"])
        raw_comp = F.linear(stpp, heads["completeness_fc.weight"], heads["completeness_fc.bias"])
        raw_reg = F.linear(stpp, heads["regressor_fc.weight"], heads["regressor_fc.bias"]).view(-1, STEP_K, 2)
        t = prop_type.view(-1)
        act_i, comp_i, reg_i = ((t == 0) | (t == 2)).nonzero().view(-1), ((t == 0) | (t == 1)).nonzero().view(-1), (t == 0).nonzero().view(-1)
        tg, rt = target.view(-1), reg_target.view(-1, 2).double()
        loss, _parts = O.total_loss((raw_act[act_i], tg[act_i], raw_comp[comp_i], tg[comp_i], raw_reg[reg_i], tg[reg_i], rt[reg_i]))
        (d,) = torch.autograd.grad(loss, f64)
    return d[:F_].float().to(feat.device)
