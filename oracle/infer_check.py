"""Float64 restatement of the test-time tail of SSN.  TEST INFRASTRUCTURE ONLY.

What runs after the backbone at test time (ssn_test.py:80-87, eval_detection_results.py:91-183), op by op:
  crop mean folded into the test FC   (ssnb_test_fc_cropmean: linear_cropmean_kernel)
  plain test FC                       (ssnb_linear_fwd: linear_fwd_kernel)
  re-organised STPP                   (ssnb_stpp_reorg_prefix: colscan_f64_kernel + stpp_reorg_prefix_kernel)
  combined scores, class-wise NMS, location regression   (ssnb_detect_postprocess: combined_scores_kernel + nms_regress_kernel)
Each function takes what the kernel consumed, so one op's rounding never reaches the next.  The error of a quantity is the
one of oracle/step_check.py (`Checker`): max |got - ref| over the tensor or the row, divided by max |ref| of the same, with
NaN positions required to match.  Orders and kept sets are compared exactly (`exact`).
"""
import math

import numpy as np
import torch

from . import ssn_oracle as O
from .step_check import Checker, Record, _d  # noqa: F401  (Checker is this module's comparator too)

# Bars, about 4x the worst value measured on an H100 80GB HBM3 (700 W) by tests/test_gpu_infer_tail.py (in brackets):
CROPMEAN_BAR = 2e-6      # linear_cropmean_kernel, per tick (row)                      [4.8e-7, in_dim 12000]
LINEAR_BAR = 3.5e-6      # linear_fwd_kernel, per row                                  [8.5e-7, out 2]
REORG_BAR = 1.3e-6       # re-organised STPP through the fp64 column prefix, act / comp / reg per proposal (row)
                         #                                                             [3.3e-7, 8-level course stage, comp]
COMBINED_BAR = 4e-6      # combined scores, per proposal (row)                         [9.1e-7, K = 200]
REGRESS_BAR = 4e-7       # regressed boxes of the survivors, per class                 [9.1e-8]


# ---- test FC (ssn_test.py:80-84, SSN.test_forward) -----------------------------------------------------------------------
def cropmean_fc64(feat, w, b, crops):
    """b + W . mean_c(x): feat [crops * nt, in] crop-major (rst.view(num_crop, -1, D).mean(0) after test_fc) -> [nt, out]"""
    x = _d(feat)
    x = x.view(crops, -1, x.shape[-1]).mean(0)
    return linear64(x, w, b)


def linear64(x, w, b):
    y = _d(x) @ _d(w, x.device).T
    return y if b is None else y + _d(b, x.device)


# ---- re-organised STPP (ops/ssn_ops.py:109-170) ----------------------------------------------------------------------------
def reorg_ticks(left, right, n_part):
    """int(np.arange(left, right + 1e-5, (right - left) / n_part)[q]) for q = 0 .. n_part: numpy stores p[0] = left,
    p[1] = left + step and fills p[q] = left + q * (p[1] - p[0]) for q >= 2, each operation rounded on its own"""
    left = float(left)
    step = (right - left) / n_part
    t1 = left + step
    delta = t1 - left
    return [int(left)] + [int(t1)] + [int(left + float(q) * delta) for q in range(2, n_part + 1)]


def _mean_rows(src, pl, pr):
    """src[pl:pr].mean(0) with Python slice semantics; an empty slice gives NaN"""
    a, b, _ = slice(pl, pr).indices(src.shape[0])
    if b <= a:
        return np.full(src.shape[1], np.nan)
    return src[a:b].mean(0)


def reorg64(scores, ticks, scaling, act_len, comp_len, reg_len, stpp_cfg=(1, 1, 1)):
    """STPPReorgainzed.forward (standalong_classifier=True, with_regression=True) in float64 -> (act, comp, reg).  scores
    [T, D], ticks [N, 4], scaling [N, 2].  activity = mean of rows [t1, max(t1 + 1, t2)); per stage, skipped when
    right <= 0 or left >= T; per part, added when pr - pl >= 1, times scaling[0] / 1 / scaling[1]"""
    cfg = tuple(O.parse_stage_config(c)[0] for c in stpp_cfg)
    mult = sum(sum(c) for c in cfg)
    src = _d(scores).cpu().numpy()
    tk = torch.as_tensor(ticks).reshape(-1, 4).tolist()
    sc = _d(torch.as_tensor(scaling)).reshape(-1, 2).cpu().tolist()
    T, n = src.shape[0], len(tk)
    a1 = act_len
    c1 = a1 + comp_len * mult
    out = [np.zeros((n, act_len)), np.zeros((n, comp_len)), np.zeros((n, reg_len))]

    def pspool(o, raw, t, s2, L):
        offset = 0
        for si, stage in enumerate(cfg):
            s = s2[0] if si == 0 else (s2[1] if si == len(cfg) - 1 else 1.0)
            left, right = t[si], max(t[si] + 1, t[si + 1])
            if right <= 0 or left >= T:
                offset += sum(stage)
                continue
            for n_part in stage:
                p = reorg_ticks(left, right, n_part)
                for q in range(n_part):
                    if p[q + 1] - p[q] >= 1:
                        o += _mean_rows(raw[:, offset * L:(offset + 1) * L], p[q], p[q + 1]) * s
                    offset += 1

    for i in range(n):
        out[0][i] = _mean_rows(src[:, :a1], tk[i][1], max(tk[i][1] + 1, tk[i][2]))
        pspool(out[1][i], src[:, a1:c1], tk[i], sc[i], comp_len)
        pspool(out[2][i], src[:, c1:], tk[i], sc[i], reg_len)
    return tuple(torch.from_numpy(o) for o in out)


def dataset_ticks(rel_props, T, starting_ratio=0.5, ending_ratio=0.5):
    """ssn_dataset.py:406-428: relative proposals [N, 2] (start < end) of a video sampled at T ticks -> (ticks [N, 4] int64,
    scaling [N, 2] float64), the augmented start / end clipped to [0, 1]"""
    ticks, scaling = [], []
    for st, ed in np.asarray(rel_props, dtype=np.float64).tolist():
        dur = ed - st
        rs, re_ = st - dur * starting_ratio, ed + dur * ending_ratio
        real_s, real_e = max(0.0, rs), min(1.0, re_)
        scaling.append(((st - real_s) / (dur * starting_ratio), (real_e - ed) / (dur * ending_ratio)))
        ticks.append((int(real_s * T), int(st * T), int(ed * T), int(real_e * T)))
    return torch.tensor(ticks, dtype=torch.int64), torch.tensor(scaling, dtype=torch.float64)


# ---- detection (eval_detection_results.py:104-168, ops/utils.py:38-82) -------------------------------------------------------
def _t(x):
    """a tensor or an array as a float64 tensor (on its device)"""
    return _d(torch.as_tensor(x))


def combined64(act, comp):
    """softmax(act)[:, 1:] * exp(comp) in float64"""
    act = _t(act)
    return torch.softmax(act, 1)[:, 1:] * torch.exp(_d(torch.as_tensor(comp), act.device))


def nms_order(scores):
    """the ranking NMS walks: NaN first (numpy's argsort()[::-1] puts NaN first), then descending, ties (and NaN against
    NaN) larger index first, which is a stable ascending argsort reversed"""
    s = np.asarray(scores, dtype=np.float64).reshape(-1)
    nan = np.isnan(s)
    return np.lexsort((-np.arange(s.size), -np.where(nan, 0.0, s), ~nan))


def nms64(props, scores, thr, order=None):
    """ops/utils.py:56-82 in numpy's arithmetic on fp32 boxes: the fp32 intersection and denominator, a double division, kept
    when IoU <= thr (NaN dropped) -> kept indices in kept order"""
    p = np.asarray(props, dtype=np.float32).reshape(-1, 2)
    t1, t2 = p[:, 0], p[:, 1]
    dur = t2 - t1
    order = nms_order(scores) if order is None else np.asarray(order)
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        rest = order[1:]
        inter = np.minimum(t2[i], t2[rest]) - np.maximum(t1[i], t1[rest])
        with np.errstate(invalid="ignore", divide="ignore"):
            iou = inter / (dur[i] + dur[rest] - inter).astype(np.float64)
        order = rest[np.where(iou <= thr)[0]]
    return np.array(keep, dtype=np.int64)


def regress64(props, loc, dur):
    """eval_detection_results.py:162-176 in float64: centre + duration * loc, duration * exp(dur), clipped to [0, 1] -> [n, 2]"""
    p = _t(props).reshape(-1, 2)
    loc, dur = _d(torch.as_tensor(loc), p.device).reshape(-1), _d(torch.as_tensor(dur), p.device).reshape(-1)
    c, d = (p[:, 0] + p[:, 1]) / 2, p[:, 1] - p[:, 0]
    nc, nd = c + d * loc, d * torch.exp(dur)
    return torch.stack([(nc - nd / 2).clamp(0, 1), (nc + nd / 2).clamp(0, 1)], 1)


# ---- checks ---------------------------------------------------------------------------------------------------------------
def exact(chk, op, quantity, got, ref, where=""):
    """an exact comparison (orders, kept sets, copied fields): error 0 when equal (NaN equal to NaN), else inf"""
    g, r = np.asarray(got), np.asarray(ref)
    same = g.shape == r.shape and bool(np.all((g == r) | (np.isnan(g.astype(np.float64)) & np.isnan(r.astype(np.float64)))))
    rec = Record(op, quantity, 0.0 if same else math.inf, 0.0, where)
    chk.records.append(rec)
    return rec


def worst(chk, op, quantity, recs):
    """fold per-class records into one: the largest error, and where it sits"""
    w = max(recs, key=lambda r: r.err) if recs else Record(op, quantity, 0.0, 0.0, "")
    chk.records.append(Record(op, quantity, w.err, w.bar, w.where))


def check_cropmean(chk, op, feat, w, b, crops, y, bar=CROPMEAN_BAR):
    chk.add(op, "y", y, cropmean_fc64(feat, w, b, crops), bar, rows=True)


def check_linear(chk, op, x, w, b, y, bar=LINEAR_BAR):
    chk.add(op, "y", y, linear64(x, w, b), bar, rows=True)


def check_reorg(chk, op, scores, ticks, scaling, act_len, comp_len, reg_len, stpp_cfg, outs, bar=REORG_BAR, ref=None):
    """outs = (act, comp, reg) of one call, each per proposal (row) against reorg64 (or `ref`, reorg64's result)"""
    ref = reorg64(scores, ticks, scaling, act_len, comp_len, reg_len, stpp_cfg) if ref is None else ref
    for q, got, r in zip(("act", "comp", "reg"), outs, ref):
        chk.add(op, q, got, r, bar, rows=True)
    return ref


def check_detect(chk, op, props, scores, thr, kept, dets=None, reg=None, act=None, comp=None, bar=REGRESS_BAR,
                 combined_bar=COMBINED_BAR):
    """one video's detection post-processing.  scores [N, K]: the scores the kernel ranked (its own combined scores, read
    back); kept: per class the kernel's surviving indices in kept order (compared exactly with nms64 of those scores);
    dets [K][n_c, 5] and reg [N, K, 2]: the kernel's regressed rows of the survivors (boxes against regress64 of the kept
    proposals, score / loc / dur copied exactly); act / comp: the kernel's inputs, for combined scores against combined64"""
    s = _t(scores).cpu().numpy()
    K = s.shape[1]
    if act is not None:
        chk.add(op, "combined", _t(scores), combined64(act, comp), combined_bar, rows=True)
    p = np.asarray(torch.as_tensor(props).float().cpu()).reshape(-1, 2)
    order_bad, fields, boxes = [], [], []
    for c in range(K):
        k = np.asarray(kept[c], dtype=np.int64)
        r = exact(Checker(), op, "order", k, nms64(p, s[:, c], thr), "class %d" % c)
        order_bad.append(r)
        if dets is None:
            continue
        d = _t(dets[c]).cpu().reshape(-1, 5)
        rg = _t(reg).cpu().reshape(-1, K, 2)[k, c]
        fields.append(exact(Checker(), op, "fields", d[:, 2:].numpy(),
                            np.stack([s[k, c], rg[:, 0].numpy(), rg[:, 1].numpy()], 1) if len(k) else np.zeros((0, 3)),
                            "class %d" % c))
        if len(k):
            ref = regress64(p[k], rg[:, 0], rg[:, 1])
            c_ = Checker()
            rec = c_.add(op, "boxes", d[:, :2], ref, bar)
            rec.where = "class %d, %s" % (c, rec.where)
            boxes.append(rec)
    worst(chk, op, "order", order_bad)
    if dets is not None:
        worst(chk, op, "fields", fields)
        worst(chk, op, "boxes", boxes)
