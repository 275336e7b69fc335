"""numpy restatement of the reference's ops/video_funcs.py and ops/metrics.py (video-level aggregation, fusion and metrics),
for one video or a packed batch, without sklearn.  float32 arithmetic is left to numpy in the reference's own order, so the
aggregates are numpy's to the bit; the metrics are restated from their definitions.

Packed layout: scores [sum T, crops, D] with int64 tick offsets [V+1]; labels as (video, label) pairs."""
import math

import numpy as np


def softmax(x, T=1):
    """metrics.py:8-11: shift by the (NaN-propagating) row max, exp, divide by the row sum.  The float32 exp is taken as the
    float64 exp rounded to float32, the same on every CPU; numpy's own float32 exp differs by CPU (its SIMD versions are
    within a few ulp; without SIMD it is libm's expf, which the golden vectors used)."""
    z = (x - x.max(axis=-1)[..., None]) * T
    e = np.exp(z.astype(np.float64)).astype(z.dtype) if z.dtype == np.float32 else np.exp(z)
    return e / e.sum(axis=-1)[..., None]


def crop_reduce(score, crop_agg="mean"):
    return score.max(axis=1) if crop_agg == "max" else score.mean(axis=1)


def default_agg(score, normalization=True, crop_agg="mean"):
    """video_funcs.py:8-18"""
    r = crop_reduce(score, crop_agg).mean(axis=0)
    return softmax(r) if normalization else r


def top_mean(x, k):
    """np.sort along ticks (NaN last), the last k rows (all when k > n), their mean: video_funcs.py:24,43"""
    return np.sort(x, axis=0)[-k:, :].mean(axis=0)


def top_k_agg(score, k, normalization=True, crop_agg="mean"):
    """video_funcs.py:21-26"""
    r = top_mean(crop_reduce(score, crop_agg), k)
    return softmax(r) if normalization else r


def window_steps(spans, overlap, fps):
    """video_funcs.py:45-47: span = t_span * fps ticks, step = int(ceil(span * (1 - overlap)))"""
    return [(s * fps, int(math.ceil(s * fps * (1 - overlap)))) for s in spans]


def sliding_agg(score, spans=(1, 2, 4, 8, 16), overlap=0.2, norm=True, fps=1):
    """video_funcs.py:29-57: the crop MEAN (named frm_max there); per span the window maxima over [i, i + span) for i in
    range(0, T, step), the mean of their max(15, n // 4) largest (Python 2 division, :49); the mean over spans"""
    frm = score.mean(axis=1)
    T = frm.shape[0]
    per_span = []
    for span, step in window_steps(spans, overlap, fps):
        win = np.array([frm[i:i + span].max(axis=0) for i in range(0, T, step)])
        per_span.append(top_mean(win, max(15, len(win) // 4)))
    r = np.mean(per_span, axis=0)
    return softmax(r) if norm else r


def tpp_agg(score, num_class):
    """video_funcs.py:60-70: crop mean; tick t adds columns [k K, (k + 1) K) of stage k = int(t * (stage / T)) into a
    float64 accumulator; divided by T"""
    frm = score.mean(axis=1)
    T, stage = frm.shape[0], frm.shape[1] // num_class
    step = float(stage) / T
    acc = np.zeros(num_class)
    for t in range(T):
        k = int(t * step)
        acc += frm[t, k * num_class:(k + 1) * num_class]
    return acc / T


def fuse(major, others, weights, norm=True):
    """video_funcs.py:73-80 without the in-place update of major"""
    out = major.copy()
    for s, w in zip(others, weights):
        out += s * w
    return softmax(out) if norm else out


def aggregate_packed(scores, offsets, mode, **kw):
    fn = {"default": default_agg, "top_k": top_k_agg, "sliding_window": sliding_agg, "tpp": tpp_agg}[mode]
    return np.stack([fn(scores[offsets[v]:offsets[v + 1]], **kw) for v in range(len(offsets) - 1)])


# ---- metrics.py ------------------------------------------------------------------------------------------------------------

def rank(scores):
    """one video's classes best first: NaN first, then descending score (-0 == +0), equal scores the higher class first (a
    stable ascending argsort reversed) -- the tie rule of ops/metrics.py"""
    s = np.asarray(scores, np.float64)
    key = np.where(np.isnan(s), np.inf, np.where(s == 0, 0.0, s))
    return np.argsort(key, kind="stable")[::-1]


def top_k_acc(lb_set, scores, k=3):
    """metrics.py:14-16"""
    idx = set(rank(scores)[:k].tolist())
    return len(set(lb_set) & idx), len(lb_set)


def top_k_hit(lb_set, scores, k=3):
    """metrics.py:19-21"""
    return top_k_acc(lb_set, scores, k)[0] > 0, 1


def average_precision(y, s):
    """sklearn average_precision_score of one column (precision_recall_curve then -sum(diff(recall) * precision[:-1])): the
    distinct thresholds in descending order, each adding (tps - previous tps) / P * tps / (rank + 1); no positive: 0"""
    y, s = np.asarray(y, np.float64), np.asarray(s, np.float64)
    order = np.argsort(-s, kind="stable")
    ys, ss = y[order], s[order]
    ends = np.r_[np.nonzero(np.diff(ss))[0], len(ss) - 1]
    tps = np.cumsum(ys)[ends]
    P = tps[-1] if len(tps) else 0.0
    if P == 0:
        return 0.0
    prev = np.r_[0.0, tps[:-1]]
    return float(np.sum((tps - prev) / P * (tps / (ends + 1))))


def video_mean_ap(scores, label_sets):
    """metrics.py:41-50: the macro mean of the per-class AP of the label indicator"""
    scores = np.asarray(scores)
    gt = np.zeros(scores.shape)
    for i, ls in enumerate(label_sets):
        gt[i, sorted(ls)] = 1
    ap = np.array([average_precision(gt[:, c], scores[:, c]) for c in range(scores.shape[1])])
    return float(ap.mean()), ap


def confusion(scores, labels):
    """argmax and the counts of metrics.py:53-60 over classes 0..K-1: label counts, prediction counts, hits"""
    K = scores.shape[1]
    pred = np.argmax(scores, axis=1)
    labels = np.asarray(labels)
    cnt = np.bincount(labels, minlength=K)
    pcnt = np.bincount(pred, minlength=K)
    hit = np.bincount(labels[labels == pred], minlength=K)
    return pred, np.stack([cnt, pcnt, hit]).astype(np.int32)


def mean_class_accuracy(scores, labels):
    """metrics.py:53-60: mean of hits / label count over the classes labelled or predicted (0 / 0 = NaN, as numpy)"""
    _, cf = confusion(scores, labels)
    used = (cf[0] > 0) | (cf[1] > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.mean(cf[2][used] / cf[0][used].astype(float)))


def top_k_accuracy(scores, label_sets, k):
    """metrics.py:28-38 over the videos present"""
    return float(np.mean([top_k_hit(ls, s, k)[0] for ls, s in zip(label_sets, scores)]))
