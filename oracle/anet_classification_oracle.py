"""numpy restatement, without pandas, of the ActivityNet toolkit's untrimmed video classification metrics:
compute_average_precision_classification per class (anet_toolkit/Evaluation/eval_classification.py:124-134,160-210),
interpolated_prec_rec (utils.py:14-23) and compute_video_hit_at_k (:212-249).  It is the reference the GPU call
(csrc/classification_ap.cu) is tested against, and it is checked against the toolkit itself, bitwise, on every golden fixture
(oracle/gen_golden_anet_classification.py).

Inputs are packed: prediction rows video / label / score, ground-truth (video, label) pairs (repeats count once, the
toolkit's drop_duplicates), V videos and K classes.  Ranking: np.argsort(score, kind="stable")[::-1], i.e. NaN first (argsort
puts NaN last), descending score, ties by descending row -- what the toolkit's argsort()[::-1] gives wherever its sort is
stable.  A class's rows and a video's rows keep the global ranking's order, as the toolkit ranks each subset on its own."""
import numpy as np


def rank(scores):
    return np.argsort(np.asarray(scores, np.float64), kind="stable")[::-1]


def interpolated_prec_rec(prec, rec):
    """utils.py:14-23; the backward max loop is np.maximum.accumulate (prec is never NaN here)"""
    mprec = np.hstack([[0], prec, [0]])
    mrec = np.hstack([[0], rec, [1]])
    mprec = np.maximum.accumulate(mprec[::-1])[::-1]
    idx = np.where(mrec[1::] != mrec[0:-1])[0] + 1
    return np.sum((mrec[idx] - mrec[idx - 1]) * mprec[idx])


def gt_pairs(gt_video, gt_label, V):
    """distinct ground-truth keys label * V + video, sorted"""
    return np.unique(np.asarray(gt_label, np.int64) * V + np.asarray(gt_video, np.int64))


def classification(video, label, score, gt_video, gt_label, V, K, top_k=3):
    """-> dict(ap float64 [K], hit_at_k, avg_hit_at_k, hits int32 [V], gt_labels int32 [V], tp uint8 [rows])"""
    video, label = np.asarray(video, np.int64), np.asarray(label, np.int64)
    score = np.asarray(score, np.float64)
    keys = gt_pairs(gt_video, gt_label, V)
    npos = np.bincount(keys // V, minlength=K)
    gt_labels = np.bincount(keys % V, minlength=V).astype(np.int32)
    order = rank(score)                                                         # the global ranking
    # per class: the first ranked row of each (class, video) is a true positive when the pair is ground truth (:190-203)
    by_class = order[np.argsort(label[order], kind="stable")]                    # (class, rank)
    by_cv = by_class[np.lexsort((video[by_class], label[by_class]))]           # (class, video, rank); lexsort is stable
    first = np.ones(len(by_cv), bool)
    first[1:] = (label[by_cv][1:] != label[by_cv][:-1]) | (video[by_cv][1:] != video[by_cv][:-1])
    tp = np.zeros(len(score), np.uint8)
    cand = by_cv[first]
    tp[cand[np.isin(label[cand] * V + video[cand], keys)]] = 1
    ap = np.zeros(K)
    bounds = np.searchsorted(label[by_class], np.arange(K + 1))
    with np.errstate(invalid="ignore", divide="ignore"):
        for c in range(K):
            rows = by_class[bounds[c]:bounds[c + 1]]
            if len(rows) == 0:
                continue
            t = tp[rows].astype(np.float64)
            cum_tp, cum_fp = np.cumsum(t), np.cumsum(1.0 - t)                    # :206-209
            ap[c] = interpolated_prec_rec(cum_tp / (cum_tp + cum_fp), cum_tp / float(npos[c]))
    # hit@k (:231-249): a video's top_k rows in its ranking; its distinct ground-truth labels among them
    by_video = order[np.argsort(video[order], kind="stable")]                    # (video, rank)
    v_sorted = video[by_video]
    start = np.searchsorted(v_sorted, v_sorted, side="left")
    top = by_video[np.arange(len(by_video)) - start < top_k]
    found = np.intersect1d(np.unique(label[top] * V + video[top]), keys)
    hits = np.bincount(found % V, minlength=V).astype(np.int32)
    with_gt = np.nonzero(gt_labels > 0)[0]                                      # np.unique order of the video ids
    frac = hits[with_gt] / gt_labels[with_gt].astype(np.float64)
    return {"ap": ap, "hit_at_k": float(np.ceil(frac).mean()), "avg_hit_at_k": float(frac.mean()), "hits": hits,
            "gt_labels": gt_labels, "tp": tp}
