"""CPU restatement (numpy) of detection evaluation over many videos -- TEST INFRASTRUCTURE ONLY (only tests/ and tools/
may import anything under oracle/).

Follows eval_detection_results.py:91-237 without pandas: the three branches of gen_detection_results (all :103-113,
top_k :114-129, cls :130-145), class-wise temporal NMS (ops/utils.py:56-82), perform_regression (:162-174), and the
ActivityNet toolkit's compute_average_precision_detection (anet_toolkit/Evaluation/eval_detection.py:160-235) with
segment_iou and interpolated_prec_rec (utils.py:14-51).  It extends oracle/detect_oracle.py (softmax, perform_regression).
Pinned by tests/golden/eval.npz, produced by oracle/gen_golden_eval.py from the REAL reference functions.

Tie rule (the GPU's, see ops/detection.py): equal scores rank the later entry first (a stable ascending argsort reversed),
NaN first; equal tIoU the larger ground-truth index first.
"""
import numpy as np

from .detect_oracle import softmax, perform_regression


def temporal_nms_stable(bboxes, thresh):
    """temporal_nms with argsort(kind="stable"): equal scores (and NaN against NaN) the later row first"""
    t1, t2, scores = bboxes[:, 0], bboxes[:, 1], bboxes[:, 2]
    durations = t2 - t1
    order = scores.argsort(kind="stable")[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        tt1 = np.maximum(t1[i], t1[order[1:]])
        tt2 = np.minimum(t2[i], t2[order[1:]])
        intersection = tt2 - tt1
        with np.errstate(invalid="ignore", divide="ignore"):
            iou = intersection / (durations[i] + durations[order[1:]] - intersection).astype(float)
        order = order[np.where(iou <= thresh)[0] + 1]
    return bboxes[keep, :]


def branch_scores(act, comp, mode, softmax_before_filter=True):
    """the combined scores each branch ranks by (fp32, as numpy computes them on the fp32 arrays)"""
    with np.errstate(invalid="ignore", over="ignore"):
        if mode == "top_k":
            return softmax(act[:, 1:]) * np.exp(comp)
        if mode == "cls" and not softmax_before_filter:
            return act[:, 1:] * np.exp(comp)
        return softmax(act)[:, 1:] * np.exp(comp)


def select_pairs(combined, mode, top_k=None, classes=None):
    """the (proposal, class) pairs a branch hands to NMS, in the order they are appended: all / cls class by class, top_k the
    argsort(combined.ravel(), kind="stable")[-top_k:] pairs from the lowest kept score up"""
    n, K = combined.shape
    if mode == "top_k":
        keep = np.argsort(combined.ravel(), kind="stable")[-top_k:]
        return keep // K, keep % K
    cls = range(K) if mode == "all" else classes
    p = np.concatenate([np.arange(n) for _ in cls]) if n else np.zeros(0, np.int64)
    c = np.concatenate([np.full(n, k) for k in cls]) if n else np.zeros(0, np.int64)
    return p.astype(np.int64), c.astype(np.int64)


def video_detections_branch(rel_props, act, comp, reg, nms_thresh, mode="all", top_k=None, classes=None, softmax_before_filter=True,
                            regress=True):
    """gen_detection_results + NMS + perform_regression for one video -> {class: [n, 5] fp32 rows} (classes with rows only)"""
    num_class = comp.shape[1]
    rel = np.squeeze(rel_props, 0) if rel_props.ndim == 3 else rel_props
    reg = np.zeros((len(rel), num_class, 2), np.float32) if reg is None else reg.reshape((-1, num_class, 2))
    combined = branch_scores(act, comp, mode, softmax_before_filter)
    p, c = select_pairs(combined, mode, top_k, classes)
    out = {}
    for k in (sorted(set(c.tolist())) if len(c) else []):
        m = c == k
        rows = np.concatenate((rel[p[m]], combined[p[m], k][:, None], reg[p[m], k, 0][:, None], reg[p[m], k, 1][:, None]), axis=1)
        rows = temporal_nms_stable(rows, nms_thresh)
        out[k] = perform_regression(rows) if regress else rows
    return out


def class_topk(scores, k):
    """the cls_top_k classes of a video's classifier scores: np.argsort(..., kind="stable")[-k:]"""
    return np.argsort(np.asarray(scores), kind="stable")[-k:]


def segment_iou(target, candidates):
    """anet_toolkit utils.segment_iou in double"""
    tt1 = np.maximum(target[0], candidates[:, 0])
    tt2 = np.minimum(target[1], candidates[:, 1])
    inter = (tt2 - tt1).clip(0)
    union = (candidates[:, 1] - candidates[:, 0]) + (target[1] - target[0]) - inter
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter.astype(float) / union


def interpolated_prec_rec(prec, rec):
    mprec = np.hstack([[0], prec, [0]])
    mrec = np.hstack([[0], rec, [1]])
    for i in range(len(mprec) - 1)[::-1]:
        mprec[i] = max(mprec[i], mprec[i + 1])
    idx = np.where(mrec[1::] != mrec[0:-1])[0] + 1
    return np.sum((mrec[idx] - mrec[idx - 1]) * mprec[idx])


def average_precision(gt_video, gt_seg, pred_video, pred_seg, pred_score, thresholds, trace=False):
    """compute_average_precision_detection for one class without pandas.  gt_video [G] / gt_seg [G, 2]: the class's ground
    truth in order; pred_*: its predictions in (video, kept position) order.  -> ap [n_thr] (and with trace: the predictions'
    ranks and tp flags [n_thr, n_pred] in input order)"""
    gt_video, gt_seg = np.asarray(gt_video), np.asarray(gt_seg, np.float64).reshape(-1, 2)
    pred_seg = np.asarray(pred_seg, np.float64).reshape(-1, 2)
    npos = float(len(gt_video))
    n_thr, n = len(thresholds), len(pred_score)
    lock = np.full((n_thr, len(gt_video)), -1)
    order = np.asarray(pred_score, np.float64).argsort(kind="stable")[::-1]
    tp, fp = np.zeros((n_thr, n)), np.zeros((n_thr, n))
    by_video = {}
    for g, v in enumerate(gt_video.tolist()):
        by_video.setdefault(v, []).append(g)
    for idx, i in enumerate(order):
        rows = by_video.get(int(pred_video[i]))
        if rows is None:
            fp[:, idx] = 1
            continue
        rows = np.array(rows)
        tiou = segment_iou(pred_seg[i], gt_seg[rows])
        srt = tiou.argsort(kind="stable")[::-1]
        for t, thr in enumerate(thresholds):
            for j in srt:
                if tiou[j] < thr:
                    fp[t, idx] = 1
                    break
                if lock[t, rows[j]] >= 0:
                    continue
                tp[t, idx] = 1
                lock[t, rows[j]] = idx
                break
            if fp[t, idx] == 0 and tp[t, idx] == 0:
                fp[t, idx] = 1
    ap = np.zeros(n_thr)
    for t in range(n_thr):
        this_tp = np.cumsum(tp[t]).astype(float)
        this_fp = np.cumsum(fp[t]).astype(float)
        with np.errstate(invalid="ignore", divide="ignore"):
            ap[t] = interpolated_prec_rec(this_tp / (this_tp + this_fp), this_tp / npos)
    if not trace:
        return ap
    rank = np.empty(n, np.int64)
    rank[order] = np.arange(n)
    return ap, rank, tp[:, rank].astype(np.uint8)


def ap_table(dets, gt, num_class, thresholds, classes=None):
    """dets: {class: [(video, rows [n, 5])...]} in video order; gt: [(video, cls, t0, t1)] -> ap [K, n_thr] (NaN rows for
    classes not in `classes`)"""
    ap = np.full((num_class, len(thresholds)), np.nan)
    for c in (range(num_class) if classes is None else classes):
        g = [(v, t0, t1) for v, k, t0, t1 in gt if k == c]
        pv = [v for v, r in dets.get(c, []) for _ in range(len(r))]
        ps = np.concatenate([r[:, :2] for _, r in dets.get(c, [])]) if pv else np.zeros((0, 2))
        sc = np.concatenate([r[:, 2] for _, r in dets.get(c, [])]) if pv else np.zeros(0)
        ap[c] = average_precision([x[0] for x in g], [x[1:] for x in g], pv, ps.astype(np.float64), sc.astype(np.float64), thresholds)
    return ap
