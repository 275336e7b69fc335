"""numpy restatement, without pandas, of the ActivityNet toolkit's proposal evaluation: average_recall_vs_avg_nr_proposals
(anet_toolkit/Evaluation/eval_proposal.py:158-273), segment_iou (utils.py:25-51) and the area ANETproposal.evaluate adds
(:148-152).  It is the reference the GPU call (csrc/proposal_ar.cu) is tested against bitwise, and it was checked against the
toolkit itself, bitwise, on the toolkit's own 4926-video sample (oracle/gen_golden_anet_proposal.py).

Videos come packed: counts[v] proposals (rows of boxes / scores, video after video) and gt_counts[v] ground-truth instances
(rows of gt).  The evaluated videos are those with gt_counts > 0, in order; a video without ground truth adds its proposals
to P_all only.  Ranking: np.argsort(score, kind="stable")[::-1], i.e. NaN first (argsort puts NaN last), descending score,
ties by descending row -- what the toolkit's pandas argsort()[::-1] gives wherever its sort is stable."""
import numpy as np

NEVER = np.iinfo(np.int32).max
THRESHOLDS = np.linspace(0.5, 0.95, 10)


def rank(scores):
    return np.argsort(np.asarray(scores, np.float64), kind="stable")[::-1]


def segment_iou(boxes, gt):
    """tIoU [G, n] of n proposals against G instances: utils.py:41-50 with the proposal as the target segment"""
    p, g = np.asarray(boxes, np.float64).reshape(-1, 2), np.asarray(gt, np.float64).reshape(-1, 2)
    with np.errstate(all="ignore"):
        tt1 = np.maximum(p[None, :, 0], g[:, None, 0])
        tt2 = np.minimum(p[None, :, 1], g[:, None, 1])
        inter = (tt2 - tt1).clip(0)
        union = (g[:, None, 1] - g[:, None, 0]) + (p[None, :, 1] - p[None, :, 0]) - inter
        return inter / union


def scaled_count(n, x):
    """min(int(n * x), n), compared before the conversion"""
    y = n * np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(y >= n, n, np.where(np.isnan(y), 0, np.minimum(y, n)).astype(np.int64))


def average_recall(boxes, scores, counts, gt, gt_counts, max_avg_nr_proposals=None, tiou_thresholds=THRESHOLDS):
    """-> dict(recall [T, 100], avg_recall [100], proposals_per_video [100], total_nr, nr int32 [videos], first_hit int32
    [sum G, T]).  total_nr == 0 (where the toolkit divides by zero): the curves are NaN."""
    counts, gt_counts = np.asarray(counts, np.int64), np.asarray(gt_counts, np.int64)
    thr = np.asarray(tiou_thresholds, np.float64).reshape(-1)
    first = np.concatenate([[0], np.cumsum(counts)])
    g_first = np.concatenate([[0], np.cumsum(gt_counts)])
    boxes, scores, gt = np.asarray(boxes, np.float64).reshape(-1, 2), np.asarray(scores, np.float64), np.asarray(gt, np.float64).reshape(-1, 2)
    V, p_all = int((gt_counts > 0).sum()), int(counts.sum())
    max_avg = max_avg_nr_proposals if max_avg_nr_proposals else (float(p_all) / V if p_all else 0.0)
    ratio = max_avg * float(V) / p_all if p_all else float("nan")
    nr = np.zeros(len(counts), np.int32)
    first_hit = np.full((int(g_first[-1]), len(thr)), NEVER, np.int32)
    cols = np.zeros(int(g_first[-1]), np.int64)
    for v in np.nonzero(gt_counts > 0)[0]:
        n, g0, g1 = int(counts[v]), int(g_first[v]), int(g_first[v + 1])
        if n == 0:
            tiou = np.zeros((g1 - g0, 1))                                          # :208-218
        else:
            nr[v] = int(scaled_count(n, ratio))
            order = rank(scores[first[v]:first[v] + n])[:nr[v]]
            tiou = segment_iou(boxes[first[v]:first[v] + n][order], gt[g0:g1])
        if tiou.shape[1]:                                                          # nr_v = 0: nothing is ever matched
            hit = tiou[:, None, :] >= thr[None, :, None]
            first_hit[g0:g1] = np.where(hit.any(-1), hit.argmax(-1), NEVER)
        cols[g0:g1] = tiou.shape[1]
    total_nr = int(nr.sum(dtype=np.int64))
    n_gt = int(g_first[-1])
    out = {"total_nr": total_nr, "nr": nr, "first_hit": first_hit}
    if total_nr == 0:
        nan = np.full(100, np.nan)
        return out | {"recall": np.full((len(thr), 100), np.nan), "avg_recall": nan, "proposals_per_video": nan.copy()}
    pcn = np.arange(1, 101) / 100.0 * (max_avg * float(V) / total_nr)              # :243
    n_vj = scaled_count(cols[:, None], pcn[None, :])                              # [sum G, 100]
    matches = (first_hit[:, :, None] < n_vj[:, None, :]).sum(0)                   # [T, 100], exact integers
    recall = matches.astype(np.float64) / float(n_gt)                             # :265
    acc = np.zeros(100)
    for t in range(len(thr)):                                                     # :268 recall.mean(axis=0)
        acc = acc + recall[t]
    out.update(recall=recall, avg_recall=acc / len(thr), proposals_per_video=pcn * (float(total_nr) / V))   # :271
    return out


def area(avg_recall, proposals_per_video):
    """ANETproposal.evaluate (:148-152): (auc, 100 * auc / proposals_per_video[-1])"""
    auc = np.trapezoid(avg_recall, proposals_per_video)
    return float(auc), 100.0 * float(auc) / proposals_per_video[-1]
