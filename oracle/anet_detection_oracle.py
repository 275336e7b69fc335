"""numpy restatement, without pandas, of the ActivityNet toolkit's detection evaluation of a results file: ANETdetection's
wrapper_compute_average_precision (anet_toolkit/Evaluation/eval_detection.py:132-145) over compute_average_precision_detection
(:160-235) with segment_iou and interpolated_prec_rec (utils.py:14-51), in double.  The per-class AP is oracle/eval_oracle.py's
average_precision, the restatement the slot path (ops/detection.py) is tested against; this module only splits packed rows
by class.  It is the reference the GPU call (ssnb_detection_ap_rows) is tested against, and it is checked against the toolkit
itself on every golden fixture (oracle/gen_golden_anet_detection.py).

Tie rule (the GPU's): a class's rows are ranked by np.argsort(score, kind="stable")[::-1] -- NaN first, descending score,
equal scores the later file row first; equal tIoU the larger ground-truth index first, NaN tIoU first."""
import numpy as np

from .eval_oracle import average_precision


def detection(video, label, seg, score, gt_offsets, gt_cls, gt_seg, num_class, thresholds):
    """packed rows (video / label / seg [rows, 2] / score, file order) and ground truth (gt_offsets [V + 1], gt_cls, gt_seg
    [n_gt, 2]; instances past gt_offsets[V] count in npos only) -> dict(ap float64 [K, n_thr], rank int32 [rows] (-1 for a
    row outside the videos or classes), tp uint8 [n_thr, rows])"""
    video, label = np.asarray(video, np.int64), np.asarray(label, np.int64)
    seg, score = np.asarray(seg, np.float64).reshape(-1, 2), np.asarray(score, np.float64)
    gt_offsets, gt_cls = np.asarray(gt_offsets, np.int64), np.asarray(gt_cls, np.int64)
    gt_seg = np.asarray(gt_seg, np.float64).reshape(-1, 2)
    V, n_thr, rows = len(gt_offsets) - 1, len(thresholds), len(score)
    gt_video = np.full(len(gt_cls), -1, np.int64)
    gt_video[:gt_offsets[-1]] = np.repeat(np.arange(V), np.diff(gt_offsets))
    valid = (video >= 0) & (video < V)
    ap = np.zeros((num_class, n_thr))
    rank = np.full(rows, -1, np.int32)
    tp = np.zeros((n_thr, rows), np.uint8)
    for c in range(num_class):
        gm, pm = gt_cls == c, valid & (label == c)
        ap[c], r, t = average_precision(gt_video[gm], gt_seg[gm], video[pm], seg[pm], score[pm], thresholds, trace=True)
        rank[pm], tp[:, pm] = r, t
    return {"ap": ap, "rank": rank, "tp": tp}
