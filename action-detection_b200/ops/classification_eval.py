"""ActivityNet untrimmed video classification on the GPU: the toolkit's per-class average precision, mAP, hit@k and average
hit@k (anet_toolkit/Evaluation/eval_classification.py:10-249; eval_kinetics.py is the same code and prints error@k = 1 -
hit@k), every class and video in one call of libssn_b200.so (csrc/classification_ap.cu).  CUDA tensors only; there is no CPU
path.

  classification_ap_packed                 compute_average_precision_classification per class and compute_video_hit_at_k
                                           (:160-249) on packed device tensors
  classification_ap_dense                  the same for a [V, K] score matrix: every class of every video is a prediction
                                           (the form of SSN's video-level cls_scores)
  classification_report                    ap / mAP / hit@k / average hit@k / error@k on the host, one small copy
  load_anet_classification_ground_truth    ANETclassification._import_ground_truth (:48-87), packed
  load_anet_classification_predictions     ANETclassification._import_prediction (:89-122), packed
  evaluate_classification                  ANETclassification(...).evaluate() without printing

Packed layout: prediction rows video int32 / label int32 / score float64 [rows]; ground truth (video, label) pairs gt_video /
gt_label int32 [n_gt], repeated pairs counted once (drop_duplicates).  Videos are numbered 0..V-1, classes 0..K-1.

Ranking rule: a class's rows (for AP) and a video's rows (for hit@k) are ranked by the toolkit's score.argsort()[::-1]: NaN
first, then descending score (-0 equal to +0), equal scores by DESCENDING row.  That is the toolkit's order wherever numpy's
sort is stable; numpy leaves the order of ties open above 16 elements, and at every size where it dispatches float64 argsort
to x86-simd-sort (CPUs with AVX2 or AVX-512), so there the toolkit's result on tied scores depends on the machine.

AP is the toolkit's to about 1e-15 (the interpolated sum is reduced in a different order than np.sum); hit@k is exact and
average hit@k is summed in a fixed order, repeatable to the bit.  The loaders number the videos with ground truth in
np.unique order (sorted ids), as compute_video_hit_at_k walks them.

Deliberate differences from the toolkit: a prediction label outside the ground truth's classes is a ValueError (the toolkit
raises KeyError); no ground-truth video in the subset is a ValueError (the toolkit returns NaN with a warning); check_status
(the blocked-video list fetched over HTTP) is not offered: blocked videos are an argument."""
import ctypes as C
import json

import numpy as np
import torch

from ssn_b200._lib import lib, check
from ops.proposal_lists import _dev_of, _on, _p, _stream

GROUND_TRUTH_FIELDS = ("database", "taxonomy", "version")
PREDICTION_FIELDS = ("results", "version", "external_data")


def classification_ap_packed(video, label, score, gt_video, gt_label, n_videos, num_class, top_k=3, trace=False):
    """-> dict of device tensors: ap float64 [K], hit_at_k float64 [1], avg_hit_at_k float64 [1]; with trace=True also hits
    int32 [V] (each video's distinct ground-truth labels among its top_k rows), gt_labels int32 [V] (its distinct ground-truth
    labels) and tp uint8 [rows] (1: the row is a true positive of its class).  score must be a CUDA tensor; the other inputs
    may be host data (then copied to the device).  Rows or pairs outside 0..V-1 / 0..K-1 are ignored.  Nothing is copied
    back and nothing waits for the device: see classification_report."""
    dev = _dev_of(score, "score")
    score = score.to(torch.float64).contiguous().reshape(-1)
    video, label = _on(dev, video, torch.int32).reshape(-1), _on(dev, label, torch.int32).reshape(-1)
    gt_video, gt_label = _on(dev, gt_video, torch.int32).reshape(-1), _on(dev, gt_label, torch.int32).reshape(-1)
    rows, n_gt, V, K = score.numel(), gt_video.numel(), int(n_videos), int(num_class)
    if video.numel() != rows or label.numel() != rows or gt_label.numel() != n_gt:
        raise ValueError("need one video and one label per score row, and one label per ground-truth video")
    ws_bytes = lib.ssnb_classification_ap_workspace_bytes(rows, n_gt, V, K)       # 0 for arguments the call rejects
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    f64 = dict(dtype=torch.float64, device=dev)
    out = {"ap": torch.empty(max(K, 1), **f64), "hit_at_k": torch.empty(1, **f64), "avg_hit_at_k": torch.empty(1, **f64)}
    if trace:
        out["hits"] = torch.empty(max(V, 1), dtype=torch.int32, device=dev)
        out["gt_labels"] = torch.empty(max(V, 1), dtype=torch.int32, device=dev)
        out["tp"] = torch.empty(max(rows, 1), dtype=torch.uint8, device=dev)
    tr = [out[k].data_ptr() if trace else None for k in ("hits", "gt_labels", "tp")]
    with torch.cuda.device(dev):
        check(lib.ssnb_classification_ap(_p(video), _p(label), _p(score), rows, _p(gt_video), _p(gt_label), n_gt, V, K, int(top_k),
                                         out["ap"].data_ptr(), out["hit_at_k"].data_ptr(), out["avg_hit_at_k"].data_ptr(), *tr,
                                         ws.data_ptr(), ws_bytes, _stream()), None, "classification_ap")
    if trace:
        out["hits"], out["gt_labels"], out["tp"] = out["hits"][:V], out["gt_labels"][:V], out["tp"][:rows]
    out["top_k"] = int(top_k)
    return out


def classification_ap_dense(scores, gt_video, gt_label, top_k=3, trace=False):
    """classification_ap_packed of a CUDA score matrix [V, K]: row v * K + c is (video v, class c, scores[v, c]), the order
    of a prediction file written video by video with the classes in index order (which decides ties)."""
    dev = _dev_of(scores, "scores")
    if scores.dim() != 2:
        raise ValueError("scores must be [V, K]")
    V, K = scores.shape
    video = torch.arange(V, dtype=torch.int32, device=dev).repeat_interleave(K)
    label = torch.arange(K, dtype=torch.int32, device=dev).repeat(V)
    return classification_ap_packed(video, label, scores.reshape(-1), gt_video, gt_label, V, K, top_k, trace)


def classification_report(result):
    """numpy ap and the scalars from one device-to-host copy: map = ap.mean() (as evaluate() prints it), hit_at_k,
    avg_hit_at_k and error_at_k = 1 - hit_at_k (eval_kinetics.py's figure)."""
    host = torch.cat([result["ap"], result["hit_at_k"], result["avg_hit_at_k"]]).cpu().numpy()
    ap, hit, avg = host[:-2], float(host[-2]), float(host[-1])
    return {"ap": ap, "map": float(ap.mean()), "hit_at_k": hit, "avg_hit_at_k": avg, "error_at_k": 1.0 - hit, "top_k": result["top_k"]}


def _json(json_or_dict):
    if isinstance(json_or_dict, dict):
        return json_or_dict
    with open(json_or_dict) as f:
        return json.load(f)


def load_anet_classification_ground_truth(json_or_dict, subset="validation", blocked_videos=()):
    """_import_ground_truth (eval_classification.py:48-87): one row per distinct (video, label) of the subset's videos,
    blocked videos left out, in the toolkit's row order.  -> dict(video_ids (the videos with a label, sorted: np.unique
    order), video int32 [n] (index into video_ids), label int32 [n] (the activity_index class), activity_index (label ->
    class, numbered in order of first appearance)).  json_or_dict: a path or the parsed JSON."""
    data = _json(json_or_dict)
    if not all(k in data for k in GROUND_TRUTH_FIELDS):
        raise IOError("Please input a valid ground truth file.")
    blocked = set(blocked_videos)
    activity_index, pairs = {}, {}
    for vid, v in data["database"].items():
        if subset != v["subset"] or vid in blocked:
            continue
        for ann in v["annotations"]:
            activity_index.setdefault(ann["label"], len(activity_index))
            pairs.setdefault((vid, activity_index[ann["label"]]), None)
    ids = sorted({vid for vid, _ in pairs})
    at = {vid: i for i, vid in enumerate(ids)}
    return {"video_ids": ids, "video": np.array([at[vid] for vid, _ in pairs], np.int32),
            "label": np.array([c for _, c in pairs], np.int32), "activity_index": activity_index}


def load_anet_classification_predictions(json_or_dict, index, blocked_videos=()):
    """_import_prediction (eval_classification.py:89-122): every result row of the file, in file order, blocked videos left
    out.  index: load_anet_classification_ground_truth's result, whose activity_index and video numbering are kept; videos
    outside the ground truth are numbered after its videos, in file order.  -> dict(video_ids, video int32 [rows], label int32
    [rows], score float64 [rows]).  A label outside activity_index is a ValueError."""
    data = _json(json_or_dict)
    if not all(k in data for k in PREDICTION_FIELDS):
        raise IOError("Please input a valid prediction file.")
    blocked, classes = set(blocked_videos), index["activity_index"]
    ids = list(index["video_ids"])
    at = {vid: i for i, vid in enumerate(ids)}
    video, label, score = [], [], []
    for vid, v in data["results"].items():
        if vid in blocked:
            continue
        for r in v:
            if r["label"] not in classes:
                raise ValueError("prediction label %r of video %r is not a ground-truth class" % (r["label"], vid))
            if vid not in at:
                at[vid] = len(ids)
                ids.append(vid)
            video.append(at[vid])
            label.append(classes[r["label"]])
            score.append(r["score"])
    return {"video_ids": ids, "video": np.array(video, np.int32), "label": np.array(label, np.int32),
            "score": np.array(score, np.float64)}


def evaluate_classification(ground_truth, prediction, subset="validation", top_k=3, blocked_videos=(), device=None):
    """ANETclassification(ground_truth, prediction, subset, top_k=top_k, check_status=False).evaluate() without printing, on
    `device` (default: the current CUDA device).  ground_truth / prediction: paths or parsed JSON.  -> dict(ap (numpy, in
    activity_index order), map, hit_at_k, avg_hit_at_k, error_at_k, top_k, activity_index)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("evaluate_classification runs on a CUDA device: libssn_b200 has no CPU path")
    gt = load_anet_classification_ground_truth(ground_truth, subset, blocked_videos)
    if not gt["video_ids"]:
        raise ValueError("no ground-truth video in subset %r: AP and hit@k are undefined" % subset)
    pr = load_anet_classification_predictions(prediction, gt, blocked_videos)
    r = classification_ap_packed(pr["video"], pr["label"], torch.as_tensor(pr["score"]).to(dev), gt["video"], gt["label"],
                                 len(pr["video_ids"]), len(gt["activity_index"]), top_k)
    return classification_report(r) | {"activity_index": gt["activity_index"]}
