"""ActivityNet temporal detection evaluation on the GPU: the toolkit's ANETdetection (anet_toolkit/Evaluation/eval_detection.py:
11-158, driven by get_detection_performance.py) for a detection results JSON, every class and tIoU threshold in one call of
libssn_b200.so (csrc/detection_ap.cu, ssnb_detection_ap_rows: the matching and AP kernels of detection_ap, fed with the file's
double rows).  CUDA tensors only; there is no CPU path.

  detection_ap_rows                  compute_average_precision_detection (:160-235) of every class and threshold, packed rows
  pack_anet_detection                the loaders' output as the device tensors detection_ap_rows takes
  detection_report                   ap [n_thr, K] / mAP / average mAP on the host, and the toolkit's verbose lines
  load_anet_detection_ground_truth   ANETdetection._import_ground_truth (:53-93), packed per video
  load_anet_detection_predictions    ANETdetection._import_prediction (:95-130), packed rows in file order
  evaluate_anet_detection            ANETdetection(...).evaluate() without printing

Packed layout: prediction rows video int32 / label int32 / seg float64 [rows, 2] / score float64 [rows] in file order; ground
truth gt_offsets int64 [V + 1] (video v's instances are gt_offsets[v] .. gt_offsets[v+1]-1), gt_cls int32 and gt_seg float64
[n_gt, 2], in the toolkit's row order.  Every value stays a double: tIoU and the ranking are computed from the file's values.

Rules (csrc/detection_ap.cu, DESIGN.md section 4 "Tie rule"): a class's rows are ranked NaN first, then by descending score
(-0 equal to +0), equal scores the later file row first -- the toolkit's argsort()[::-1] wherever numpy's sort is stable (up
to 16 rows of a class; on CPUs where numpy dispatches float64 argsort to x86-simd-sort, at no size), so there the toolkit's
result on tied scores depends on the machine.  A row is matched in its own video and class to the unlocked ground truth of the
highest tIoU not below the threshold; equal tIoU takes the larger ground-truth index first, a NaN tIoU (two zero-length
segments) ranks first.  A row of a video without ground truth of its class is a false positive.  AP is the toolkit's to about
1e-15 (the interpolated sum is reduced in a different order than np.sum).

Deliberate differences from the toolkit: a prediction label outside the ground truth's classes is a ValueError naming the
video and the label (the toolkit raises KeyError); no ground-truth video in the subset is a ValueError (the toolkit returns
NaN with a warning); check_status (the blocked-video list fetched over HTTP) is not offered: blocked videos are an argument."""
import ctypes as C
import json

import numpy as np
import torch

from ssn_b200._lib import lib, check
from ops.proposal_lists import _dev_of, _on, _p, _stream

GROUND_TRUTH_FIELDS = ("database", "taxonomy", "version")
PREDICTION_FIELDS = ("results", "version", "external_data")
TIOU_THRESHOLDS = np.linspace(0.5, 0.95, 10)


def detection_ap_rows(video, label, seg, score, gt_offsets, gt_cls, gt_seg, num_class, tiou_thresholds=TIOU_THRESHOLDS, trace=False):
    """-> dict: ap float64 [K, n_thr] on the device; trace=True adds rank int32 [rows] (a row's position in its class's
    ranking; -1 for a row outside the videos or classes) and tp uint8 [n_thr, rows] (1 = true positive).  score must be a
    CUDA tensor; the other inputs may be host data (then copied to the device).  V = len(gt_offsets) - 1 videos; rows outside
    0..V-1 / 0..K-1 are ignored.  Nothing is copied back and nothing waits for the device: see detection_report."""
    dev = _dev_of(score, "score")
    score = score.to(torch.float64).contiguous().reshape(-1)
    video, label = _on(dev, video, torch.int32).reshape(-1), _on(dev, label, torch.int32).reshape(-1)
    seg = _on(dev, seg, torch.float64).reshape(-1)
    goff, gcls = _on(dev, gt_offsets, torch.int64).reshape(-1), _on(dev, gt_cls, torch.int32).reshape(-1)
    gseg = _on(dev, gt_seg, torch.float64).reshape(-1)
    rows, n_gt, V, K = score.numel(), gcls.numel(), goff.numel() - 1, int(num_class)
    if video.numel() != rows or label.numel() != rows or seg.numel() != 2 * rows or gseg.numel() != 2 * n_gt:
        raise ValueError("need one video, label and (t0, t1) segment per score row, and one segment per ground-truth instance")
    thr = [float(t) for t in np.asarray(tiou_thresholds, np.float64).reshape(-1)]
    n_thr = len(thr)
    ws_bytes = lib.ssnb_detection_ap_rows_workspace_bytes(rows, V, K, n_gt, n_thr)     # 0 for arguments the call rejects
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    out = {"ap": torch.empty(max(K, 1), max(n_thr, 1), dtype=torch.float64, device=dev)}
    if trace:
        out["rank"] = torch.full((max(rows, 1),), -1, dtype=torch.int32, device=dev)
        out["tp"] = torch.zeros(max(n_thr, 1), max(rows, 1), dtype=torch.uint8, device=dev)
    thr_c = (C.c_double * max(n_thr, 1))(*thr)
    with torch.cuda.device(dev):
        check(lib.ssnb_detection_ap_rows(_p(video), _p(label), _p(seg), _p(score), rows, V, K, _p(goff), _p(gcls), _p(gseg), n_gt,
                                         thr_c, n_thr, out["ap"].data_ptr(), out["rank"].data_ptr() if trace else None,
                                         out["tp"].data_ptr() if trace else None, ws.data_ptr(), ws_bytes, _stream()),
              None, "detection_ap_rows")
    if trace:
        out["rank"], out["tp"] = out["rank"][:rows], out["tp"][:, :rows]
    out["tiou_thresholds"] = np.array(thr)
    return out


def detection_report(result, activity_index=None):
    """numpy ap in the toolkit's orientation [n_thr, K] and its figures from one device-to-host copy: map [n_thr] =
    ap.mean(axis=1), average_map = map.mean() (evaluate()'s Average-mAP), tiou_thresholds, and `lines`, the toolkit's
    verbose [RESULTS] output"""
    ap = result["ap"].cpu().numpy().T.copy()
    m = ap.mean(axis=1)
    out = {"ap": ap, "map": m, "average_map": float(m.mean()), "tiou_thresholds": result["tiou_thresholds"],
           "lines": ["[RESULTS] Performance on ActivityNet detection task.", "\tAverage-mAP: {}".format(m.mean())]}
    if activity_index is not None:
        out["activity_index"] = activity_index
    return out


def _json(json_or_dict):
    if isinstance(json_or_dict, dict):
        return json_or_dict
    with open(json_or_dict) as f:
        return json.load(f)


def load_anet_detection_ground_truth(json_or_dict, subset="validation", blocked_videos=()):
    """_import_ground_truth (eval_detection.py:53-93): every annotation of the subset's videos, blocked videos left out, in the
    toolkit's row order (database order, each video's annotations in order).  -> dict(video_ids (the videos with an
    annotation, in database order), offsets int64 [V + 1], cls int32 [n_gt] (the activity_index class), seg float64 [n_gt, 2],
    activity_index (label -> class, numbered in order of first appearance)).  json_or_dict: a path or the parsed JSON."""
    data = _json(json_or_dict)
    if not all(k in data for k in GROUND_TRUTH_FIELDS):
        raise IOError("Please input a valid ground truth file.")
    blocked = set(blocked_videos)
    activity_index, ids, offsets, cls, seg = {}, [], [0], [], []
    for vid, v in data["database"].items():
        if subset != v["subset"] or vid in blocked or not v["annotations"]:
            continue
        for ann in v["annotations"]:
            cls.append(activity_index.setdefault(ann["label"], len(activity_index)))
            seg.append((ann["segment"][0], ann["segment"][1]))
        ids.append(vid)
        offsets.append(len(cls))
    return {"video_ids": ids, "offsets": np.array(offsets, np.int64), "cls": np.array(cls, np.int32),
            "seg": np.array(seg, np.float64).reshape(-1, 2), "activity_index": activity_index}


def load_anet_detection_predictions(json_or_dict, ground_truth, blocked_videos=()):
    """_import_prediction (eval_detection.py:95-130): every result row of the file, in file order, blocked videos left out.
    ground_truth: load_anet_detection_ground_truth's result, whose activity_index and video numbering are kept; videos without
    ground truth are numbered after its videos, in file order (their rows are false positives).  -> dict(video_ids, video
    int32 [rows], label int32 [rows], seg float64 [rows, 2], score float64 [rows]).  A label outside activity_index is a
    ValueError naming the video and the label."""
    data = _json(json_or_dict)
    if not all(k in data for k in PREDICTION_FIELDS):
        raise IOError("Please input a valid prediction file.")
    blocked, classes = set(blocked_videos), ground_truth["activity_index"]
    ids = list(ground_truth["video_ids"])
    at = {vid: i for i, vid in enumerate(ids)}
    video, label, seg, score = [], [], [], []
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
            seg.append((r["segment"][0], r["segment"][1]))
            score.append(r["score"])
    return {"video_ids": ids, "video": np.array(video, np.int32), "label": np.array(label, np.int32),
            "seg": np.array(seg, np.float64).reshape(-1, 2), "score": np.array(score, np.float64)}


def pack_anet_detection(ground_truth, prediction, device):
    """the two loaders' results as detection_ap_rows' device tensors: dict(video, label, seg, score, gt_offsets (padded to the
    prediction's videos: those without ground truth own no instance), gt_cls, gt_seg, num_class)"""
    V = len(prediction["video_ids"])
    off = np.concatenate([ground_truth["offsets"], np.full(V + 1 - len(ground_truth["offsets"]), ground_truth["offsets"][-1])])
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt).to(device)          # noqa: E731
    return {"video": T(prediction["video"], torch.int32), "label": T(prediction["label"], torch.int32),
            "seg": T(prediction["seg"], torch.float64), "score": T(prediction["score"], torch.float64),
            "gt_offsets": T(off, torch.int64), "gt_cls": T(ground_truth["cls"], torch.int32), "gt_seg": T(ground_truth["seg"], torch.float64),
            "num_class": len(ground_truth["activity_index"])}


def evaluate_anet_detection(ground_truth, prediction, subset="validation", tiou_thresholds=TIOU_THRESHOLDS, blocked_videos=(),
                            device=None):
    """ANETdetection(ground_truth, prediction, subset=subset, tiou_thresholds=tiou_thresholds, check_status=False).evaluate()
    without printing, on `device` (default: the current CUDA device).  ground_truth / prediction: paths or parsed JSON.
    -> dict(ap [n_thr, K] numpy (the toolkit's self.ap), map [n_thr] (self.mAP), average_map, tiou_thresholds,
    activity_index, lines (what verbose=True prints after evaluating))."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("evaluate_anet_detection runs on a CUDA device: libssn_b200 has no CPU path")
    gt = load_anet_detection_ground_truth(ground_truth, subset, blocked_videos)
    if not gt["video_ids"]:
        raise ValueError("no ground-truth video in subset %r: AP is undefined" % subset)
    pr = load_anet_detection_predictions(prediction, gt, blocked_videos)
    pk = pack_anet_detection(gt, pr, dev)
    r = detection_ap_rows(pk["video"], pk["label"], pk["seg"], pk["score"], pk["gt_offsets"], pk["gt_cls"], pk["gt_seg"],
                          pk["num_class"], tiou_thresholds)
    return detection_report(r, gt["activity_index"])
