"""ActivityNet proposal evaluation on the GPU: the toolkit's average recall against the average number of proposals per
video (AR-AN) and the area under that curve (anet_toolkit/Evaluation/eval_proposal.py:12-273, utils.py:25-75), every video
and tIoU threshold in one call of libssn_b200.so (csrc/proposal_ar.cu).  CUDA tensors only; there is no CPU path.

  average_recall_packed   average_recall_vs_avg_nr_proposals (:158-273) on packed device tensors
  ar_an_report            recall / avg_recall / proposals_per_video on the host and the area (:148-152), one small copy
  load_anet_ground_truth  ANETproposal._import_ground_truth (:56-99), packed
  load_anet_proposals     ANETproposal._import_proposal (:101-136), packed in the ground truth's video order
  evaluate_proposals      ANETproposal(...).evaluate() without printing

Packed layout (as ops/proposal_lists.py): boxes [rows, 2] float64 (t-start, t-end) and scores [rows] with first [V] int64 and
count [V] int32 (video v owns rows first[v] .. first[v] + count[v] - 1), so the seconds / slot0 / counts of
ops.proposals.bottom_up_proposals_packed are read in place.  Ground truth gt_seg [sum G, 2] float64 packed by V + 1 host
gt_offsets.  The evaluated videos are those with G_v > 0 (the toolkit's ground_truth['video-id'].unique()); a packed video with
G_v = 0 adds its proposals to P_all only, which is how proposals of videos outside the ground truth are counted.

Ranking rule: a video's proposals are ranked by the toolkit's proposals['score'].argsort()[::-1]: NaN scores first, then
descending score (-0 equal to +0), and ties -- NaN among them -- by DESCENDING row within the video.  That is what the toolkit
computes wherever numpy's sort is stable: numpy's portable sort is for up to 16 elements (insertion sort); above 16 it leaves
the tie order open, and so does numpy 2's x86-simd-sort, which it uses for float64 on CPUs with AVX2 or AVX-512, at every
size (there the toolkit's result on tied scores depends on the machine).  This rule is applied at every size.  It differs on purpose from the "ties keep input order" of ops/proposals.py and
ops/detection.py: here it is the toolkit's own order.

Deliberate differences from the toolkit:
  - total_nr == 0 (no evaluated video keeps a proposal): the toolkit raises ZeroDivisionError or divides by zero, depending on
    the integer type involved; here the curves are NaN and ar_an_report / evaluate_proposals raise ValueError.
  - a negative or non-finite max_avg_nr_proposals is rejected (None and 0 mean the default, P_all / V, as in the toolkit).
  - min(int(n * x), n) compares before converting, so a huge budget keeps every proposal where numpy's conversion overflows.
  - check_status=True (the blocked-video list fetched over HTTP) is not offered: blocked videos are an argument."""
import ctypes as C
import json
import math

import numpy as np
import torch

from ssn_b200._lib import lib, check
from ops.proposal_lists import _cuda, _dev_of, _on, _p, _stream

TIOU_THRESHOLDS = np.linspace(0.5, 0.95, 10)        # eval_proposal.py:20
GROUND_TRUTH_FIELDS = ("database", "taxonomy", "version")
PROPOSAL_FIELDS = ("results", "version", "external_data")


def average_recall_packed(boxes, scores, first, count, gt_seg, gt_offsets, max_avg_nr_proposals=None,
                          tiou_thresholds=TIOU_THRESHOLDS, trace=False):
    """-> dict of device tensors: recall float64 [T, 100], avg_recall [100], proposals_per_video [100], total_nr int64 [1];
    with trace=True also nr int32 [V] (proposals kept per video) and first_hit int32 [sum G, T] (the first ranked proposal
    with tIoU >= threshold, 2**31 - 1 for none).  boxes and scores must be CUDA tensors; first / count / gt_seg may be host
    data (then copied to the device); gt_offsets are V + 1 host ints.  Nothing is copied back: see ar_an_report."""
    dev = _dev_of(boxes)
    boxes, scores = _cuda(boxes, torch.float64, "boxes").reshape(-1, 2), _cuda(scores, torch.float64, "scores").reshape(-1)
    first, count = _on(dev, first, torch.int64).reshape(-1), _on(dev, count, torch.int32).reshape(-1)
    off = [int(o) for o in (gt_offsets.tolist() if hasattr(gt_offsets, "tolist") else gt_offsets)]
    V, rows = len(off) - 1, boxes.shape[0]
    if first.numel() != V or count.numel() != V or scores.numel() != rows:
        raise ValueError("need V first / count entries, V + 1 gt_offsets and one score per box row")
    max_avg = 0.0 if not max_avg_nr_proposals else float(max_avg_nr_proposals)
    if not math.isfinite(max_avg) or max_avg < 0:
        raise ValueError("max_avg_nr_proposals must be None, 0 or a positive finite number")
    thr = [float(t) for t in np.asarray(tiou_thresholds, np.float64).reshape(-1)]
    n = len(thr)
    gt_seg, off_dev = _on(dev, gt_seg, torch.float64).reshape(-1, 2), _on(dev, off, torch.int64)
    off_c, thr_c = (C.c_int64 * len(off))(*off), (C.c_double * n)(*thr)
    ws_bytes = lib.ssnb_proposal_ar_workspace_bytes(V, rows, off_c, n)          # 0 for arguments the call rejects
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    f64 = dict(dtype=torch.float64, device=dev)
    out = {"recall": torch.empty(n, 100, **f64), "avg_recall": torch.empty(100, **f64), "proposals_per_video": torch.empty(100, **f64),
           "total_nr": torch.empty(1, dtype=torch.int64, device=dev)}
    if trace:
        out["nr"] = torch.empty(max(V, 1), dtype=torch.int32, device=dev)
        out["first_hit"] = torch.empty(max(off[-1], 1), n, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssnb_proposal_ar(_p(boxes), _p(scores), rows, _p(first), _p(count), V, _p(gt_seg), off_c, off_dev.data_ptr(), thr_c, n,
                                   max_avg, out["recall"].data_ptr(), out["avg_recall"].data_ptr(), out["proposals_per_video"].data_ptr(),
                                   out["total_nr"].data_ptr(), out["nr"].data_ptr() if trace else None,
                                   out["first_hit"].data_ptr() if trace else None, ws.data_ptr(), ws_bytes, _stream()), None, "proposal_ar")
    if trace:
        out["nr"], out["first_hit"] = out["nr"][:V], out["first_hit"][:off[-1]]
    out["tiou_thresholds"] = np.asarray(thr)
    return out


def ar_an_report(result):
    """numpy recall, avg_recall, proposals_per_video and total_nr from one device-to-host copy, and the area under the AR-AN
    curve as ANETproposal.evaluate computes it: auc = trapezoid(avg_recall, proposals_per_video), auc_percent = 100 * auc /
    proposals_per_video[-1].  Raises ValueError when no evaluated video kept a proposal (total_nr == 0)."""
    n = result["recall"].shape[0]
    host = torch.cat([result["recall"].reshape(-1), result["avg_recall"], result["proposals_per_video"],
                      result["total_nr"].view(torch.float64)]).cpu().numpy()
    total_nr = int(host[-1:].view(np.int64)[0])
    if total_nr == 0:
        raise ValueError("no evaluated video kept a proposal (total_nr == 0): the average number of proposals is undefined")
    recall, avg, ppv = host[:100 * n].reshape(n, 100), host[100 * n:100 * n + 100], host[100 * n + 100:100 * n + 200]
    auc = float(np.trapezoid(avg, ppv))
    return {"recall": recall, "avg_recall": avg, "proposals_per_video": ppv, "total_nr": total_nr, "auc": auc,
            "auc_percent": 100.0 * auc / ppv[-1]}


def _json(json_or_dict):
    if isinstance(json_or_dict, dict):
        return json_or_dict
    with open(json_or_dict) as f:
        return json.load(f)


def load_anet_ground_truth(json_or_dict, subset="validation", blocked_videos=()):
    """_import_ground_truth (eval_proposal.py:56-99): the instances of the subset's videos, blocked videos left out.  -> dict(
    video_ids (the videos with at least one instance, in file order), segments float64 [sum G, 2], labels int32 [sum G] (the
    activity_index class, numbered in order of first appearance), gt_offsets (V + 1 ints), activity_index).  json_or_dict: a
    path or the parsed JSON."""
    data = _json(json_or_dict)
    if not all(k in data for k in GROUND_TRUTH_FIELDS):
        raise IOError("Please input a valid ground truth file.")
    blocked = set(blocked_videos)
    activity_index, ids, seg, lab, off = {}, [], [], [], [0]
    for vid, v in data["database"].items():
        if subset != v["subset"] or vid in blocked:
            continue
        for ann in v["annotations"]:
            activity_index.setdefault(ann["label"], len(activity_index))
            seg.append((ann["segment"][0], ann["segment"][1]))
            lab.append(activity_index[ann["label"]])
        if len(seg) > off[-1]:
            ids.append(vid)
            off.append(len(seg))
    return {"video_ids": ids, "segments": np.array(seg, np.float64).reshape(-1, 2), "labels": np.array(lab, np.int32),
            "gt_offsets": off, "activity_index": activity_index}


def load_anet_proposals(json_or_dict, video_ids, blocked_videos=()):
    """_import_proposal (eval_proposal.py:101-136) packed for average_recall_packed: the videos `video_ids` first, in that
    order (none of their proposals: count 0), then every other video of the file in file order, blocked videos left out.  A
    video's rows keep the file's order.  -> dict(video_ids, boxes float64 [rows, 2], scores float64 [rows], counts (host
    ints), first int64 [V] (numpy))."""
    data = _json(json_or_dict)
    if not all(k in data for k in PROPOSAL_FIELDS):
        raise IOError("Please input a valid proposal file.")
    blocked = set(blocked_videos)
    results = {vid: v for vid, v in data["results"].items() if vid not in blocked}
    known = set(video_ids)
    ids = list(video_ids) + [vid for vid in results if vid not in known]
    rows = [r for vid in ids for r in results.get(vid, ())]
    counts = [len(results.get(vid, ())) for vid in ids]
    return {"video_ids": ids, "boxes": np.array([(r["segment"][0], r["segment"][1]) for r in rows], np.float64).reshape(-1, 2),
            "scores": np.array([r["score"] for r in rows], np.float64), "counts": counts,
            "first": np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64) if counts else np.zeros(0, np.int64)}


def evaluate_proposals(ground_truth, proposals, subset="validation", max_avg_nr_proposals=None, tiou_thresholds=TIOU_THRESHOLDS,
                       blocked_videos=(), device=None):
    """ANETproposal(ground_truth, proposals, ..., check_status=False).evaluate() without printing, on `device` (default: the
    current CUDA device).  ground_truth / proposals: paths or parsed JSON.  -> ar_an_report's dict plus the video_ids of the
    evaluated videos."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("evaluate_proposals runs on a CUDA device: libssn_b200 has no CPU path")
    gt = load_anet_ground_truth(ground_truth, subset, blocked_videos)
    pr = load_anet_proposals(proposals, gt["video_ids"], blocked_videos)
    off = gt["gt_offsets"] + [gt["gt_offsets"][-1]] * (len(pr["video_ids"]) - len(gt["video_ids"]))
    r = average_recall_packed(torch.as_tensor(pr["boxes"]).to(dev), torch.as_tensor(pr["scores"]).to(dev), pr["first"], pr["counts"],
                              gt["segments"], off, max_avg_nr_proposals, tiou_thresholds)
    return ar_an_report(r) | {"video_ids": gt["video_ids"]}
