"""Detection post-processing on the GPU — the per-video work of the reference's eval_detection_results.py:91-183
(combined scores, class-wise temporal NMS, location regression) and ops/utils.py:56-82 (temporal_nms), executed by
libssn_b200.so (csrc/detect.cu) instead of numpy loops.  Inputs and outputs are CUDA tensors; nothing here has a CPU path.
"""
import ctypes as C

import torch

from ssn_b200._lib import lib, check


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def video_detections(rel_props, act_scores, comp_scores, reg_scores, nms_threshold, regress=True):
    """rel_props [N,2], act_scores [N,K+1], comp_scores [N,K], reg_scores [N,K,2] (or [N,2K]) of ONE video ->
    (detections [K,N,5], counts [K] int32): for class c the first counts[c] rows of detections[c] are the surviving
    (t0, t1, score, loc, dur) in descending score order — `dataset_detections[c][video]` after gen_detection_results, NMS and
    perform_regression (eval_detection_results.py:104-114,139-142,147-168; default branch, top_k <= 0)."""
    for t, nm in ((rel_props, "rel_props"), (act_scores, "act_scores"), (comp_scores, "comp_scores"), (reg_scores, "reg_scores")):
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: libssn_b200 has no CPU path" % nm)
    dev = act_scores.device
    props = rel_props.reshape(-1, 2).contiguous().float()
    act, comp = act_scores.contiguous().float(), comp_scores.contiguous().float()
    n, K = comp.shape
    reg = reg_scores.reshape(n, K, 2).contiguous().float()
    det = torch.zeros(K, max(n, 1), 5, dtype=torch.float32, device=dev)
    cnt = torch.zeros(K, dtype=torch.int32, device=dev)
    ws = torch.empty(max(n * K, 1), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssnb_detect_postprocess(props.data_ptr(), act.data_ptr(), comp.data_ptr(), reg.data_ptr(), n, K, float(nms_threshold),
                                          int(bool(regress)), det.data_ptr(), cnt.data_ptr(), ws.data_ptr(), _stream()), None, "detect_postprocess")
    return det, cnt


def temporal_nms(bboxes, thresh):
    """ops/utils.py:56-82 on the GPU: bboxes [n, >=3] rows (st, ed, score, ...) -> the kept rows in descending score order."""
    if not bboxes.is_cuda:
        raise RuntimeError("bboxes must be a CUDA tensor: libssn_b200 has no CPU path")
    n = bboxes.shape[0]
    if n == 0:
        return bboxes
    dev = bboxes.device
    b = bboxes.contiguous().float()
    props = b[:, :2].contiguous()
    scores = b[:, 2].contiguous()                       # [n, K=1]: ranked as they are
    # carry the row index through the "regression" slots: (loc, dur) = (row index, 0)
    reg = torch.stack([torch.arange(n, device=dev, dtype=torch.float32), torch.zeros(n, device=dev)], dim=1).contiguous()
    det = torch.zeros(1, n, 5, dtype=torch.float32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(lib.ssnb_detect_postprocess(props.data_ptr(), None, None, reg.data_ptr(), n, 1, float(thresh), 0, det.data_ptr(), cnt.data_ptr(),
                                          scores.data_ptr(), _stream()), None, "detect_postprocess")
    keep = det[0, :int(cnt.item()), 3].long()
    return bboxes[keep]


# ---- many videos at once: the three branches of gen_detection_results and the toolkit's AP --------------------------------
# Tie rule (numpy's default argsort leaves equal keys in an open order; this is the one the library and the numpy oracle
# oracle/eval_oracle.py follow):
#   - equal scores: the later entry ranks first, as in a stable ascending sort reversed -- the larger proposal index in the
#     top-k, cls and NMS stages, the later (video, kept position) in the class-wide AP ranking;
#   - equal tIoU: the larger ground-truth index (its position in the video's ground truth) is matched first;
#   - NaN ranks first, whatever its sign (a NaN score ahead of +inf; a NaN tIoU, from two zero-length segments, is not below
#     any threshold and is matched first, as argsort()[::-1] puts it first in the toolkit).
import os

import numpy as np

from ssn_b200._lib import DetectBatchCfg, DET_ALL, DET_TOPK, DET_CLS

# data/dataset_cfg.yaml:16-19 and :51-54 (evaluation: top_k, nms_threshold, softmax_before_filter), num_class :4 / :37, and
# the tIoU ranges of eval_detection_results.py:209-214
DATASETS = {
    "thumos14": dict(num_class=20, top_k=2000, nms_threshold=0.2, softmax_before_filter=True, iou_range=np.arange(0.1, 1.0, 0.1)),
    "activitynet1.2": dict(num_class=100, top_k=60, nms_threshold=0.6, softmax_before_filter=False,
                           iou_range=np.arange(0.5, 1.0, 0.05)),
}
_MODES = {"all": DET_ALL, "top_k": DET_TOPK, "cls": DET_CLS}


def detection_slots(offsets, num_class, mode, top_k=None, n_sel=None):
    """slot0 [V + 1] of the packed layout: video v owns slots slot0[v] .. slot0[v+1] - 1"""
    per = n_sel if mode == "cls" else num_class
    s = [0]
    for v in range(len(offsets) - 1):
        n = (offsets[v + 1] - offsets[v]) * per
        s.append(s[-1] + (min(top_k, n) if mode == "top_k" else n))
    return s


def detections_packed(rel_props, act, comp, reg, offsets, nms_threshold, mode="all", top_k=None, cls_sel=None,
                      softmax_before_filter=True, regress=True, trace=False):
    """Every video of a packed batch in one library call (csrc/detect.cu, ssnb_detect_batch).  rel_props [sum N, 2],
    act [sum N, K+1], comp [sum N, K], reg [sum N, K, 2] or None (zeros) as CUDA tensors; offsets: V + 1 ints.
    mode 'all' (top_k <= 0, eval_detection_results.py:103-113), 'top_k' (:114-129) or 'cls' (:130-145, cls_sel: [V, n_sel]
    selected classes per video).  -> dict of device tensors: dets [slots, 5] (t0, t1, score, loc, dur), counts [V, K]
    int32 and the host list slot0 [V + 1]: video v's survivors start at slot0[v], class by class in ascending order, counts[v, c]
    of class c in descending score order; slot0_dev is slot0 on the device.  trace=True adds combined [sum N, K] (the ranked
    scores) and sel [slots] (the selected pairs row * K + class, per video in ranking order)."""
    for t, nm in ((rel_props, "rel_props"), (act, "act"), (comp, "comp")):
        if not t.is_cuda:
            raise RuntimeError("%s must be a CUDA tensor: libssn_b200 has no CPU path" % nm)
    if mode not in _MODES:
        raise ValueError("mode must be one of %s" % sorted(_MODES))
    offsets = [int(o) for o in offsets]
    V = len(offsets) - 1
    dev = act.device
    comp = comp.contiguous().float()
    N, K = comp.shape
    if N != offsets[-1] or act.shape != (N, K + 1):
        raise ValueError("act [sum N, K+1] / comp [sum N, K] do not match offsets[-1] = %d" % offsets[-1])
    props = rel_props.reshape(-1, 2).contiguous().float()
    act = act.contiguous().float()
    regt = None if reg is None else reg.reshape(N, K, 2).contiguous().float()
    n_sel = 0
    sel_t = None
    if mode == "cls":
        sel_t = torch.as_tensor(cls_sel, dtype=torch.int32).to(dev).reshape(V, -1).contiguous()
        n_sel = sel_t.shape[1]
    cfg = DetectBatchCfg(_MODES[mode], int(top_k or 0), n_sel, int(bool(softmax_before_filter)), int(bool(regress)), 0, float(nms_threshold))
    offs = (C.c_int64 * (V + 1))(*offsets)
    ws_bytes = lib.ssnb_detect_batch_workspace_bytes(C.byref(cfg), K, offs, V)    # 0 for arguments the call rejects
    slot0 = detection_slots(offsets, K, mode, top_k, n_sel)
    S = slot0[-1]
    out = {"dets": torch.empty(max(S, 1), 5, dtype=torch.float32, device=dev),
           "counts": torch.empty(max(V, 1), K, dtype=torch.int32, device=dev)}
    if trace:
        out["combined"] = torch.empty(max(N, 1), K, dtype=torch.float32, device=dev)
        out["sel"] = torch.empty(max(S, 1), dtype=torch.int32, device=dev)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    offs_dev = torch.tensor(offsets, dtype=torch.int64, device=dev)

    def ptr(t):
        return None if t is None else t.data_ptr()
    with torch.cuda.device(dev):
        check(lib.ssnb_detect_batch(C.byref(cfg), props.data_ptr(), act.data_ptr(), comp.data_ptr(), ptr(regt), K, offs, offs_dev.data_ptr(), V,
                                    ptr(sel_t), out["dets"].data_ptr(), out["counts"].data_ptr(), ptr(out.get("combined")), ptr(out.get("sel")),
                                    ws.data_ptr(), ws_bytes, _stream()), None, "detect_batch")
    out["counts"] = out["counts"][:V]
    out["slot0"] = slot0
    out["slot0_dev"] = torch.tensor(slot0, dtype=torch.int64, device=dev)
    return out


def pack_ground_truth(gt_list, video_ids, device):
    """get_all_gt()'s [(video id, class, t0, t1)] -> dict(offsets [V + 1] host list, cls int32 [G], seg float64 [G, 2]) packed
    in the order of `video_ids`, each video's instances in list order; instances of videos not in video_ids follow, in
    list order (they count in npos only)"""
    pos = {v: i for i, v in enumerate(video_ids)}
    rows = [[] for _ in range(len(video_ids) + 1)]
    for g in gt_list:
        rows[pos.get(g[0], len(video_ids))].append(g)
    offsets = [0]
    for r in rows[:-1]:
        offsets.append(offsets[-1] + len(r))
    flat = [g for r in rows for g in r]
    cls = torch.tensor([int(g[1]) for g in flat], dtype=torch.int32, device=device)
    seg = torch.tensor([[float(g[2]), float(g[3])] for g in flat], dtype=torch.float64, device=device).reshape(-1, 2)
    return {"offsets": offsets, "cls": cls, "seg": seg}


def detection_ap(dets, gt, tiou_thresholds, trace=False):
    """compute_average_precision_detection (anet_toolkit/Evaluation/eval_detection.py:160-235) for every class and threshold
    in one library call (csrc/detection_ap.cu).  dets: detections_packed's dict; gt: pack_ground_truth's dict for the same
    videos.  -> dict: ap [K, n_thr] float64 on the device; trace=True adds rank [slots] (a survivor's position in its class's
    ranking) and tp [n_thr, slots] uint8 (written at survivor slots only)."""
    counts = dets["counts"]
    V, K = counts.shape
    dev = counts.device
    S = int(dets["slot0"][-1])
    thr = [float(t) for t in tiou_thresholds]
    G = int(gt["cls"].numel())
    if len(gt["offsets"]) != V + 1:
        raise ValueError("ground truth packed for %d videos, detections for %d" % (len(gt["offsets"]) - 1, V))
    ws_bytes = lib.ssnb_detection_ap_workspace_bytes(V, K, S, G, len(thr))
    out = {"ap": torch.empty(K, max(len(thr), 1), dtype=torch.float64, device=dev)}
    if trace:
        out["rank"] = torch.full((max(S, 1),), -1, dtype=torch.int32, device=dev)
        out["tp"] = torch.full((max(len(thr), 1), max(S, 1)), 255, dtype=torch.uint8, device=dev)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    goff = torch.tensor(gt["offsets"], dtype=torch.int64, device=dev)
    cls = gt["cls"].to(dev, torch.int32).contiguous()
    seg = gt["seg"].to(dev, torch.float64).contiguous()
    thr_c = (C.c_double * max(len(thr), 1))(*thr)
    with torch.cuda.device(dev):
        check(lib.ssnb_detection_ap(dets["dets"].data_ptr(), counts.contiguous().data_ptr(), dets["slot0_dev"].data_ptr(), V, K, S,
                                    goff.data_ptr(), cls.data_ptr(), seg.data_ptr(), G, thr_c, len(thr), out["ap"].data_ptr(),
                                    out["rank"].data_ptr() if trace else None, out["tp"].data_ptr() if trace else None,
                                    ws.data_ptr(), ws_bytes, _stream()), None, "detection_ap")
    return out


def _base_name(k):
    if isinstance(k, bytes):
        k = k.decode("utf-8")
    return os.path.splitext(os.path.basename(k))[0]


def evaluate_detections(score_dicts, gt_list, dataset=None, *, weights=None, nms_threshold=None, top_k=None, cls_scores=None,
                        cls_top_k=1, softmax_before_filter=None, regress=True, iou_range=None, device=None):
    """The body of eval_detection_results.py:45-251 without files, pickling or printing, on the GPU.
    score_dicts: one or several ssn_test.py --save_scores dicts, video id -> (rel_props, act, comp, reg or None); several are
    merged as a weighted sum in fp32 (weights: normalised to sum 1; default equal).  gt_list: SSNDataSet.get_all_gt()'s list.
    dataset ('thumos14' / 'activitynet1.2') supplies the defaults of nms_threshold, top_k, softmax_before_filter and
    iou_range.  cls_scores: video-level classifier scores, matched by file base name without extension (:85); given, the cls
    branch keeps each video's cls_top_k best classes.  regress=False is --no_regression.
    -> dict(ap [K, n_thr] numpy float64, map [n_thr] = ap.mean(0), average_map = map.mean(), iou_range) -- the script's table."""
    cfg = DATASETS[dataset] if dataset is not None else {}
    nms_threshold = nms_threshold if nms_threshold else cfg.get("nms_threshold")
    top_k = top_k if top_k else cfg.get("top_k", 0)
    softmax_before_filter = softmax_before_filter if softmax_before_filter else cfg.get("softmax_before_filter", False)
    iou_range = cfg.get("iou_range") if iou_range is None else iou_range
    if nms_threshold is None or iou_range is None:
        raise ValueError("give a dataset, or nms_threshold and iou_range")
    if isinstance(score_dicts, dict):
        score_dicts = [score_dicts]
    n = len(score_dicts)
    w = [1.0 / n] * n if weights is None else [float(x) / sum(weights) for x in weights]
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    vids = list(score_dicts[0])

    def t(x):
        return torch.as_tensor(np.asarray(x, dtype=np.float32), device=dev)

    def merged(vid, i):                                       # np.sum([a[i] * w ...], axis=0) in fp32
        acc = None
        for d, wi in zip(score_dicts, w):
            x = t(d[vid][i]) * wi
            acc = x if acc is None else acc + x
        return acc
    rel, act, comp, reg, offsets = [], [], [], [], [0]
    any_reg = any(score_dicts[0][v][3] is not None for v in vids)
    for vid in vids:
        r = t(score_dicts[0][vid][0])
        r = r.squeeze(0) if r.dim() == 3 else r
        a, c = merged(vid, 1), merged(vid, 2)
        rel.append(r.reshape(-1, 2))
        act.append(a)
        comp.append(c)
        if any_reg:
            K = c.shape[1]
            reg.append(merged(vid, 3).reshape(-1, K, 2) if score_dicts[0][vid][3] is not None
                       else torch.zeros(c.shape[0], K, 2, device=dev))
        offsets.append(offsets[-1] + c.shape[0])
    K = comp[0].shape[1]
    if cls_scores is None:
        mode, sel = ("all" if top_k <= 0 else "top_k"), None
    else:
        mode = "cls"
        by_name = {_base_name(k): v for k, v in cls_scores.items()}
        k = min(int(cls_top_k), K)
        sel = np.stack([np.argsort(np.asarray(by_name[_base_name(v)]), kind="stable")[-k:] for v in vids]).astype(np.int32)
    dets = detections_packed(torch.cat(rel), torch.cat(act), torch.cat(comp), torch.cat(reg) if any_reg else None, offsets,
                             nms_threshold, mode=mode, top_k=top_k, cls_sel=sel, softmax_before_filter=softmax_before_filter,
                             regress=regress)
    gt = pack_ground_truth(gt_list, vids, dev)
    ap = detection_ap(dets, gt, iou_range)["ap"].cpu().numpy()
    m = ap.mean(axis=0)
    return {"ap": ap, "map": m, "average_map": float(m.mean()), "iou_range": np.asarray(iou_range)}
