"""Proposal labelling on the GPU: the stage of the reference between "boxes" and "what SSN trains and tests on", for many
ragged videos per call of libssn_b200.so (csrc/proposal_lists.cu).  CUDA tensors only; there is no CPU path.

  name_proposals_packed     name_proposal (ops/detection_metrics.py:54-76) + per-ground-truth maximum tIoU
  proposal_recall           temporal_recall / get_temporal_proposal_recall (:31-51,79-83) at many thresholds
  sliding_window_proposals  gen_exponential_sw_proposal (ops/sequence_funcs.py:37-54)
  proposal_frames           dump_window_list / process_proposal_list frame windows (ops/io.py:44-47,109-127) and
                            SSNVideoRecord's validity rules (ssn_dataset.py:13-21,81-93)
  proposal_targets          SSNDataSet._parse_prop_file: pools, regression targets, reg_stats (ssn_dataset.py:29-55,103-131,382-391)
  test_proposals            get_test_data's rel_prop / proposal_ticks / scaling (ssn_dataset.py:393-428)
  label_proposals           the tail of gen_bottom_up_proposals.py:158-193 / gen_sliding_window_proposals.py:44-60 in one call
  format_proposal_list / write_proposal_list / load_proposal_list / record_rows    the list file, both ways

Packed layout: boxes [rows, 2] float64 with first [V] int64 and count [V] int32 on the device (video v owns rows first[v] ..
first[v] + count[v] - 1): the seconds / slot0 / counts of ops.proposals.bottom_up_proposals_packed as they are, or a compact
tensor with first = cumsum.  Ground truth: gt [sum G, 2] float64, gt_label [sum G] int32, gt_offsets V + 1 host ints.
Not provided (they stay with the reference's SSNDataSet on the DataLoader workers): the random draws of training,
parse_directory's file-system scan, annotation parsing."""
import ctypes as C

import numpy as np
import torch

from ssn_b200 import _lib
from ssn_b200._lib import lib, check

RECALL_THRESHOLDS = (0.5, 0.7, 0.8999999999999999)       # np.arange(0.5, 1, 0.2), gen_bottom_up_proposals.py:170


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cuda(t, dtype, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: libssn_b200 has no CPU path" % what)
    return t.to(dtype).contiguous()


def _dev_of(t, what="boxes"):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: libssn_b200 has no CPU path" % what)
    return t.device


def _on(dev, x, dtype):
    """a host sequence / numpy array / tensor as a contiguous device tensor"""
    if torch.is_tensor(x):
        return x.to(device=dev, dtype=dtype).contiguous()
    return torch.as_tensor(np.asarray(x), dtype=dtype).to(dev).contiguous()


_SCRATCH = {}


def _p(t):
    """data pointer of an input; an empty tensor has none, and the library refuses NULL, so it gets a scratch address"""
    if t.numel():
        return t.data_ptr()
    if t.device not in _SCRATCH:
        _SCRATCH[t.device] = torch.zeros(64, dtype=torch.uint8, device=t.device)
    return _SCRATCH[t.device].data_ptr()


def _offsets(gt_offsets):
    off = [int(o) for o in (gt_offsets.tolist() if hasattr(gt_offsets, "tolist") else gt_offsets)]
    return off, (C.c_int64 * len(off))(*off)


def _empty(dev, n, dtype, width=None):
    return torch.empty((max(n, 1),) if width is None else (max(n, 1), width), dtype=dtype, device=dev)


def compact_layout(counts, device):
    """first / count tensors of a compact [sum N, 2] box tensor from V host counts"""
    c = np.asarray(counts, np.int64).reshape(-1)
    first = np.concatenate([[0], np.cumsum(c)[:-1]]) if len(c) else c
    return torch.as_tensor(first, dtype=torch.int64).to(device), torch.as_tensor(c, dtype=torch.int32).to(device)


def name_proposals_packed(boxes, first, count, gt, gt_label, gt_offsets, thresh=0.0, max_count=None):
    """-> dict(label int32 [rows], max_overlap, overlap_self float64 [rows] at the rows' own indices; gt_best float64 [sum G])."""
    dev = _dev_of(boxes)
    boxes, first, count = _cuda(boxes, torch.float64, "boxes"), _cuda(first, torch.int64, "first"), _cuda(count, torch.int32, "count")
    off, off_c = _offsets(gt_offsets)
    V, rows = len(off) - 1, boxes.shape[0]
    if first.numel() != V or count.numel() != V:
        raise ValueError("need V first / count entries and V + 1 gt_offsets")
    gt, gt_label, off_dev = _on(dev, gt, torch.float64).reshape(-1, 2), _on(dev, gt_label, torch.int32), _on(dev, off, torch.int64)
    out = {"label": _empty(dev, rows, torch.int32), "max_overlap": _empty(dev, rows, torch.float64),
           "overlap_self": _empty(dev, rows, torch.float64), "gt_best": _empty(dev, off[-1], torch.float64)}
    with torch.cuda.device(dev):
        check(lib.ssnb_name_proposals(_p(boxes), first.data_ptr(), count.data_ptr(), V, rows if max_count is None else int(max_count),
                                      _p(gt), _p(gt_label), off_c, off_dev.data_ptr(), float(thresh), out["label"].data_ptr(),
                                      out["max_overlap"].data_ptr(), out["overlap_self"].data_ptr(), out["gt_best"].data_ptr(), _stream()),
              None, "name_proposals")
    out = {k: v[:rows] for k, v in out.items() if k != "gt_best"} | {"gt_best": out["gt_best"][:off[-1]]}
    return out


def proposal_recall(gt_best, gt_offsets, thresholds=RECALL_THRESHOLDS):
    """-> dict(hits int32 [V, n_thr], totals int64 [2 n_thr + 1]) on the device: per threshold the videos with every instance
    recalled, per threshold the recalled instances, then the instances.  recall_report() turns them into the printed numbers."""
    dev = _dev_of(gt_best, "gt_best")
    gt_best = _cuda(gt_best, torch.float64, "gt_best")
    off, off_c = _offsets(gt_offsets)
    V, n = len(off) - 1, len(thresholds)
    off_dev = _on(dev, off, torch.int64)
    hits, totals = _empty(dev, V * n, torch.int32), torch.empty(2 * n + 1, dtype=torch.int64, device=dev)
    thr = (C.c_double * n)(*[float(t) for t in thresholds])
    with torch.cuda.device(dev):
        check(lib.ssnb_proposal_recall(_p(gt_best), off_c, off_dev.data_ptr(), V, thr, n, hits.data_ptr(), totals.data_ptr(), _stream()),
              None, "proposal_recall")
    return {"hits": hits[:V * n].view(V, n), "totals": totals, "thresholds": [float(t) for t in thresholds], "videos": V}


def recall_report(recall, count=None):
    """The numbers gen_bottom_up_proposals.py:169-176 prints, from one small device-to-host copy: per_video / per_instance
    recall per threshold (the reference's two divisions, in its order), their means, and the average number of proposals."""
    n = len(recall["thresholds"])
    t = recall["totals"].cpu().numpy()
    with np.errstate(all="ignore"):
        pv = np.array([t[k] / float(recall["videos"]) for k in range(n)])
        pi = np.array([t[n + k] / float(t[2 * n]) for k in range(n)])
    out = {"per_video": pv, "per_instance": pi, "average": np.mean(np.stack([pv, pi], 1), axis=0), "ground_truth": int(t[2 * n])}
    if count is not None:
        out["average_proposals"] = float(np.mean(count.cpu().numpy())) if count.numel() else float("nan")
    return out


def sliding_window_proposals(durations, time_step=1, max_level=8, overlap=0.4, capacity=None):
    """gen_exponential_sw_proposal for V videos.  durations: V seconds (a host sequence, or a CUDA float64 tensor together with
    `capacity`, a bound of the total number of windows).  -> dict(boxes [total bound, 2], first, count, level_count [V, levels],
    total int64 [1]) on the device; the boxes are compact (first = cumsum), level-major and start-ascending per video."""
    if max_level < 1 or max_level > 32:
        raise ValueError("max_level must be 1..32")
    spans = [float(2 ** x) for x in range(max_level)]
    steps = [float(int(np.ceil(2 ** x * time_step * (1 - overlap)))) for x in range(max_level)]     # per call, not per video
    if torch.is_tensor(durations):
        dev = _dev_of(durations, "durations")
        if capacity is None:
            raise ValueError("a device tensor of durations needs `capacity` (the call does not synchronise to size its output)")
        d, V, per_video = _cuda(durations, torch.float64, "durations"), durations.numel(), int(capacity)
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
        host = np.asarray(durations, np.float64).reshape(-1)
        V = len(host)
        bound = [sum(int(np.ceil(x / s)) for s in steps if s >= 1) if np.isfinite(x) and x > 0 else 0 for x in host]
        per_video = max(bound) if V else 0
        capacity = sum(bound) if capacity is None else int(capacity)
        d = torch.as_tensor(host).to(dev)
    out = {"boxes": _empty(dev, capacity, torch.float64, 2), "first": _empty(dev, V, torch.int64), "count": _empty(dev, V, torch.int32),
           "level_count": _empty(dev, V * max_level, torch.int32), "total": torch.zeros(1, dtype=torch.int64, device=dev)}
    with torch.cuda.device(dev):
        check(lib.ssnb_sliding_windows(_p(d), V, (C.c_double * max_level)(*spans), (C.c_double * max_level)(*steps), max_level,
                                       per_video, int(capacity), out["boxes"].data_ptr(), out["first"].data_ptr(), out["count"].data_ptr(),
                                       out["level_count"].data_ptr(), out["total"].data_ptr(), _stream()), None, "sliding_windows")
    out.update(boxes=out["boxes"][:capacity], first=out["first"][:V], count=out["count"][:V],
               level_count=out["level_count"][:V * max_level].view(V, max_level))
    return out


_MODES = {"seconds": _lib.PROPFRAMES_SECONDS, "normalised": _lib.PROPFRAMES_NORMALISED, "frames": _lib.PROPFRAMES_AS_GIVEN}


def proposal_frames(boxes, first, count, frame_cnts, durations=None, mode="seconds", max_count=None):
    """-> dict(frames int64 [rows, 2] as a list file holds them, keep bool [rows], valid int64 [rows, 2] (end clipped to the
    frame count), coverage float64 [rows]).  mode: "seconds" (needs durations), "normalised" or "frames"."""
    dev = _dev_of(boxes)
    boxes, first, count = _cuda(boxes, torch.float64, "boxes"), _cuda(first, torch.int64, "first"), _cuda(count, torch.int32, "count")
    V, rows = first.numel(), boxes.shape[0]
    fc = _on(dev, frame_cnts, torch.int32)
    dur = None if durations is None else _on(dev, durations, torch.float64)
    if fc.numel() != V or count.numel() != V or (dur is not None and dur.numel() != V):
        raise ValueError("need V first / count / frame_cnts / durations")
    if mode not in _MODES:
        raise ValueError("mode must be one of %s" % sorted(_MODES))
    out = {"frames": _empty(dev, rows, torch.int64, 2), "valid": _empty(dev, rows, torch.int64, 2),
           "coverage": _empty(dev, rows, torch.float64), "keep": _empty(dev, rows, torch.uint8)}
    with torch.cuda.device(dev):
        check(lib.ssnb_proposal_frames(_p(boxes), first.data_ptr(), count.data_ptr(), V, rows if max_count is None else int(max_count),
                                       None if dur is None else dur.data_ptr(), fc.data_ptr(), _MODES[mode], out["frames"].data_ptr(),
                                       out["valid"].data_ptr(), out["coverage"].data_ptr(), out["keep"].data_ptr(), _stream()),
              None, "proposal_frames")
    return {k: v[:rows] for k, v in out.items()}


def proposal_targets(frames, best_iou, overlap_self, coverage, first, count, gt_frames, gt_offsets, fg_iou_thresh=0.7,
                     incomplete_iou_thresh=0.3, bg_iou_thresh=0.01, bg_coverage_thresh=0.02, incomplete_overlap_thresh=0.7,
                     exclude_empty=True):
    """Kept rows (record_rows) -> dict(tags uint8 [rows] (bits TAG_FG / TAG_INCOMPLETE / TAG_BACKGROUND), reg float64 [rows, 2],
    pool_counts int32 [V, 4] (fg, incomplete, background, ground truth), totals int64 [5] (their sums, videos used),
    reg_stats float64 [2, 2] ((mean loc, mean size), (std loc, std size)): SSNDataSet's `stats`)."""
    dev = _dev_of(frames, "frames")
    frames, first, count = _cuda(frames, torch.int64, "frames"), _cuda(first, torch.int64, "first"), _cuda(count, torch.int32, "count")
    iou, osf, cov = (_cuda(t, torch.float64, n) for t, n in ((best_iou, "best_iou"), (overlap_self, "overlap_self"), (coverage, "coverage")))
    off, off_c = _offsets(gt_offsets)
    V, rows = len(off) - 1, frames.shape[0]
    if first.numel() != V or count.numel() != V or min(iou.numel(), osf.numel(), cov.numel()) < rows:
        raise ValueError("need V first / count entries, V + 1 gt_offsets and one best_iou / overlap_self / coverage per row")
    gtf, off_dev = _on(dev, gt_frames, torch.int64).reshape(-1, 2), _on(dev, off, torch.int64)
    cfg = _lib.ProposalTargetsCfg(float(fg_iou_thresh), float(incomplete_iou_thresh), float(bg_iou_thresh), float(bg_coverage_thresh),
                                  float(incomplete_overlap_thresh), int(bool(exclude_empty)), 0)
    ws_bytes = lib.ssnb_proposal_targets_workspace_bytes(V)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    out = {"tags": _empty(dev, rows, torch.uint8), "reg": _empty(dev, rows, torch.float64, 2), "pool_counts": _empty(dev, V, torch.int32, 4),
           "totals": torch.empty(5, dtype=torch.int64, device=dev), "reg_stats": torch.empty(2, 2, dtype=torch.float64, device=dev)}
    with torch.cuda.device(dev):
        check(lib.ssnb_proposal_targets(C.byref(cfg), _p(frames), _p(iou), _p(osf), _p(cov), first.data_ptr(),
                                        count.data_ptr(), V, _p(gtf), off_c, off_dev.data_ptr(), out["tags"].data_ptr(),
                                        out["reg"].data_ptr(), out["pool_counts"].data_ptr(), out["totals"].data_ptr(),
                                        out["reg_stats"].data_ptr(), ws.data_ptr(), ws_bytes, _stream()), None, "proposal_targets")
    out.update(tags=out["tags"][:rows], reg=out["reg"][:rows], pool_counts=out["pool_counts"][:V])
    return out


def test_proposals(frames, counts, frame_cnts, new_length=1, test_interval=6):
    """get_test_data's proposal half for V videos.  frames: compact kept valid frames int64 [sum N, 2] (CUDA); counts: V host
    ints.  A video without proposals gets the reference's fallback row (0, frame_cnt - 1).  -> dict(num_ticks int32 [V],
    rel_prop float64 [R, 2], proposal_ticks int64 [R, 4], scaling float64 [R, 2] as the reference returns them, ticks32 int32 /
    scaling32 float32 as ssnb_stpp_reorg_prefix takes them, offsets: V + 1 host row offsets into those R rows)."""
    dev = _dev_of(frames, "frames")
    frames = _cuda(frames, torch.int64, "frames")
    c = np.asarray(counts, np.int64).reshape(-1)
    V = len(c)
    if int(c.sum()) != frames.shape[0] or (c < 0).any():
        raise ValueError("counts must be non-negative and sum to the rows of frames")
    first, count = compact_layout(c, dev)
    offsets = np.concatenate([[0], np.cumsum(np.maximum(c, 1))]).astype(np.int64)
    R = int(offsets[-1])
    out_first, fc = torch.as_tensor(offsets[:-1]).to(dev), _on(dev, frame_cnts, torch.int32)
    if fc.numel() != V:
        raise ValueError("need V frame_cnts")
    out = {"num_ticks": _empty(dev, V, torch.int32), "rel_prop": _empty(dev, R, torch.float64, 2), "proposal_ticks": _empty(dev, R, torch.int64, 4),
           "scaling": _empty(dev, R, torch.float64, 2), "ticks32": _empty(dev, R, torch.int32, 4), "scaling32": _empty(dev, R, torch.float32, 2)}
    with torch.cuda.device(dev):
        check(lib.ssnb_test_proposals(_p(frames), first.data_ptr(), count.data_ptr(), out_first.data_ptr(), V, int(c.max()) if V else 0,
                                      fc.data_ptr(), int(new_length), int(test_interval), out["num_ticks"].data_ptr(), out["rel_prop"].data_ptr(),
                                      out["proposal_ticks"].data_ptr(), out["scaling"].data_ptr(), out["ticks32"].data_ptr(),
                                      out["scaling32"].data_ptr(), _stream()), None, "test_proposals")
    out = {k: v[:(V if k == "num_ticks" else R)] for k, v in out.items()}
    out["offsets"] = offsets.tolist()
    return out


test_proposals.__test__ = False      # not a pytest test


def _as_packed(props):
    """a bottom_up_proposals_packed result, a dict(boxes, first, count) or a list of per-video CUDA [n, 2] tensors -> packed"""
    if isinstance(props, dict) and "seconds" in props:
        dev = props["seconds"].device
        return props["seconds"], props["slot0"].to(dev), props["counts"]
    if isinstance(props, dict):
        return props["boxes"], props["first"], props["count"]
    for t in props:
        _dev_of(t)
    if not len(props):
        raise ValueError("no videos")
    first, count = compact_layout([t.shape[0] for t in props], props[0].device)
    return torch.cat([t.double().reshape(-1, 2) for t in props]), first, count


def label_proposals(props, gt, gt_label, gt_offsets, durations, frame_cnts, iou_thresholds=RECALL_THRESHOLDS, thresh=0.0):
    """gen_bottom_up_proposals.py:158-193 after the boxes exist: name every proposal, the recall table, frame windows of the
    proposals and the ground truth.  props: see _as_packed (a TAG result is read in its slot layout, on the device).  gt
    [sum G, 2] seconds and gt_label [sum G] packed by the V + 1 host gt_offsets.  Nothing is copied to the host; pass the
    result to recall_report / format_proposal_list for that.  -> dict(boxes, first, count, label, max_overlap, overlap_self,
    gt_best, recall, frames, gt, gt_label, gt_offsets, gt_frames, frame_cnt, duration)."""
    boxes, first, count = _as_packed(props)
    dev = _dev_of(boxes)
    off = [int(o) for o in gt_offsets]
    gt_d, lab_d = _on(dev, gt, torch.float64).reshape(-1, 2), _on(dev, gt_label, torch.int32)
    fc, dur = _on(dev, frame_cnts, torch.int32), _on(dev, durations, torch.float64)
    out = {"boxes": boxes, "first": first, "count": count, "gt": gt_d, "gt_label": lab_d, "gt_offsets": off, "frame_cnt": fc, "duration": dur}
    out.update(name_proposals_packed(boxes, first, count, gt_d, lab_d, off, thresh))
    out["recall"] = proposal_recall(out["gt_best"], off, iou_thresholds)
    out["frames"] = proposal_frames(boxes, first, count, fc, dur, "seconds")["frames"]
    g_first, g_count = compact_layout(np.diff(off), dev)
    out["gt_frames"] = proposal_frames(gt_d, g_first, g_count, fc, dur, "seconds", max_count=int(max(np.diff(off), default=0)))["frames"]
    return out


def _one_copy(tensors):
    """several device tensors -> numpy arrays through ONE device-to-host copy"""
    flat = [t.contiguous().view(torch.uint8).reshape(-1) for t in tensors]
    host = torch.cat(flat).cpu().numpy()
    out, at = [], 0
    for t, f in zip(tensors, flat):
        out.append(host[at:at + f.numel()].view(np.dtype(str(t.dtype).replace("torch.", ""))).reshape(tuple(t.shape)))
        at += f.numel()
    return out


def format_proposal_list(result, frame_dirs, style="dump"):
    """The text of a proposal list, one block per video.  result: label_proposals' dict (or any dict with first, count, label,
    max_overlap, overlap_self, frames, gt_label, gt_offsets, gt_frames, frame_cnt).  frame_dirs: the V frame directories the
    list names (dump_window_list globs them for the frame count; here frame_cnt is an argument).
      style="dump"       dump_window_list (ops/io.py:95-134) under '# i' headers from 1 (gen_bottom_up_proposals.py:188-191);
                         ground-truth labels are written + 1
      style="processed"  process_proposal_list's blocks (ops/io.py:49-59): headers from 0, labels as given
    The kept rows are gathered on the device and reach the host in one copy; the '%.4f' formatting is Python's."""
    first, count = result["first"], result["count"]
    dev = count.device
    c64 = count.to(torch.int64)
    total = int(c64.sum())                                   # sizes the gather
    start = torch.cumsum(c64, 0) - c64
    idx = torch.repeat_interleave(first.to(dev) - start, c64, output_size=total) + torch.arange(total, device=dev)
    cols = [result[k].index_select(0, idx) for k in ("label", "max_overlap", "overlap_self", "frames")]
    label, mo, ms, frames, cnt, gl, gf, fc = _one_copy(cols + [count, result["gt_label"], result["gt_frames"], result["frame_cnt"]])
    off, blocks, at = result["gt_offsets"], [], 0
    if len(frame_dirs) != len(cnt):
        raise ValueError("need one frame directory per video")
    add = 1 if style == "dump" else 0
    for v, n in enumerate(cnt.tolist()):
        gts = ["{} {} {}".format(int(gl[j]) + add, int(gf[j, 0]), int(gf[j, 1])) for j in range(off[v], off[v + 1])]
        prs = ["{} {:.04f} {:.04f} {} {}".format(int(label[i]), float(mo[i]), float(ms[i]), int(frames[i, 0]), int(frames[i, 1]))
               for i in range(at, at + n)]
        at += n
        gt_txt = "\n".join(gts) + ("\n" if gts else "")
        if style == "dump":
            blocks.append("# {}\n{}\n{}\n1\n{}\n{}{}\n{}\n".format(v + 1, frame_dirs[v], int(fc[v]), len(gts), gt_txt, len(prs), "\n".join(prs)))
        else:
            blocks.append("# {}\n{}\n{}\n1\n{}\n{}{}\n{}".format(v, frame_dirs[v], int(fc[v]), len(gts), gt_txt, len(prs),
                                                               "\n".join(prs) + ("\n" if prs else "")))
    return "".join(blocks)


def write_proposal_list(path, result, frame_dirs, style="dump"):
    text = format_proposal_list(result, frame_dirs, style)
    with open(path, "w") as f:
        f.write(text)
    return text


def load_proposal_list(path, device="cuda"):
    """load_proposal_file (ops/io.py:7-31) into the packed layout on `device`: dict(ids, frame_cnt int32 [V] (int(float(line 2)
    * float(line 3)): 1 for a normalised list), boxes float64 [sum N, 2] (columns 4-5: frames, or fractions in a normalised
    list), label, max_overlap, overlap_self (columns 1-3), first, count, counts (host), gt float64 [sum G, 2], gt_label,
    gt_offsets (host)).  Labels are the file's (ground truth already + 1 in a dumped list)."""
    from itertools import groupby
    ids, fcs, counts, off, gt, pr = [], [], [], [0], [], []
    with open(path) as f:
        for k, g in groupby(f, lambda x: x.startswith("#")):
            if k:
                continue
            info = [x.strip() for x in g]
            n_gt = int(info[3])
            n_pr = int(info[4 + n_gt])
            ids.append(info[0])
            fcs.append(int(float(info[1]) * float(info[2])))
            gt += [x.split() for x in info[4:4 + n_gt]]
            pr += [x.split() for x in info[5 + n_gt:5 + n_gt + n_pr]]
            counts.append(n_pr)
            off.append(off[-1] + n_gt)
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("load_proposal_list fills CUDA tensors: libssn_b200 has no CPU path")
    g = np.array([[float(c) for c in r[:3]] for r in gt], np.float64).reshape(-1, 3)
    p = np.array([[float(c) for c in r[:5]] for r in pr], np.float64).reshape(-1, 5)
    first, count = compact_layout(counts, dev)
    T = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to(dev).to(dt)
    return {"ids": ids, "frame_cnt": T(np.array(fcs, np.int32), torch.int32), "boxes": T(p[:, 3:5], torch.float64), "label": T(p[:, 0], torch.int32),
            "max_overlap": T(p[:, 1], torch.float64), "overlap_self": T(p[:, 2], torch.float64), "first": first, "count": count, "counts": counts,
            "gt": T(g[:, 1:3], torch.float64), "gt_label": T(g[:, 0], torch.int32), "gt_offsets": off}


def record_rows(loaded, frame_cnts=None, mode="frames"):
    """SSNVideoRecord (ssn_dataset.py:74-93) of every video of a loaded list: frame windows (mode "frames" for a dumped /
    processed list, "normalised" with frame_cnts for a shipped normalised list), then the kept rows compacted (one host
    synchronisation for the kept counts).  -> dict(frames (valid), best_iou, overlap_self, coverage, label, first, count, counts,
    gt_frames, gt_label, gt_offsets, frame_cnt): what proposal_targets and test_proposals take."""
    dev = loaded["boxes"].device
    fc = loaded["frame_cnt"] if frame_cnts is None else _on(dev, frame_cnts, torch.int32)
    V = fc.numel()
    p = proposal_frames(loaded["boxes"], loaded["first"], loaded["count"], fc, None, mode, max_count=max(loaded["counts"], default=0))
    g_n = np.diff(loaded["gt_offsets"])
    g_first, g_count = compact_layout(g_n, dev)
    g = proposal_frames(loaded["gt"], g_first, g_count, fc, None, mode, max_count=int(max(g_n, default=0)))
    keep, gkeep = p["keep"].bool(), g["keep"].bool()
    vid = torch.repeat_interleave(torch.arange(V, device=dev), loaded["count"].long(), output_size=int(sum(loaded["counts"])))
    gvid = torch.repeat_interleave(torch.arange(V, device=dev), g_count.long(), output_size=int(g_n.sum()))
    counts = torch.bincount(vid[keep], minlength=V).cpu().numpy()
    g_counts = torch.bincount(gvid[gkeep], minlength=V).cpu().numpy()
    first, count = compact_layout(counts, dev)
    return {"frames": p["valid"][keep], "coverage": p["coverage"][keep], "best_iou": loaded["max_overlap"][keep],
            "overlap_self": loaded["overlap_self"][keep], "label": loaded["label"][keep], "first": first, "count": count,
            "counts": counts.tolist(), "gt_frames": g["valid"][gkeep], "gt_label": loaded["gt_label"][gkeep],
            "gt_offsets": np.concatenate([[0], np.cumsum(g_counts)]).astype(np.int64).tolist(), "frame_cnt": fc}
