"""TAG bottom-up proposals on the GPU — gen_bottom_up_proposals.py:76-142 of the reference (score merge, then gen_prop
with ops/sequence_funcs.py's label_frame_by_threshold / build_box_by_search / temporal_nms), for many videos in one call
of libssn_b200.so (csrc/proposals.cu) instead of numpy loops in a process pool.  Scores are CUDA tensors; there is no CPU
path.

Deliberate differences from the reference:
  - gen_prop returns the scores of all NMS survivors next to the boxes that pass the minimum-length filter, so the two lists
    disagree once minimum_len > 0; here every returned box comes with its own score.
  - numpy's argsort leaves the order of tied scores open; here tied boxes stay in the order the search emitted them.
  - a box whose score is NaN (a NaN or +inf and -inf inside its window) ranks first, as the reference's
    argsort()[::-1] puts NaN first; among themselves NaN-scored boxes keep the search order too, whatever the NaN's sign
    (numpy's order among several NaNs is not a rule).
  - the regression branch (:130-132, which calls the undefined regress_box) is not provided.
"""
import collections
import ctypes as C

import torch

from ssn_b200._lib import lib, check, TagProposalsCfg

THRESHOLDS = (0.01, 0.05, 0.1, .15, 0.25, .4, .5, .6, .7, .8, .9, .95)      # gen_bottom_up_proposals.py:124
TOLERANCES = (0.05, .1, .2, .3, .4, .5, .6, 0.8, 1.0)                      # gen_bottom_up_proposals.py:127

# one video's proposals: pr_box [n, 2] float64 seconds and scores [n] float32 (gen_prop's pr_box and scores), frames [n, 2]
# int32 (start, end frame), all in NMS order on the scores' device
Proposals = collections.namedtuple("Proposals", ["pr_box", "scores", "frames"])


def merge_scores(streams, weights=None):
    """gen_bottom_up_proposals.py:76-91 for one video: streams are [T_i, crops, K] score tensors (RGB, Flow, ...) ->
    the merged [T, K] fp32 crop mean.  A shorter stream truncates the result; a longer one is resampled at int(x * tick),
    tick = T_i / float(T)."""
    out = streams[0].float().mean(1) * (1.0 if weights is None else float(weights[0]))
    for i in range(1, len(streams)):
        add = streams[i].float().mean(1)
        if add.shape[0] < out.shape[0]:
            out = out[:add.shape[0]]
        elif add.shape[0] > out.shape[0]:
            tick = add.shape[0] / float(out.shape[0])
            idx = torch.tensor([int(x * tick) for x in range(out.shape[0])], dtype=torch.long, device=add.device)
            add = add[idx]
        out = out + add * (1.0 if weights is None else float(weights[i]))
    return out


def _double_array(seq):
    return (C.c_double * len(seq))(*[float(x) for x in seq])


def bottom_up_proposals_packed(f_score, offsets, durations, cls=0, bw=3, thresholds=THRESHOLDS, tolerances=TOLERANCES,
                               nms_threshold=0.9, minimum_len=0.0, trace=False):
    """Every video of a packed score in one library call.  f_score: CUDA [sum T_v, K]; offsets: V + 1 ints (video v is rows
    offsets[v]:offsets[v+1]); durations: V seconds.  -> dict of device tensors in the library's slot layout:
    frames [slots, 2], scores [slots], seconds [slots, 2], counts [V], slot0 [V] (video v's boxes are rows slot0[v] ..
    slot0[v] + counts[v] - 1), and with trace=True also smoothed [sum T], labels [sum T] (bit k: threshold k),
    raw_frames / raw_scores / raw_counts (the boxes before NMS in the reference's order)."""
    if not f_score.is_cuda:
        raise RuntimeError("f_score must be a CUDA tensor: libssn_b200 has no CPU path")
    if f_score.dim() != 2:
        raise ValueError("f_score must be [sum T, K]")
    offsets = [int(o) for o in offsets]
    V = len(offsets) - 1
    if V < 0 or len(durations) != V:
        raise ValueError("need V + 1 offsets and V durations")
    dev = f_score.device
    f = f_score.contiguous().float()
    N = offsets[-1] if V else 0
    if N != f.shape[0]:
        raise ValueError("offsets[-1] = %d but f_score has %d rows" % (N, f.shape[0]))
    n_thr, n_tol = len(thresholds), len(tolerances)
    sigma = 0.0 if bw is None else float(bw)
    thr_c, tol_c = _double_array(thresholds), _double_array(tolerances)
    cfg = TagProposalsCfg(int(cls), n_thr, n_tol, 0, sigma, float(nms_threshold), float(minimum_len), thr_c, tol_c)
    slots = n_thr * n_tol * (N + V)
    ws_bytes = lib.ssnb_tag_proposals_workspace_bytes(V, N, n_thr, n_tol)    # 0 for arguments the call below rejects
    i32, f32, f64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev), dict(dtype=torch.float64, device=dev)
    out = {"frames": torch.empty(max(slots, 1), 2, **i32), "scores": torch.empty(max(slots, 1), **f32),
           "seconds": torch.empty(max(slots, 1), 2, **f64), "counts": torch.zeros(max(V, 1), **i32)}
    if trace:
        out.update({"smoothed": torch.empty(max(N, 1), **f32), "labels": torch.empty(max(N, 1), **i32),
                    "raw_frames": torch.empty(max(slots, 1), 2, **i32), "raw_scores": torch.empty(max(slots, 1), **f32),
                    "raw_counts": torch.zeros(max(V, 1), **i32)})
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    offs = (C.c_int64 * (V + 1))(*offsets)
    offs_dev = torch.tensor(offsets, dtype=torch.int64, device=dev)
    durs_dev = torch.tensor([float(d) for d in durations], dtype=torch.float64, device=dev)

    def ptr(k):
        return out[k].data_ptr() if k in out else None
    with torch.cuda.device(dev):
        check(lib.ssnb_tag_proposals(C.byref(cfg), f.data_ptr(), f.shape[1], offs, offs_dev.data_ptr(), V, durs_dev.data_ptr(),
                                     ptr("frames"), ptr("scores"),
                                     ptr("seconds"), ptr("counts"), ptr("smoothed"), ptr("labels"), ptr("raw_frames"),
                                     ptr("raw_scores"), ptr("raw_counts"), ws.data_ptr(), ws_bytes,
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "tag_proposals")
    out["counts"] = out["counts"][:V]
    if trace:
        out["raw_counts"] = out["raw_counts"][:V]
    out["slot0"] = torch.tensor([n_thr * n_tol * (offsets[v] + v) for v in range(V)], dtype=torch.int64)
    return out


def bottom_up_proposals(f_scores, durations, cls=0, bw=3, thresholds=THRESHOLDS, tolerances=TOLERANCES, nms_threshold=0.9,
                        minimum_len=0.0, offsets=None):
    """gen_prop (gen_bottom_up_proposals.py:116-142) for many videos at once.  f_scores: a list of CUDA [T_v, K] merged scores
    (merge_scores), or one packed CUDA [sum T_v, K] tensor with `offsets` (V + 1 row offsets); durations: V seconds.
    bw=None: no Gaussian smoothing.  -> list of V Proposals(pr_box, scores, frames).  The kept boxes are gathered out of the
    call's slot-sized buffers into compact tensors, so a result holds only the batch's kept boxes, not its box slots."""
    if offsets is None:
        for t in f_scores:
            if not t.is_cuda:
                raise RuntimeError("f_scores must be CUDA tensors: libssn_b200 has no CPU path")
        offsets = [0]
        for t in f_scores:
            offsets.append(offsets[-1] + t.shape[0])
        packed = torch.cat([t.float() for t in f_scores]) if len(f_scores) else None
        if packed is None:
            return []
    else:
        packed = f_scores
    r = bottom_up_proposals_packed(packed, offsets, durations, cls, bw, thresholds, tolerances, nms_threshold, minimum_len)
    counts = r["counts"].cpu()
    starts = torch.repeat_interleave(r["slot0"], counts)
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    idx = (starts + torch.arange(int(counts.sum())) - first).to(packed.device)
    seconds, scores, frames = (r[k].index_select(0, idx) for k in ("seconds", "scores", "frames"))
    n = counts.tolist()
    return [Proposals(*p) for p in zip(seconds.split(n), scores.split(n), frames.split(n))]
