"""Video-level class scores from snippet scores on the GPU: the reference's ops/video_funcs.py, with the same names and
signatures per video, and packed calls over many ragged videos (csrc/video_agg.cu, ssnb_video_aggregate / ssnb_video_fuse).

  default_aggregation_func / top_k_aggregation_func / sliding_window_aggregation_func / tpp_aggregation_func /
  default_fusion_func     one video, as the reference: numpy in -> numpy out (run on the current CUDA device), CUDA tensor in
                          -> CUDA tensor out
  aggregate_packed        scores [sum T, crops, D] with tick offsets [V+1] -> [V, K] on the device, one call
  fuse_packed             default_fusion_func over [V, K] streams on the device

The scores are fp32 (what BinaryClassifier.test_forward or a backbone with a linear head gives): a float64 array is refused
rather than computed at another precision than the reference would.  Every fp32 sum runs in numpy's order and each operation
is rounded as numpy rounds it, so the aggregates are bitwise numpy's without normalisation; the softmax's exp is CUDA's expf,
within a few ulp of numpy's.  tpp returns float64, as the reference's np.zeros accumulator does.

Differences from the reference, on purpose: crop_agg takes np.mean / np.max (or 'mean' / 'max'), not any callable; fps and
spans are integers; a video needs at least one tick; default_fusion_func does not add into major_score in place (the reference
updates the caller's array); fusion weights are applied as fp32, which is what numpy does for Python float weights."""
import ctypes as C

import numpy as np
import torch

from ssn_b200._lib import lib, check
from ops.proposal_lists import _stream

MODES = {"default": 0, "top_k": 1, "sliding_window": 2, "tpp": 3}
CROP_AGG = {"mean": 0, "max": 1}


def _crop_agg(crop_agg):
    if crop_agg is None or crop_agg is np.mean or crop_agg == "mean":
        return CROP_AGG["mean"]
    if crop_agg is np.max or crop_agg is np.amax or crop_agg == "max":
        return CROP_AGG["max"]
    raise ValueError("crop_agg must be np.mean or np.max (or 'mean' / 'max')")


def _fp32_on_device(x, what):
    """-> (fp32 contiguous CUDA tensor, was_numpy)"""
    if torch.is_tensor(x):
        if not x.is_cuda:
            raise RuntimeError("%s must be a numpy array or a CUDA tensor: libssn_b200 has no CPU path" % what)
        if x.dtype != torch.float32:
            raise TypeError("%s must be float32, not %s" % (what, x.dtype))
        return x.contiguous(), False
    a = np.asarray(x)
    if a.dtype != np.float32:
        raise TypeError("%s must be float32, not %s" % (what, a.dtype))
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", torch.cuda.current_device())), True


def aggregate_packed(scores, offsets, mode="default", crop_agg=None, normalization=True, k=None, spans=(1, 2, 4, 8, 16),
                     overlap=0.2, fps=1, num_class=None):
    """scores: CUDA fp32 [sum T, crops, D] (or [sum T, D]: one crop); offsets: host int64 [V+1], video v's ticks at
    offsets[v] .. offsets[v+1].  mode: 'default' | 'top_k' (k) | 'sliding_window' (spans, overlap, fps; crop mean) | 'tpp'
    (num_class; crop mean, no normalisation).  -> device [V, K]: fp32, float64 for tpp.  Nothing waits for the device."""
    if not torch.is_tensor(scores) or not scores.is_cuda:
        raise RuntimeError("scores must be a CUDA tensor: libssn_b200 has no CPU path")
    if scores.dtype != torch.float32:
        raise TypeError("scores must be float32, not %s" % scores.dtype)
    if scores.dim() == 2:
        scores = scores.unsqueeze(1)
    if scores.dim() != 3:
        raise ValueError("scores must be [sum T, crops, D]")
    if mode not in MODES:
        raise ValueError("mode must be one of %s" % sorted(MODES))
    scores = scores.contiguous()
    dev = scores.device
    off = np.ascontiguousarray(np.asarray(offsets, dtype=np.int64).reshape(-1))
    V = len(off) - 1
    if V < 1 or off[-1] != scores.shape[0]:
        raise ValueError("offsets must be [V+1] with offsets[-1] == scores.shape[0]")
    _, crops, D = scores.shape
    m, ca = MODES[mode], _crop_agg(crop_agg)
    norm = int(bool(normalization)) if mode != "tpp" else 0
    sp = np.ascontiguousarray(np.asarray(spans, dtype=np.int32).reshape(-1)) if mode == "sliding_window" else np.zeros(1, np.int32)
    if mode == "sliding_window" and not np.array_equal(sp, np.asarray(spans).reshape(-1)):
        raise ValueError("spans must be integers")
    if mode == "sliding_window" and int(fps) != fps:
        raise ValueError("fps must be an integer")
    topk = int(k) if mode == "top_k" else 1
    K = int(num_class) if mode == "tpp" else D
    args = (off.ctypes.data_as(C.POINTER(C.c_int64)), V, crops, D, m, ca, topk, sp.ctypes.data_as(C.POINTER(C.c_int)),
            len(sp) if mode == "sliding_window" else 0, float(overlap), int(fps), K)
    ws_bytes = lib.ssnb_video_aggregate_workspace_bytes(*args)        # 0 for arguments the call rejects
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    out = torch.empty((V, K), dtype=torch.float64 if mode == "tpp" else torch.float32, device=dev)
    off_dev = torch.from_numpy(off).to(dev)
    with torch.cuda.device(dev):
        check(lib.ssnb_video_aggregate(scores.data_ptr(), args[0], off_dev.data_ptr(), V, crops, D, m, ca, norm, topk, args[7], args[8],
                                       float(overlap), int(fps), K, out.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), None,
              "video_aggregate")
    return out


def _one_video(score, mode, **kw):
    s, was_numpy = _fp32_on_device(score, "score")
    if s.dim() != 3:
        raise ValueError("score must be [ticks, crops, classes]")
    out = aggregate_packed(s, [0, s.shape[0]], mode, **kw)[0]
    return out.cpu().numpy() if was_numpy else out


def default_aggregation_func(score_arr, normalization=True, crop_agg=None):
    """video_funcs.py:8-18: crop reduction (np.mean or np.max), the mean over ticks, optionally the softmax."""
    return _one_video(score_arr, "default", normalization=normalization, crop_agg=crop_agg)


def top_k_aggregation_func(score_arr, k, normalization=True, crop_agg=None):
    """video_funcs.py:21-26: crop reduction, the mean of each class's k largest ticks (all ticks when k > T)."""
    return _one_video(score_arr, "top_k", normalization=normalization, crop_agg=crop_agg, k=k)


def sliding_window_aggregation_func(score, spans=[1, 2, 4, 8, 16], overlap=0.2, norm=True, fps=1):
    """video_funcs.py:29-57, the ActivityNet 2016 rule: crop mean; per span the window maxima, the mean of the
    max(15, n_windows // 4) largest; the mean over spans; optionally the softmax."""
    return _one_video(score, "sliding_window", normalization=norm, spans=spans, overlap=overlap, fps=fps)


def tpp_aggregation_func(score, num_class):
    """video_funcs.py:60-70: crop mean; tick t reads stage int(t * stage / T) of the stage * num_class columns; float64."""
    return _one_video(score, "tpp", num_class=num_class)


def fuse_packed(major, others, weights, norm=True):
    """default_fusion_func over CUDA fp32 [V, K] streams: major + sum of others[i] * weights[i] in stream order, optionally
    the row softmax.  -> a new device tensor [V, K] (major is left as it is)."""
    if not torch.is_tensor(major) or not major.is_cuda or major.dtype != torch.float32:
        raise TypeError("major must be a float32 CUDA tensor")
    others = list(others)
    weights = [float(w) for w in weights]
    if len(others) != len(weights):
        raise ValueError("one weight per other stream")
    if len(others) > 8:
        raise ValueError("at most 8 other streams")
    major = major.contiguous()
    K = major.shape[-1] if major.dim() else 1
    rows = major.numel() // max(K, 1)
    oth = []
    for o in others:
        if not torch.is_tensor(o) or o.device != major.device or o.dtype != torch.float32 or o.shape != major.shape:
            raise ValueError("every stream must be a float32 tensor of major's shape on its device")
        oth.append(o.contiguous())
    out = torch.empty_like(major)
    ptrs = (C.c_void_p * max(len(oth), 1))(*[o.data_ptr() for o in oth])
    w = (C.c_double * max(len(weights), 1))(*weights)
    with torch.cuda.device(major.device):
        check(lib.ssnb_video_fuse(major.data_ptr(), ptrs, w, len(oth), rows, K, int(bool(norm)), 1.0, out.data_ptr(), _stream()), None,
              "video_fuse")
    return out


def default_fusion_func(major_score, other_scores, fusion_weights, norm=True):
    """video_funcs.py:73-80 for one video's (or a [V, K] batch of) scores."""
    assert len(other_scores) == len(fusion_weights)
    m, was_numpy = _fp32_on_device(major_score, "major_score")
    out = fuse_packed(m, [_fp32_on_device(s, "other score")[0] for s in other_scores], fusion_weights, norm)
    return out.cpu().numpy() if was_numpy else out
