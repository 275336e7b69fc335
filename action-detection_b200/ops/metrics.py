"""Video classification metrics on the GPU: the reference's ops/metrics.py, with the same names and signatures, and a packed
call over many videos (csrc/video_agg.cu, ssnb_video_metrics).  sklearn is not needed: average_precision_score and
confusion_matrix are restated in the kernels.

  softmax                                 metrics.py:8-11 over the last axis (fp32)
  top_k_acc / top_k_hit                   one video's label set against its scores
  top_3_accuracy / top_k_accuracy         over score_dict / video_list (videos missing from score_dict are skipped)
  video_mean_ap                           sklearn average_precision_score(average='macro') of the label indicator
  mean_class_accuracy                     np.argmax, confusion_matrix, mean(diag / row sum)
  video_metrics_packed                    all of them for a [V, K] device score matrix and (video, label) pairs, on the device

Tie rule: numpy's argsort is not stable, so a tie at the k-th place of np.argsort(scores)[-k:] has no portable answer.  Here
each video's classes are ranked NaN first, then by descending score (-0 equal to +0), and equal scores the HIGHER class
first, which is what a stable ascending argsort's [-k:] keeps.  numpy gives the same wherever its sort is stable (up to 16
classes without SIMD sorting).  Top-k means do not depend on the tie order, and AP does not either (tied scores form one
threshold, as in sklearn).  np.argmax picks the first maximum (the first NaN if any), as numpy does.

NaN scores: the reference's video_mean_ap raises (sklearn refuses non-finite scores); here NaN ranks first, as rank_key.cuh
orders it.  A class that is predicted but never labelled makes mean_class_accuracy NaN, as numpy's 0 / 0 does.  A class with
no positive video has AP 0 (sklearn 1.9) and counts in the macro mean."""
import ctypes as C

import numpy as np
import torch

from ssn_b200._lib import lib, check
from ops.proposal_lists import _on, _p, _stream
from ops.video_funcs import _fp32_on_device


def softmax(raw_score, T=1):
    """metrics.py:8-11: exp((x - max) * T) / sum over the last axis.  numpy in -> numpy out; CUDA tensor in -> CUDA tensor."""
    s, was_numpy = _fp32_on_device(raw_score, "raw_score")
    K = s.shape[-1] if s.dim() else 1
    out = torch.empty_like(s)
    with torch.cuda.device(s.device):
        check(lib.ssnb_video_fuse(s.data_ptr(), None, None, 0, s.numel() // max(K, 1), K, 1, float(T), out.data_ptr(), _stream()),
              None, "softmax")
    return out.cpu().numpy() if was_numpy else out


def _scores_on_device(scores):
    if torch.is_tensor(scores):
        if not scores.is_cuda:
            raise RuntimeError("scores must be a numpy array or a CUDA tensor: libssn_b200 has no CPU path")
        return scores
    a = np.asarray(scores)
    if a.dtype not in (np.float32, np.float64):
        a = a.astype(np.float64)
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", torch.cuda.current_device()))


def video_metrics_packed(scores, label_video, label, top_k=3, class_label=None, trace=False):
    """scores: [V, K] fp32 or float64 (CUDA tensor, or host data copied once); label_video / label: the (video, label)
    pairs, int [n] (repeated pairs count once); class_label: optional int [V], one label per video for mean_class_accuracy.
    -> dict of device tensors: hits int32 [V], label_count int32 [V], top_k_accuracy / mean_ap / mean_class_accuracy
    float64 [1], ap float64 [K]; confusion int32 [3, K] (label counts, prediction counts, hits) with class_label; with
    trace=True top_k_idx int32 [V, min(top_k, K)], best first.  Nothing waits for the device."""
    s = _scores_on_device(scores)
    if s.dim() != 2:
        raise ValueError("scores must be [V, K]")
    if s.dtype not in (torch.float32, torch.float64):
        raise TypeError("scores must be float32 or float64")
    s = s.contiguous()
    dev = s.device
    V, K = s.shape
    lv, lab = _on(dev, label_video, torch.int32).reshape(-1), _on(dev, label, torch.int32).reshape(-1)
    if lv.numel() != lab.numel():
        raise ValueError("one video per label")
    cl = None if class_label is None else _on(dev, class_label, torch.int32).reshape(-1)
    if cl is not None and cl.numel() != V:
        raise ValueError("class_label must hold one label per video")
    ws_bytes = lib.ssnb_video_metrics_workspace_bytes(V, K)           # 0 for arguments the call rejects
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    i32, f64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float64, device=dev)
    kk = min(int(top_k), K) if int(top_k) >= 1 else 1
    out = {"hits": torch.empty(max(V, 1), **i32), "label_count": torch.empty(max(V, 1), **i32), "top_k_accuracy": torch.empty(1, **f64),
           "ap": torch.empty(max(K, 1), **f64), "mean_ap": torch.empty(1, **f64), "mean_class_accuracy": torch.empty(1, **f64)}
    if cl is not None:
        out["confusion"] = torch.empty((3, max(K, 1)), **i32)
    if trace:
        out["top_k_idx"] = torch.empty((max(V, 1), kk), **i32)
    opt = lambda k: out[k].data_ptr() if k in out else None           # noqa: E731
    with torch.cuda.device(dev):
        check(lib.ssnb_video_metrics(s.data_ptr(), int(s.dtype == torch.float64), V, K, _p(lv), _p(lab), lv.numel(),
                                     None if cl is None else _p(cl), int(top_k), out["hits"].data_ptr(), out["label_count"].data_ptr(),
                                     opt("top_k_idx"), out["top_k_accuracy"].data_ptr(), out["ap"].data_ptr(), out["mean_ap"].data_ptr(),
                                     opt("confusion"), out["mean_class_accuracy"].data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
              None, "video_metrics")
    out["top_k"] = int(top_k)
    return out


def _one(lb_set, scores, k):
    s = _scores_on_device(scores).reshape(1, -1)
    labels = sorted(int(x) for x in lb_set)
    r = video_metrics_packed(s, [0] * len(labels), labels, k)
    return int(r["hits"][0]), int(r["label_count"][0])


def top_k_acc(lb_set, scores, k=3):
    """metrics.py:14-16 -> (labels of lb_set among the k best classes, len(lb_set)).  Labels must be class indices."""
    return _one(lb_set, scores, k)


def top_k_hit(lb_set, scores, k=3):
    """metrics.py:19-21 -> (True when a label of lb_set is among the k best classes, 1)."""
    return _one(lb_set, scores, k)[0] > 0, 1


def _dict_to_packed(score_dict, video_list):
    vids = [v for v in video_list if v.id in score_dict]
    if not vids:
        raise ValueError("no video of video_list is in score_dict")
    scores = np.stack([np.asarray(score_dict[v.id]) for v in vids])
    lv, lab = [], []
    for i, v in enumerate(vids):
        for c in sorted({inst.num_label for inst in v.instances}):
            lv.append(i)
            lab.append(c)
    return scores, np.array(lv, np.int32), np.array(lab, np.int32)


def top_k_accuracy(score_dict, video_list, k):
    """metrics.py:28-38: the fraction of the videos in score_dict with a label among their k best classes."""
    s, lv, lab = _dict_to_packed(score_dict, video_list)
    return float(video_metrics_packed(s, lv, lab, k)["top_k_accuracy"][0])


def top_3_accuracy(score_dict, video_list):
    return top_k_accuracy(score_dict, video_list, 3)


def video_mean_ap(score_dict, video_list):
    """metrics.py:41-50: sklearn's macro average precision of the videos in score_dict against their label indicator."""
    s, lv, lab = _dict_to_packed(score_dict, video_list)
    return float(video_metrics_packed(s, lv, lab, 1)["mean_ap"][0])


def mean_class_accuracy(scores, labels):
    """metrics.py:53-60: np.argmax per video, the confusion matrix over the labelled and predicted classes, the mean of
    diag / row sum (NaN when a predicted class is never labelled).  Labels must be in 0..K-1."""
    s = _scores_on_device(scores)
    lab = np.asarray(labels).reshape(-1)
    if s.dim() != 2 or len(lab) != s.shape[0]:
        raise ValueError("scores must be [V, K] with one label per video")
    if len(lab) and (lab.min() < 0 or lab.max() >= s.shape[1]):
        raise ValueError("labels must be class indices 0..K-1")
    r = video_metrics_packed(s, np.zeros(0, np.int32), np.zeros(0, np.int32), 1, class_label=lab.astype(np.int32))
    return float(r["mean_class_accuracy"][0])
