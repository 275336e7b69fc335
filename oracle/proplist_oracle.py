"""Pure-Python / numpy restatement of the reference's proposal labelling, float64 throughout, in the reference's own
operation order -- what csrc/proposal_lists.cu is held to (tests/test_proplist_host.py pins this file to golden vectors of
the real reference, tests/test_gpu_proplist.py pins the library to this file).  Each function names the lines it follows."""
import math

import numpy as np


def temporal_iou(a, b):
    """ops/detection_metrics.py:7-20 and ops/utils.py:40-53"""
    union = min(a[0], b[0]), max(a[1], b[1])
    inter = max(a[0], b[0]), min(a[1], b[1])
    if inter[0] >= inter[1]:
        return 0
    return float(inter[1] - inter[0]) / float(union[1] - union[0])


def overlap_over_b(a, b):
    """ops/detection_metrics.py:23-28"""
    inter = max(a[0], b[0]), min(a[1], b[1])
    if inter[0] >= inter[1]:
        return 0
    return float(inter[1] - inter[0]) / float(b[1] - b[0])


def name_proposals(gt, gt_label, boxes, thresh=0.0):
    """ops/detection_metrics.py:54-76 -> label int32 [n], max_overlap [n], overlap_self [n]"""
    n = len(boxes)
    label, mo, ms = np.zeros(n, np.int32), np.zeros(n), np.zeros(n)
    for i, es in enumerate(boxes):
        es = (float(es[0]), float(es[1]))
        for g, lab in zip(gt, gt_label):
            g = (float(g[0]), float(g[1]))
            with np.errstate(all="ignore"):
                ov, pr = np.float64(temporal_iou(g, es)), np.float64(overlap_over_b(g, es))
            if ov > thresh and ov > mo[i]:
                label[i], mo[i], ms[i] = int(lab) + 1, ov, pr
    return label, mo, ms


def gt_best_iou(gt, boxes):
    """per ground truth the largest tIoU over the boxes (NaN ignored): temporal_recall (:31-51) hits iff this is > thresh"""
    out = np.zeros(len(gt))
    for j, g in enumerate(gt):
        for es in boxes:
            with np.errstate(all="ignore"):
                ov = np.float64(temporal_iou((float(g[0]), float(g[1])), (float(es[0]), float(es[1]))))
            if ov > out[j]:
                out[j] = ov
    return out


def proposal_recall(gt_best_list, thresholds):
    """ops/detection_metrics.py:79-83 for several thresholds -> hits [V, n_thr], per_video [n_thr], per_instance [n_thr]"""
    hits = np.array([[int((b > th).sum()) for th in thresholds] for b in gt_best_list], np.int64).reshape(len(gt_best_list), len(thresholds))
    total = np.array([len(b) for b in gt_best_list])
    with np.errstate(all="ignore"):
        pv = np.array([np.sum(hits[:, t] == total) / float(len(total)) for t in range(len(thresholds))])
        pi = np.array([np.sum(hits[:, t]) / float(np.sum(total)) for t in range(len(thresholds))])
    return hits, pv, pi


def sliding_windows(duration, time_step=1, max_level=8, overlap=0.4):
    """ops/sequence_funcs.py:37-54 -> float64 [n, 2]"""
    pr = []
    for t_span in [2 ** x for x in range(max_level)]:
        step = int(np.ceil(t_span * time_step * (1 - overlap)))
        pr.extend((i, i + t_span) for i in np.arange(0, duration, step))
    pr = [x for x in pr if min(duration, x[1]) - x[0] >= 1]
    return np.array(pr, np.float64).reshape(-1, 2)


def sliding_window_steps(time_step=1, max_level=8, overlap=0.4):
    return [2 ** x for x in range(max_level)], [int(np.ceil(2 ** x * time_step * (1 - overlap))) for x in range(max_level)]


def seconds_to_frames(boxes, duration, frame_cnt):
    """ops/io.py:109-123 -> int64 [n, 2]"""
    real_fps = float(frame_cnt) / float(duration)
    return np.array([(int(float(b[0]) * real_fps), int(float(b[1]) * real_fps)) for b in boxes], np.int64).reshape(-1, 2)


def normalised_to_frames(boxes, frame_cnt):
    """ops/io.py:44-47 -> int64 [n, 2]"""
    return np.array([(int(float(b[0]) * frame_cnt), int(float(b[1]) * frame_cnt)) for b in boxes], np.int64).reshape(-1, 2)


def record_rows(frames, frame_cnt):
    """SSNInstance / SSNVideoRecord (ssn_dataset.py:13-21,81-93) -> keep bool [n], valid int64 [n, 2], coverage [n]"""
    frames = np.asarray(frames, np.int64).reshape(-1, 2)
    keep = np.array([int(e) > int(s) and int(s) < frame_cnt for s, e in frames], bool).reshape(-1)
    valid = np.array([(int(s), min(int(e), frame_cnt)) for s, e in frames], np.int64).reshape(-1, 2)
    cov = np.array([(int(e) - int(s)) / frame_cnt for s, e in frames], np.float64).reshape(-1)
    return keep, valid, cov


def format_window_list(path, frame_cnt, gt_label, gt_frames, label, max_overlap, overlap_self, frames):
    """ops/io.py:113-134: one video's block of a proposal list (labels already + 1)"""
    dump_gt = ['{} {} {}'.format(int(l), int(f[0]), int(f[1])) for l, f in zip(gt_label, gt_frames)]
    dump_pr = ['{} {:.04f} {:.04f} {} {}'.format(int(l), float(o), float(s), int(f[0]), int(f[1]))
               for l, o, s, f in zip(label, max_overlap, overlap_self, frames)]
    return '{path}\n{duration}\n{fps}\n{num_gt}\n{gts}{num_window}\n{prs}\n'.format(
        path=path, duration=frame_cnt, fps=1, num_gt=len(dump_gt), gts='\n'.join(dump_gt) + ('\n' if len(dump_gt) else ''),
        num_window=len(dump_pr), prs='\n'.join(dump_pr))


def parse_proposal_list(text):
    """ops/io.py:7-31 load_proposal_file on the file's text -> [(vid, n_frame, gt rows, proposal rows)] of split strings"""
    from itertools import groupby
    lines = text.splitlines(True)
    out = []
    for k, g in groupby(lines, lambda x: x.startswith('#')):
        if k:
            continue
        info = [x.strip() for x in g]
        n_gt = int(info[3])
        gt = [x.split() for x in info[4:4 + n_gt]]
        n_pr = int(info[4 + n_gt])
        out.append((info[0], int(float(info[1]) * float(info[2])), gt, [x.split() for x in info[5 + n_gt:5 + n_gt + n_pr]]))
    return out


def proposal_targets(videos, fg_thresh=0.7, incomplete_iou_thresh=0.3, bg_iou_thresh=0.01, bg_coverage_thresh=0.02,
                     incomplete_overlap_thresh=0.7, exclude_empty=True):
    """ssn_dataset.py:29-55,103-131,196-227,382-391.  videos: dicts of kept rows: frames int64 [n, 2] (valid), best_iou,
    overlap_self, coverage [n], gt_frames int64 [g, 2] (valid).  -> per video dict(tags, reg, pools) and stats [2, 2], totals"""
    out, targets, totals = [], [], [0, 0, 0, 0, 0]
    for v in videos:
        n = len(v["frames"])
        tags, reg = np.zeros(n, np.uint8), np.zeros((n, 2))
        gt = [(int(a), int(b)) for a, b in v["gt_frames"]]
        used = not (exclude_empty and len(gt) == 0)
        for i in range(n if used else 0):
            iou, osf, cov = float(v["best_iou"][i]), float(v["overlap_self"][i]), float(v["coverage"][i])
            fg = iou > fg_thresh
            inc = iou < incomplete_iou_thresh and osf > incomplete_overlap_thresh
            bg = (not inc) and iou < bg_iou_thresh and cov > bg_coverage_thresh
            tags[i] = (1 if fg else 0) | (2 if inc else 0) | (4 if bg else 0)
            if fg and gt:
                s, e = int(v["frames"][i][0]), int(v["frames"][i][1])
                ious = [temporal_iou((s, e), g) for g in gt]
                b = gt[int(np.argmax(ious))]
                prop_center, gt_center = (s + e) / 2, (b[0] + b[1]) / 2
                prop_size, gt_size = e - s + 1, b[1] - b[0] + 1
                reg[i] = ((gt_center - prop_center) / prop_size, math.log(gt_size / prop_size))
            if fg:
                targets.append(list(reg[i]))
        pools = [int((tags & 1 > 0).sum()), int((tags & 2 > 0).sum()), int((tags & 4 > 0).sum()), len(gt) if used else 0]
        for k in range(4):
            totals[k] += pools[k]
        totals[4] += int(used)
        out.append({"tags": tags, "reg": reg, "pools": pools})
    with np.errstate(all="ignore"):
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            stats = np.array((np.mean(targets, axis=0), np.std(targets, axis=0))) if targets else np.full((2, 2), np.nan)
    return out, stats, totals


def test_proposals(frames, frame_cnt, new_length=1, test_interval=6):
    """ssn_dataset.py:393-428 from a video's kept valid frames -> num_ticks, rel_prop [n, 2], ticks int64 [n, 4], scaling [n, 2]"""
    n_ticks = len(np.arange(0, frame_cnt - new_length, test_interval, dtype=int))
    props = [(int(s), int(e)) for s, e in np.asarray(frames, np.int64).reshape(-1, 2)] or [(0, frame_cnt - 1)]
    rel, ticks, scaling = [], [], []
    for s, e in props:
        rel_prop = s / frame_cnt, e / frame_cnt
        rel_duration = rel_prop[1] - rel_prop[0]
        rel_starting_duration = rel_duration * 0.5
        rel_ending_duration = rel_duration * 0.5
        rel_starting = rel_prop[0] - rel_starting_duration
        rel_ending = rel_prop[1] + rel_ending_duration
        real_rel_starting = max(0.0, rel_starting)
        real_rel_ending = min(1.0, rel_ending)
        scaling.append(((rel_prop[0] - real_rel_starting) / rel_starting_duration, (real_rel_ending - rel_prop[1]) / rel_ending_duration))
        ticks.append((int(real_rel_starting * n_ticks), int(rel_prop[0] * n_ticks), int(rel_prop[1] * n_ticks), int(real_rel_ending * n_ticks)))
        rel.append(rel_prop)
    return n_ticks, np.array(rel, np.float64), np.array(ticks, np.int64), np.array(scaling, np.float64)


test_proposals.__test__ = False      # not a pytest test
