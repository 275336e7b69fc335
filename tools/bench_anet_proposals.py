#!/usr/bin/env python
"""Benchmark of ActivityNet AR-AN evaluation on one H100 (ops/proposal_eval.py, csrc/proposal_ar.cu); prints ONE JSON line.

  python tools/bench_anet_proposals.py [--windows 7] [--calls 10] [--oracle-videos 300]

Three seeded synthetic sets, proposals and ground truth already packed on the device, default tIoU thresholds
(0.5:0.05:0.95) and the toolkit's default budget (every proposal kept, AN = proposals per video):
  anet100   4926 videos (ActivityNet-1.3 validation), ~1.55 instances per video (~7.7 k), 100 uniform random proposals each
            -- the shape of the toolkit's own sample (uniform_random_proposals.json)
  anet1000  the same videos with 1000 proposals each
  thumos    213 videos (THUMOS14 test), ~15.5 instances per video (~3.3 k), ~2000 TAG-like proposals per video
Timed with CUDA events after a warm-up: a window is `calls` back-to-back average_recall_packed + ar_an_report calls (the
report copies the curves to the host, so every call ends in a synchronisation); the figure is the median window / calls.
Pairs are the (kept proposal, instance) tIoUs the toolkit computes, sum_v nr_v * G_v; bytes are counted from the shapes
(boxes and scores read, the ranking's keys and rows written and read once, ground truth read, first hits written and read),
not measured.  For comparison the repository's numpy oracle (oracle/anet_proposal_oracle.py, one CPU core) evaluates the
first `oracle-videos` videos of each set.  The card's name and power limit are read in the same run.  Needs a CUDA device:
without one it fails.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

THR = np.linspace(0.5, 0.95, 10)


def synth(n_videos, per_video, inst, tag_like, seed):
    """-> (boxes [rows, 2], scores [rows], counts [V], gt [G, 2], gt_counts [V]) in seconds"""
    g = np.random.RandomState(seed)
    boxes, scores, counts, gts, gcounts = [], [], [], [], []
    for _ in range(n_videos):
        dur = float(g.uniform(30, 1600) if tag_like else g.uniform(10, 230))
        ng = int(g.randint(1, 2 * inst + 1)) if tag_like else int(g.choice([1, 2, 3], p=[0.6, 0.25, 0.15]))
        c, d = g.uniform(0, dur, ng), (g.uniform(1, 25, ng) if tag_like else g.uniform(0.05, 0.8, ng) * dur)
        gt = np.stack([np.clip(c - d / 2, 0, dur), np.clip(c + d / 2, 0, dur)], 1)
        n = int(g.randint(per_video // 2, 3 * per_video // 2 + 1)) if tag_like else per_video
        if tag_like:
            pc, pd = g.uniform(0, dur, n), np.exp(g.normal(1.5, 1.0, n))
            b = np.stack([np.clip(pc - pd / 2, 0, None), np.minimum(pc + pd / 2, dur)], 1)
        else:
            b = np.sort(g.uniform(0, dur, (n, 2)), 1)
        boxes.append(b), scores.append(g.rand(n)), counts.append(n), gts.append(gt), gcounts.append(ng)
    return np.concatenate(boxes), np.concatenate(scores), np.array(counts), np.concatenate(gts), np.array(gcounts)


def timed(fn, calls, windows):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / calls)
    return {"gpu_ms": float(np.median(ms)), "gpu_ms_min": float(min(ms)), "gpu_ms_max": float(max(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--oracle-videos", type=int, default=300)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_anet_proposals.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from bench_proposals import card_info
    from ops import proposal_eval as E
    from ops.proposal_lists import compact_layout
    from oracle import anet_proposal_oracle as O
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {}
    for name, (V, per, inst, tag_like, seed) in (("anet100", (4926, 100, 0, False, 31)), ("anet1000", (4926, 1000, 0, False, 31)),
                                                 ("thumos", (213, 2000, 15, True, 32))):
        boxes, scores, counts, gt, gcounts = synth(V, per, inst, tag_like, seed)
        off = np.concatenate([[0], np.cumsum(gcounts)]).tolist()
        B, S, G = (torch.as_tensor(x).to(dev) for x in (boxes, scores, gt))
        first, count = compact_layout(counts, dev)

        def call():
            return E.ar_an_report(E.average_recall_packed(B, S, first, count, G, off, None, THR))
        row = timed(call, args.calls, args.windows)
        rep = call()
        nv = min(args.oracle_videos, V)
        n_rows, n_gt = int(counts[:nv].sum()), int(gcounts[:nv].sum())
        t0 = time.perf_counter()
        O.average_recall(boxes[:n_rows], scores[:n_rows], counts[:nv], gt[:n_gt], gcounts[:nv], None, THR)
        oracle_s = time.perf_counter() - t0
        full = O.average_recall(boxes, scores, counts, gt, gcounts, None, THR)
        same = all(rep[k].tobytes() == full[k].tobytes() for k in ("recall", "avg_recall", "proposals_per_video"))
        rows, inst_total, T = int(counts.sum()), int(gcounts.sum()), len(THR)
        pairs = int((full["nr"].astype(np.int64) * gcounts).sum())
        moved = rows * (16 + 8 + 2 * 12) + inst_total * (16 + 2 * 4 * T + 8)
        row.update({"videos": V, "proposals": rows, "ground_truth": inst_total, "pairs": pairs, "bytes_moved": moved,
                    "gb_per_s": moved / row["gpu_ms"] / 1e6, "pairs_per_s": pairs / row["gpu_ms"] * 1e3,
                    "average_number": float(rep["proposals_per_video"][-1]), "auc_percent": float(rep["auc_percent"]),
                    "gpu_equals_oracle": bool(same), "oracle_videos": nv, "oracle_cpu_s": oracle_s,
                    "oracle_cpu_s_per_video": oracle_s / nv})
        res[name] = row
    line = {"metric": "anet_ar_an_gpu_ms_anet100", "value": res["anet100"]["gpu_ms"], "unit": "ms", "higher_is_better": False,
            "windows": args.windows, "calls_per_window": args.calls, "datasets": res,
            "timing": "CUDA events around `calls` back-to-back average_recall_packed + ar_an_report calls after a warm-up call; "
                      "median window / calls",
            "card": card_info(), "torch": torch.__version__}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
