#!/usr/bin/env python
"""Benchmark of proposal labelling on one H100 (ops/proposal_lists.py, csrc/proposal_lists.cu); prints ONE JSON line.

  python tools/bench_proposal_lists.py [--windows 7] [--calls 20] [--oracle-videos 32]

Two seeded synthetic sets, boxes already on the device:
  thumos  1600 videos, TAG-like box counts (median ~150, up to ~3000), ~15 ground-truth instances per video
  anet    4800 videos, sliding windows at the script defaults (overlap 0.7, 8 levels), ~1.5 instances per video; the window
          generation itself is timed as its own row
Timed with CUDA events after a warm-up: a window is `calls` back-to-back calls of label_proposals (name_proposal + recall +
frame windows of proposals and ground truth), the figure is the median window divided by `calls`.  Bytes moved are counted
from the shapes (boxes and ground truth read, labels / overlaps / frames / maxima written), not measured.  For comparison the
repository's Python oracle (oracle/proplist_oracle.py, one CPU core) labels the first `oracle-videos` videos.  The card's name
and power limit are read in the same run.  Needs a CUDA device: without one it fails.
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


def synth_thumos(n, seed):
    g = np.random.RandomState(seed)
    vids = []
    for _ in range(n):
        duration = float(g.uniform(30, 1600))
        nb = int(min(3000, np.exp(g.normal(5.0, 0.9)))) + 1
        ng = int(g.randint(1, 30))
        c, d = g.uniform(0, duration, ng), g.uniform(1, 25, ng)
        gt = np.stack([np.clip(c - d / 2, 0, duration), np.clip(c + d / 2, 0, duration)], 1)
        pc, pd = g.uniform(0, duration, nb), np.exp(g.normal(1.5, 1.0, nb))
        vids.append(dict(duration=duration, frame_cnt=int(duration * 30), gt=gt, gt_label=g.randint(0, 20, ng).astype(np.int32),
                         boxes=np.stack([np.clip(pc - pd / 2, 0, None), np.minimum(pc + pd / 2, duration)], 1)))
    return vids


def synth_anet(n, seed):
    g = np.random.RandomState(seed)
    vids = []
    for _ in range(n):
        duration = float(g.uniform(10, 230))
        ng = int(g.choice([1, 1, 2, 3]))
        c, d = g.uniform(0, duration, ng), g.uniform(0.1, 0.9, ng) * duration
        gt = np.stack([np.clip(c - d / 2, 0, duration), np.clip(c + d / 2, 0, duration)], 1)
        vids.append(dict(duration=duration, frame_cnt=int(duration * 30), gt=gt, gt_label=g.randint(0, 100, ng).astype(np.int32)))
    return vids


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
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--oracle-videos", type=int, default=32)
    ap.add_argument("--thumos-videos", type=int, default=1600)
    ap.add_argument("--anet-videos", type=int, default=4800)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_proposal_lists.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from bench_proposals import card_info
    from ops import proposal_lists as L
    from oracle import proplist_oracle as P
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt).to(dev)
    res = {}
    for name, vids in (("thumos", synth_thumos(args.thumos_videos, 21)), ("anet", synth_anet(args.anet_videos, 22))):
        durs, fcs = [v["duration"] for v in vids], [v["frame_cnt"] for v in vids]
        goff = np.concatenate([[0], np.cumsum([len(v["gt"]) for v in vids])]).tolist()
        gt, glab = T(np.concatenate([v["gt"] for v in vids]), torch.float64), T(np.concatenate([v["gt_label"] for v in vids]), torch.int32)
        row = {}
        if name == "anet":
            sw = L.sliding_window_proposals(durs, 1, 8, 0.7)
            d_dev, cap = T(durs, torch.float64), sw["boxes"].shape[0]
            row["sliding_windows"] = timed(lambda: L.sliding_window_proposals(d_dev, 1, 8, 0.7, capacity=cap), args.calls, args.windows)
            props = {"boxes": sw["boxes"], "first": sw["first"], "count": sw["count"]}
            counts = sw["count"].cpu().numpy()
            for v, f, c in zip(vids, sw["first"].cpu().numpy(), counts):
                v["boxes"] = sw["boxes"][f:f + c].cpu().numpy()
        else:
            counts = np.array([len(v["boxes"]) for v in vids])
            first, count = L.compact_layout(counts, dev)
            props = {"boxes": T(np.concatenate([v["boxes"] for v in vids]), torch.float64), "first": first, "count": count}
        n_box, n_gt = int(counts.sum()), goff[-1]
        fc_dev, dur_dev = T(fcs, torch.int32), T(durs, torch.float64)
        row.update(timed(lambda: L.label_proposals(props, gt, glab, goff, dur_dev, fc_dev), args.calls, args.windows))
        r = L.label_proposals(props, gt, glab, goff, dur_dev, fc_dev)
        rep = L.recall_report(r["recall"], r["count"])
        # the Python oracle on the first videos, one CPU core; its labels must be the GPU's
        nv = min(args.oracle_videos, len(vids))
        t0 = time.perf_counter()
        named = [P.name_proposals(v["gt"], v["gt_label"], v["boxes"]) for v in vids[:nv]]
        best = [P.gt_best_iou(v["gt"], v["boxes"]) for v in vids[:nv]]
        for v in vids[:nv]:
            P.seconds_to_frames(v["boxes"], v["duration"], v["frame_cnt"])
        oracle_s = time.perf_counter() - t0
        first_h = props["first"].cpu().numpy()
        same = all((r["max_overlap"][first_h[i]:first_h[i] + counts[i]].cpu().numpy().tobytes() == named[i][1].tobytes()) for i in range(nv))
        same &= np.concatenate(best).tobytes() == r["gt_best"][:goff[nv]].cpu().numpy().tobytes()
        pairs = int(sum(int(c) * (goff[i + 1] - goff[i]) for i, c in enumerate(counts)))
        # read: boxes 16 B (twice: naming, frames), ground truth 20 B per staging CTA is not counted, only once; written: label 4,
        # overlaps 16, frames 16 per box; maxima 8 and frames 16 per ground truth
        moved = n_box * (16 * 2 + 4 + 16 + 16) + n_gt * (20 + 16 + 8 + 8 + 16)
        row.update({"videos": len(vids), "proposals": n_box, "ground_truth": n_gt, "pairs": pairs, "bytes_moved": moved,
                    "gb_per_s": moved / row["gpu_ms"] / 1e6, "pairs_per_s": pairs / row["gpu_ms"] * 1e3,
                    "oracle_videos": nv, "oracle_cpu_s": oracle_s, "oracle_cpu_s_per_video": oracle_s / nv, "gpu_equals_oracle_on_those": bool(same),
                    "average_proposals": rep["average_proposals"], "per_instance_recall": rep["per_instance"].tolist()})
        res[name] = row
    line = {"metric": "proposal_labelling_gpu_ms_thumos", "value": res["thumos"]["gpu_ms"], "unit": "ms", "higher_is_better": False,
            "windows": args.windows, "calls_per_window": args.calls, "datasets": res,
            "timing": "CUDA events around `calls` back-to-back label_proposals calls after a warm-up call; median window / calls",
            "card": card_info(), "torch": torch.__version__}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
