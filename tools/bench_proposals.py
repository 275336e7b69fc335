#!/usr/bin/env python
"""Benchmark of TAG bottom-up proposal generation on one H100 (ops/proposals.py, csrc/proposals.cu); prints ONE JSON line.

  python tools/bench_proposals.py [--anet-videos 5000] [--thumos-videos 200] [--batch 500] [--thumos-batch 50] [--steps 3]

Two seeded synthetic datasets of merged actionness scores (K = 2, gen_prop's defaults: bw 3, 12 thresholds, 9 tolerances,
NMS 0.9):
  anet    ActivityNet-like: T uniform in [300, 2500] ticks, smooth scores (a few slow sinusoids plus mild noise)
  thumos  THUMOS-like long videos: T uniform in [4000, 12000] ticks, noisy scores as from an early checkpoint, which
          give tens of thousands of boxes per video before NMS
Each dataset is cut into batches of videos (one library call per batch; the box workspace is bounded by
12 * 9 * (T + 1) slots per video, so a batch of 500 ActivityNet-like videos takes a few GB).  GPU time per batch is measured
with CUDA events after one warm-up pass over every batch, `steps` times, with the host-side slicing of the results outside
the events.  For comparison the repository's numpy oracle (oracle/proposal_oracle.py, one CPU core) runs on the first few
videos of each dataset, whose GPU results must equal it exactly.  The card's name and power limit are read in the same run.
Needs a CUDA device: without one it fails.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def synth_dataset(n, t_lo, t_hi, noisy, seed):
    """-> (list of [T, 2] fp32 arrays, durations)"""
    g = np.random.RandomState(seed)
    scores, durs = [], []
    for _ in range(n):
        T = int(g.randint(t_lo, t_hi + 1))
        x = np.arange(T)
        fg = sum(g.uniform(1.0, 2.5) * np.sin(2 * np.pi * x / g.uniform(150, 900) + g.uniform(0, 6.3)) for _ in range(3))
        fg = fg + g.randn(T) * (7.0 if noisy else 0.4)
        f = (g.randn(T, 2) * 0.3).astype(np.float32)
        f[:, 1] += fg.astype(np.float32)
        scores.append(f)
        durs.append(T / g.uniform(2.0, 8.0))
    return scores, durs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--anet-videos", type=int, default=5000)
    ap.add_argument("--thumos-videos", type=int, default=200)
    ap.add_argument("--batch", type=int, default=500)
    ap.add_argument("--thumos-batch", type=int, default=50)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--oracle-videos", type=int, default=8)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_proposals.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from ops.proposals import bottom_up_proposals_packed
    from oracle import proposal_oracle as P
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {}
    for name, n, t_lo, t_hi, noisy, bs, seed in (("anet", args.anet_videos, 300, 2500, False, args.batch, 1),
                                                 ("thumos", args.thumos_videos, 4000, 12000, True, args.thumos_batch, 2)):
        scores, durs = synth_dataset(n, t_lo, t_hi, noisy, seed)
        batches = []
        for lo in range(0, n, bs):
            part = scores[lo:lo + bs]
            offs = np.concatenate([[0], np.cumsum([len(s) for s in part])]).tolist()
            batches.append((torch.tensor(np.concatenate(part), device=dev), offs, durs[lo:lo + bs]))
        def run(b, trace=False):
            return bottom_up_proposals_packed(b[0], b[1], b[2], trace=trace)
        raw = kept = 0
        for i, b in enumerate(batches):                                 # warm-up; the first batch's results are checked below
            o = run(b, trace=True)
            raw += int(o["raw_counts"].sum())
            kept += int(o["counts"].sum())
            if i == 0:
                first = {k: o[k] for k in ("slot0", "counts", "frames", "scores")}
            del o
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.steps):
            for b in batches:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(b)
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
        total_s = sum(ms) / args.steps / 1e3
        # the repository oracle on one CPU core, on the first videos; the GPU must give the same boxes
        t0 = time.perf_counter()
        ref = [P.gen_prop(scores[v], durs[v]) for v in range(min(args.oracle_videos, n))]
        oracle_s = (time.perf_counter() - t0) / max(len(ref), 1)
        same = True
        for v, r in enumerate(ref):
            a, c = int(first["slot0"][v]), int(first["counts"][v])
            fr = first["frames"][a:a + c].cpu().numpy()
            same &= fr.shape[0] == len(r["pr_frames"]) and bool((fr == r["pr_frames"]).all())
            same &= bool((first["scores"][a:a + c].cpu().numpy() == r["pr_score"]).all())
        res[name] = {"videos": n, "ticks": int(sum(len(s) for s in scores)), "batches": len(batches), "videos_per_batch": bs,
                     "gpu_ms_per_batch": total_s * 1e3 / len(batches), "gpu_ms_per_batch_max": max(ms),
                     "videos_per_s": n / total_s, "boxes_before_nms": raw, "boxes_kept": kept,
                     "oracle_cpu_s_per_video": oracle_s, "oracle_videos": len(ref), "oracle_videos_per_s": 1.0 / oracle_s,
                     "gpu_equals_oracle_on_those": bool(same)}
        del batches, first
        torch.cuda.empty_cache()
    line = {"metric": "tag_proposals_videos_per_s", "value": res["anet"]["videos_per_s"], "unit": "videos/s", "higher_is_better": True,
            "steps": args.steps, "config": {"num_class": 2, "bw": 3, "thresholds": 12, "tolerances": 9, "nms_threshold": 0.9,
                                            "data": "synthetic", "timing": "CUDA events per batch call, after one warm-up pass"},
            "datasets": res, "card": card_info(), "torch": torch.__version__}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
