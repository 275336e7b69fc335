#!/usr/bin/env python
"""Benchmark of TV-L1 optical flow on one H100 (ops/optical_flow.py, csrc/optical_flow.cu); prints ONE JSON line.

  python tools/bench_optical_flow.py [--videos 8] [--frames 33] [--calls 3] [--oracle-pairs 1]

THUMOS-like input: `videos` videos of `frames` 340 x 256 RGB frames in one call (8 x 33 = 256 pairs), each a seeded texture
moving by a random sub-pixel to two-pixel step per frame.  Two modes, OpenCV's defaults otherwise:
  stop    the stopping rule (epsilon 0.01)
  fixed   fixed_iterations: 300 iterations in every warp
Per mode:
  pairs_per_s        pairs / (median over `calls` calls of CUDA events around one tvl1_flow call, after a warm-up call)
  stage_ms           device time per kernel of one call, from torch.profiler in a separate call
  bytes_per_iter     the least HBM traffic of one primal + one dual update of the call, from shapes (88 B per pixel: the
                     primal reads 10 and writes 2 floats, the dual reads 6 and writes 4; neighbour reads counted as cache hits)
  hbm_share          fixed mode: iterations' bytes / (primal + dual device time) / 3.35 TB/s (the H100 SXM data sheet figure)
oracle_s_per_pair: oracle/tvl1_oracle.py (float64 numpy, one core) on the first `oracle-pairs` pairs with the stopping rule.
The card's name, power limit and SM clocks are read in the same run.  Needs a CUDA device: without one it fails.
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

H, W = 256, 340
HBM = 3.35e12


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def synth_frames(videos, frames, seed=0):
    from oracle import tvl1_oracle as O
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    out = []
    for v in range(videos):
        step = rng.uniform(-2, 2, 2)
        for k in range(frames):
            ch = [O.texture(xs - k * step[0], ys - k * step[1], seed=3 * v + c, waves=6) for c in range(3)]
            out.append(np.clip(np.rint(np.stack(ch, -1)), 0, 255).astype(np.uint8))
    return np.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=8)
    ap.add_argument("--frames", type=int, default=33)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--oracle-pairs", type=int, default=1)
    a = ap.parse_args()
    import torch
    from oracle import tvl1_oracle as O
    from ops.optical_flow import TVL1Plan
    if not torch.cuda.is_available():
        raise SystemExit("bench_optical_flow needs a CUDA device")
    dev = torch.device("cuda:0")
    frames = synth_frames(a.videos, a.frames)
    off = np.arange(a.videos + 1) * a.frames
    x = torch.from_numpy(frames).to(dev)
    P = int(off[-1]) - a.videos
    res = {"workload": "%d videos x %d frames of %dx%d (%d pairs per call)" % (a.videos, a.frames, W, H, P), "card": card_info()}
    for mode, fixed in (("stop", False), ("fixed", True)):
        plan = TVL1Plan(off, H, W, dev, fixed_iterations=fixed)
        sizes = O.level_sizes(H, W)
        plan.run(x)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            plan.run(x)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = float(np.median(times))
        its = plan.iterations.cpu().numpy()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            plan.run(x)
            torch.cuda.synchronize()
        stage = {}
        for ev in prof.key_averages():
            if "tvl1" in ev.key:
                name = ev.key.split("tvl1_")[1].split("_kernel")[0]
                stage[name] = round(stage.get(name, 0.0) + ev.device_time_total / 1e3, 2)
        bytes_iter = 88 * P * H * W
        it_bytes = sum(88.0 * P * h * w * int(its[:, l].sum()) / P for l, (h, w) in enumerate(sizes))
        r = {"s_per_call": round(t, 4), "s_range": [round(min(times), 4), round(max(times), 4)], "pairs_per_s": round(P / t, 1),
             "mean_iterations_per_pair": round(float(its.sum((1, 2)).mean()), 1), "stage_ms": stage, "bytes_per_iter_level0": bytes_iter}
        it_ms = stage.get("primal", 0.0) + stage.get("dual", 0.0)
        if it_ms > 0:
            r["iteration_bytes"] = it_bytes
            r["hbm_share"] = round(it_bytes / (it_ms / 1e3) / HBM, 3)
        res[mode] = r
        del plan
        torch.cuda.empty_cache()
    g = O.grey(frames[:a.oracle_pairs + 1]).astype(np.float64)
    t0 = time.perf_counter()
    for k in range(a.oracle_pairs):
        O.tvl1(g[k], g[k + 1])
    res["oracle_s_per_pair"] = round((time.perf_counter() - t0) / max(a.oracle_pairs, 1), 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
