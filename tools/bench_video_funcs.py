"""Video-level aggregation and metrics on the GPU (ops/video_funcs.py, ops/metrics.py) over two seeded synthetic sets, one JSON
line on stdout:

  anet       ActivityNet-1.3-like: 4926 videos, T uniform in 50..600 ticks, 10 crops, 200 classes; every aggregation mode, in
             calls of whole videos below 2 GB of scores each (a few hundred videos)
  kinetics   Kinetics-400-like: 19881 videos, 25 ticks, 10 crops, 400 classes; default aggregation in one call
  metrics    top-k hits, per-class AP and mean class accuracy of each set's video scores; fusion of two Kinetics streams

Each figure is the median of several CUDA-event windows after a warm-up, with the range.  For comparison, on one CPU core:
the oracle (oracle/video_funcs_oracle.py) and the reference's own functions (the copy build() vendors under oracle/_ref/ops,
when present) on a sample of videos, scaled to the whole set.  Scores are generated on the device from a seed; nothing is
written."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import video_funcs_oracle as O                      # noqa: E402
from ops.video_funcs import aggregate_packed, fuse_packed       # noqa: E402
from ops.metrics import video_metrics_packed                    # noqa: E402

MAX_CALL_BYTES = 2 << 30


def timed(fn, windows, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / reps)
    return {"median_ms": float(np.median(ms)), "min_ms": float(min(ms)), "max_ms": float(max(ms)), "windows": windows, "reps": reps}


def make_set(V, tlo, thi, crops, K, seed):
    rng = np.random.default_rng(seed)
    Ts = rng.integers(tlo, thi + 1, V) if thi > tlo else np.full(V, tlo)
    off = np.r_[0, np.cumsum(Ts)].astype(np.int64)
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.randn((int(off[-1]), crops, K), generator=g, device="cuda") * 3
    labels = rng.integers(0, K, V).astype(np.int32)
    return s, off, labels


def batches(off, row_bytes):
    """whole videos per call, each call below MAX_CALL_BYTES of scores"""
    out, b = [], 0
    for v in range(1, len(off)):
        if (off[v] - off[b]) * row_bytes > MAX_CALL_BYTES and v - 1 > b:
            out.append((b, v - 1))
            b = v - 1
    out.append((b, len(off) - 1))
    return out


def run_batched(s, off, parts, mode, **kw):
    outs = []
    for b, e in parts:
        outs.append(aggregate_packed(s[off[b]:off[e]], off[b:e + 1] - off[b], mode, **kw))
    return torch.cat(outs)


def cpu_per_video(fn, scores, off, sample):
    t = time.perf_counter()
    for v in sample:
        fn(scores[off[v]:off[v + 1]])
    return (time.perf_counter() - t) / len(sample)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--sample", type=int, default=20, help="videos per CPU comparison")
    args = ap.parse_args()
    torch.set_num_threads(1)
    dev = torch.cuda.get_device_name(0)
    res = {"device": dev}
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        res["power_limit_and_clocks"] = q
    except Exception as e:                                          # noqa: BLE001
        res["power_limit_and_clocks"] = "unavailable: %s" % e
    ref = None
    ref_ops = os.path.join(ROOT, "oracle", "_ref", "ops")
    if os.path.exists(os.path.join(ref_ops, "video_funcs.py")):
        try:
            from oracle.gen_golden_video_funcs import load_reference
            ref = load_reference(ref_ops)
        except Exception as e:                                      # noqa: BLE001
            res["reference"] = "not importable: %s" % e

    # ActivityNet-1.3-like
    s, off, labels = make_set(4926, 50, 600, 10, 200, seed=13)
    parts = batches(off, 10 * 200 * 4)
    gb = s.numel() * 4 / 1e9
    anet = {"videos": 4926, "ticks": int(off[-1]), "score_gb": gb, "calls": len(parts)}
    modes = {"sliding_window": dict(), "default": dict(), "top_k": dict(k=40), "tpp": dict(num_class=100)}
    for m, kw in modes.items():
        anet[m] = timed(lambda: run_batched(s, off, parts, m, **kw), args.windows, 1)
        anet[m]["score_gb_per_s"] = gb / (anet[m]["median_ms"] / 1e3)
    vs = run_batched(s, off, parts, "sliding_window")
    lv = np.arange(4926, dtype=np.int32)
    anet["metrics"] = timed(lambda: video_metrics_packed(vs, lv, labels, 3, class_label=labels), args.windows, 3)
    rng = np.random.default_rng(0)
    sample = np.sort(rng.choice(4926, args.sample, replace=False))
    host = {v: s[off[v]:off[v + 1]].cpu().numpy() for v in sample}
    hs = np.concatenate([host[v] for v in sample])
    hoff = np.r_[0, np.cumsum([len(host[v]) for v in sample])]
    t_or = cpu_per_video(lambda x: O.sliding_agg(x), hs, hoff, range(len(sample)))
    anet["oracle_one_core_s"] = t_or * 4926
    if ref is not None:
        t_ref = cpu_per_video(lambda x: ref[0].sliding_window_aggregation_func(x), hs, hoff, range(len(sample)))
        anet["reference_one_core_s"] = t_ref * 4926
    anet["sample_videos"] = int(args.sample)
    res["anet"] = anet
    del s, vs
    torch.cuda.empty_cache()

    # Kinetics-400-like
    s, off, labels = make_set(19881, 25, 25, 10, 400, seed=17)
    gb = s.numel() * 4 / 1e9
    kin = {"videos": 19881, "ticks": int(off[-1]), "score_gb": gb}
    kin["default"] = timed(lambda: aggregate_packed(s, off, "default"), args.windows, 3)
    kin["default"]["score_gb_per_s"] = gb / (kin["default"]["median_ms"] / 1e3)
    kin["top_k"] = timed(lambda: aggregate_packed(s, off, "top_k", k=5), args.windows, 3)
    vs = aggregate_packed(s, off, "default")
    lv = np.arange(19881, dtype=np.int32)
    kin["metrics"] = timed(lambda: video_metrics_packed(vs, lv, labels, 5, class_label=labels), args.windows, 3)
    other = torch.randn_like(vs)
    kin["fusion"] = timed(lambda: fuse_packed(vs, [other], [1.5]), args.windows, 10)
    sample = list(range(args.sample))
    hs = s[:int(off[args.sample])].cpu().numpy()
    kin["oracle_one_core_s"] = cpu_per_video(lambda x: O.default_agg(x), hs, off, sample) * 19881
    hv = vs.cpu().numpy()
    t = time.perf_counter()
    O.video_mean_ap(hv[:2000], [{int(c)} for c in labels[:2000]])
    kin["oracle_video_mean_ap_2000_videos_s"] = time.perf_counter() - t
    if ref is not None:
        kin["reference_one_core_s"] = cpu_per_video(lambda x: ref[0].default_aggregation_func(x), hs, off, sample) * 19881
    res["kinetics"] = kin
    print(json.dumps(res))


if __name__ == "__main__":
    main()
