#!/usr/bin/env python
"""Benchmark of a ragged test-time scoring loop on one H100: one reserved engine against one engine per frame count and
against padding every chunk; prints ONE JSON line.

  python tools/bench_ragged_test.py [--videos 16] [--chunk-ticks 40] [--crops 10] [--seed 0]

A THUMOS14-like set of videos (seeded tick counts, log-normal around 180 ticks, 40 to 1200), RGB, 10 crops, scored as
ssn_test.py does: SSN.test_scores over chunks of `chunk_ticks` ticks, so every video ends in a ragged chunk of 10 x (1 ..
chunk_ticks) frames.  Three ways of scoring the same chunks, for InceptionV3 and BNInception in EXACT_TC and FAST:

  reserved   base_model.reserve_frames(chunk_ticks x crops): one engine runs every chunk at its own frame count
  per_count  one engine per frame count, as without reserve_frames; `oom` records whether the card ran out of memory and
             `chunks_done` how far it got (InceptionV3 EXACT_TC plans about 106 MB per frame)
  padded     every chunk zero-padded to chunk_ticks x crops frames on one engine; only the real frames count

Per way: peak torch.cuda.max_memory_allocated, frames/s of real frames from CUDA events around the whole loop (engine
planning, allocation and weight packing included, after one warm-up call per precision), and the engines planned.  Seeded
synthetic weights and frames.  The card's name, power limit and SM clocks are read in the same run; the SM clock again
after each way.  Needs a CUDA device: without one it fails.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_inception_v3 import card_info  # noqa: E402


def sm_clock_mhz():
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=clocks.sm",
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    return out or None


def thumos_like_ticks(videos, seed):
    import numpy as np
    t = np.random.default_rng(seed).lognormal(np.log(180.0), 0.8, videos)
    return [int(v) for v in np.clip(np.rint(t), 40, 1200)]


def chunk_frames(ticks, chunk_ticks, crops):
    return [min(chunk_ticks, t - c) * crops for t in ticks for c in range(0, t, chunk_ticks)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--chunk-ticks", type=int, default=40)
    ap.add_argument("--crops", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_ragged_test.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    import ssn_models
    from oracle import inception_v3_oracle as IV
    from oracle import synth
    from ssn_b200 import _lib
    dev = torch.device("cuda:0")
    F = args.chunk_ticks * args.crops
    ticks = thumos_like_ticks(args.videos, args.seed)
    chunks = chunk_frames(ticks, args.chunk_ticks, args.crops)
    line = {"workload": "ragged_test_scoring", "videos": args.videos, "ticks": ticks, "chunks": len(chunks),
            "frames": sum(chunks), "distinct_frame_counts": len(set(chunks)), "chunk_ticks": args.chunk_ticks,
            "crops": args.crops, "card": card_info()}

    for arch, size, feat_dim in (("InceptionV3", IV.INPUT_SIZE, IV.FEAT_DIM), ("BNInception", 224, 1024)):
        w = IV.synth_weights(3, seed=0) if arch == "InceptionV3" else synth.synth_backbone(3, seed=0, calib_frames=2)
        m = ssn_models.SSN(20, 2, 5, 2, "RGB", base_model=arch, dropout=0, test_mode=True)
        sd = m.state_dict()
        with torch.no_grad():
            for k, v in w.items():
                sd["base_model." + k].copy_(v)
            for k, v in synth.synth_heads(20, m.stpp.feat_multiplier, feat_dim=feat_dim, seed=0, std=0.02, bias_std=0.1).items():
                sd[k].copy_(v)
        m.prepare_test_fc()
        m = m.to(dev).eval()
        x = synth.synth_frames(F, 3, size, seed=3).to(dev)
        pad = torch.zeros_like(x)
        for pname, prec in (("exact_tc", _lib.EXACT_TC), ("fast", _lib.FAST_FP16)):
            res = {}
            for way in ("reserved", "per_count", "padded"):
                m.set_precision(prec, 1024.0)                     # drops every engine of the previous way
                m.base_model.reserve_frames(F if way == "reserved" else None)
                torch.cuda.empty_cache()
                m.test_scores(x[:args.crops], num_crop=args.crops)   # warm-up: module loads, kernel attributes
                m.base_model._engines.clear()
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                done, oom = 0, False
                a.record()
                try:
                    for n in chunks:
                        if way == "padded":
                            pad[:n].copy_(x[:n])
                            m.test_scores(pad, num_crop=args.crops)
                        else:
                            m.test_scores(x[:n], num_crop=args.crops)
                        done += 1
                except torch.cuda.OutOfMemoryError:
                    oom = True
                b.record()
                b.synchronize()
                ms = a.elapsed_time(b)
                real = sum(chunks[:done])
                res[way] = {"oom": oom, "chunks_done": done, "engines": len(m.base_model._engines),
                            "peak_allocated_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2), "ms": round(ms, 1),
                            "frames_per_s": round(real / ms * 1e3, 1) if done else None, "sm_mhz_after": sm_clock_mhz()}
                m.base_model._engines.clear()
                torch.cuda.empty_cache()
            line["%s_%s" % (arch, pname)] = res
        del m, x, pad
        torch.cuda.empty_cache()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
