#!/usr/bin/env python
"""Benchmark of the tail of ssn_test.py's worker loop (:87-92: re-organised STPP + regression de-normalisation) on one H100;
prints ONE JSON line.

  python tools/bench_test_tail.py [--windows 7]

Two seeded synthetic test sets, tick scores already on the device:
  anet12    ActivityNet-1.2-like: 400 videos of 100..1500 ticks and 50..300 proposals, K = 100, (1,(1,2),1) (D = 1601),
            packed in batches of 200 videos (about 3.1 GB of scores + prefix tables per call)
  thumos14  THUMOS14-like: 213 videos of 500..5000 ticks and 1500..2500 proposals, K = 20, (1,(1,2),1) (D = 321), one batch
Two ways to the same tensors:
  loop    one STPPReorgainzed.forward per video (ssnb_stpp_reorg_prefix) and the reference's two torch lines
  packed  one ops.ssn_ops.reorg_packed call per batch (ssnb_stpp_reorg_batch, de-normalisation in the gather's epilogue)
A window is one pass over the whole set; CUDA events after a warm-up pass; median of `windows` windows with their range.
The packed outputs are compared bitwise with the loop's before timing.  Bytes are counted from the shapes: the scan reads the
scores once (4 B per tick and column) and writes the prefix tables (8 B), and the gather reads two doubles per pooled part
and column and writes the fp32 rows.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

CFG = (1, (1, 2), 1)
MULT = 5                                                   # pooled parts of (1,(1,2),1)
REG_STATS = np.array([[0.0123, -0.0457], [0.1789, 0.2345]])
# name -> (videos, ticks range, proposals range, K, videos per batch, seed)
SETS = (("anet12", (400, (100, 1500), (50, 300), 100, 200, 1)), ("thumos14", (213, (500, 5000), (1500, 2500), 20, 213, 2)))


def synth(V, t_rng, n_rng, K, seed, dev):
    """-> scores [sum T, D] (device), tick offsets, ticks32 [sum N, 4], scaling32 [sum N, 2] (device), row offsets"""
    import torch
    g = np.random.RandomState(seed)
    T = g.randint(t_rng[0], t_rng[1] + 1, V)
    N = g.randint(n_rng[0], n_rng[1] + 1, V)
    toff, off = np.concatenate([[0], np.cumsum(T)]), np.concatenate([[0], np.cumsum(N)])
    st = g.rand(off[-1]) * 0.9
    ed = np.minimum(st + g.rand(off[-1]) * 0.3 + 0.01, 1.0)
    dur = ed - st
    Tr = np.repeat(T, N).astype(np.float64)
    # ssn_dataset.py:406-428's ticks of the augmented proposal (starting / ending ratio 0.5)
    rs, re_ = np.maximum(0.0, st - dur / 2), np.minimum(1.0, ed + dur / 2)
    ticks = np.stack([rs * Tr, st * Tr, ed * Tr, re_ * Tr], 1).astype(np.int32)
    scaling = np.stack([(st - rs) / (dur / 2), (re_ - ed) / (dur / 2)], 1).astype(np.float32)
    D = K + 1 + MULT * 3 * K
    scores = torch.randn(int(toff[-1]), D, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
    return scores, toff.tolist(), torch.from_numpy(ticks).to(dev), torch.from_numpy(scaling).to(dev), off.tolist()


def model_bytes(T, V, N, K):
    D = K + 1 + MULT * 3 * K
    scan = T * D * 4 + (T + V) * D * 8
    gather = N * ((K + 1) * 2 * 8 + MULT * 3 * K * 2 * 8 + (K + 1 + 3 * K) * 4)
    return scan + gather


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_test_tail.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from bench_proposals import card_info
    from ops.ssn_ops import STPPReorgainzed, reorg_packed
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = {"metric": "test_tail_packed_ms_anet12", "unit": "ms", "higher_is_better": False, "windows": args.windows,
            "card": card_info(), "torch": torch.__version__}
    res = {}
    for name, (V, t_rng, n_rng, K, per_batch, seed) in SETS:
        scores, toff, ticks, sc, off = synth(V, t_rng, n_rng, K, seed, dev)
        D = scores.shape[1]
        reorg = STPPReorgainzed(D, K + 1, K, 2 * K, True, stpp_cfg=CFG)
        batches = [(b, min(b + per_batch, V)) for b in range(0, V, per_batch)]

        def loop():
            out = []
            for v in range(V):
                act, comp, reg = reorg.forward(scores[toff[v]:toff[v + 1]], ticks[off[v]:off[v + 1]], sc[off[v]:off[v + 1]])
                reg_scores = reg.view(-1, K, 2)                                    # ssn_test.py:89-92
                reg_scores[:, :, 0] = reg_scores[:, :, 0] * REG_STATS[1, 0] + REG_STATS[0, 0]
                reg_scores[:, :, 1] = reg_scores[:, :, 1] * REG_STATS[1, 1] + REG_STATS[0, 1]
                out.append((act, comp, reg_scores))
            return out

        def packed():
            out = []
            for b0, b1 in batches:
                t0, r0 = toff[b0], off[b0]
                out.append(reorg_packed(scores[t0:toff[b1]], [t - t0 for t in toff[b0:b1 + 1]], ticks[r0:off[b1]], sc[r0:off[b1]],
                                        [r - r0 for r in off[b0:b1 + 1]], CFG, K + 1, K, 2 * K, reg_stats=REG_STATS))
            return out

        lp, pk = loop(), packed()
        cat_l = [torch.cat([x[i] for x in lp]) for i in range(3)]
        cat_p = [torch.cat([x[i] for x in pk]) for i in range(3)]
        same = all(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)) for a, b in zip(cat_l, cat_p))
        del lp, pk, cat_l, cat_p
        row = {"videos": V, "ticks": toff[-1], "proposals": off[-1], "num_class": K, "D": D, "videos_per_batch": per_batch,
               "batches": len(batches), "packed_bitwise_equal_loop": bool(same),
               "peak_call_bytes": max((toff[b1] - toff[b0] + b1 - b0) * D * 8 + (toff[b1] - toff[b0]) * D * 4 for b0, b1 in batches),
               "model_bytes": model_bytes(toff[-1], V, off[-1], K)}
        for arm, fn in (("loop", loop), ("packed", packed), ("loop_again", loop), ("packed_again", packed)):
            fn()
            torch.cuda.synchronize()
            ms = []
            for _ in range(args.windows):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            row[arm + "_ms"], row[arm + "_ms_min"], row[arm + "_ms_max"] = float(np.median(ms)), float(min(ms)), float(max(ms))
        row["speedup"] = row["loop_ms"] / row["packed_ms"]
        row["packed_model_gb_per_s"] = row["model_bytes"] / row["packed_ms"] / 1e6
        res[name] = row
        del scores, ticks, sc
        torch.cuda.empty_cache()
    line["value"] = res["anet12"]["packed_ms"]
    line["datasets"] = res
    line["timing"] = ("CUDA events around one pass over the set after a warm-up pass; median of the windows, min and max beside "
                      "it; each arm timed twice (loop, packed, loop_again, packed_again)")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
