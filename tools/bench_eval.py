#!/usr/bin/env python
"""Benchmark of detection evaluation on one H100 (ops/detection.py detections_packed + detection_ap; csrc/detect.cu,
csrc/detection_ap.cu); prints ONE JSON line.

  python tools/bench_eval.py [--steps 5] [--oracle-videos 40]

Two seeded synthetic sets with the shapes of the shipped test sets (tests/test_gpu_eval.synth_set):
  thumos  1574 videos, K 20, N median ~111 (max 2914), top_k 2000, NMS 0.2, tIoU 0.1:0.9 (9 thresholds)
  anet    2383 videos, K 100, N median ~45 (max 187), top_k 60, NMS 0.6, tIoU 0.5:0.95 (10 thresholds)
GPU time from packed scores (already on the device) to the AP table [K, n_thr], both library calls, measured with CUDA
events after one warm-up call, over `steps` passes.  For comparison the repository's numpy oracle (oracle/eval_oracle.py,
one CPU core) runs gen_detection_results + NMS + regression and the AP of every class on the first `oracle-videos` videos.
The reference script itself (pandas, a 32-process pool) is not measured here.  The card's name and power limit are read in
the same run.  Needs a CUDA device: without one it fails.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--oracle-videos", type=int, default=40)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_eval.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from bench_proposals import card_info
    from ops.detection import detections_packed, detection_ap
    from oracle import eval_oracle as D
    from test_gpu_eval import synth_set
    torch.cuda.set_device(0)
    res = {}
    for name, top_k, nms, thr, seed in (("thumos", 2000, 0.2, np.arange(0.1, 1.0, 0.1), 11), ("anet", 60, 0.6, np.arange(0.5, 1.0, 0.05), 12)):
        props, act, comp, reg, offsets, K, gt = synth_set(name, seed)
        T = lambda x: torch.tensor(x, device="cuda")
        tp_, ta, tc, tr = T(props), T(act), T(comp), T(reg)

        def run():
            d = detections_packed(tp_, ta, tc, tr, offsets, nms, mode="top_k", top_k=top_k)
            return d, detection_ap(d, gt, thr)["ap"]
        d, a = run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        # the numpy oracle on the first videos, one CPU core
        nv = min(args.oracle_videos, len(offsets) - 1)
        t0 = time.perf_counter()
        dets = {}
        for v in range(nv):
            lo, hi = offsets[v], offsets[v + 1]
            for c, rows in D.video_detections_branch(props[lo:hi], act[lo:hi], comp[lo:hi], reg[lo:hi], nms, "top_k", top_k).items():
                dets.setdefault(c, []).append((v, rows))
        gcls, gseg, goff = gt["cls"].cpu().numpy(), gt["seg"].cpu().numpy(), gt["offsets"]
        gl = [(v, int(gcls[i]), gseg[i, 0], gseg[i, 1]) for v in range(nv) for i in range(goff[v], goff[v + 1])]
        D.ap_table(dets, gl, K, thr)
        oracle_s = time.perf_counter() - t0
        res[name] = {"videos": len(offsets) - 1, "proposals": offsets[-1], "num_class": K, "top_k": top_k, "nms_threshold": nms,
                     "thresholds": len(thr), "ground_truth": int(gt["cls"].numel()), "survivors": int(d["counts"].sum()),
                     "gpu_ms": float(np.median(ms)), "gpu_ms_min": float(min(ms)), "gpu_ms_max": float(max(ms)),
                     "oracle_videos": nv, "oracle_cpu_s": oracle_s, "oracle_cpu_s_per_video": oracle_s / nv,
                     "mAP": [float(x) for x in np.nanmean(a.cpu().numpy(), 0)]}
    line = {"metric": "detection_eval_gpu_ms_thumos", "value": res["thumos"]["gpu_ms"], "unit": "ms", "higher_is_better": False,
            "steps": args.steps, "datasets": res, "reference_script": "not measured (pandas + process pool; it does not run on the GPU machine)",
            "timing": "CUDA events around detections_packed + detection_ap, after one warm-up call; median over steps",
            "card": card_info(), "torch": torch.__version__}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
