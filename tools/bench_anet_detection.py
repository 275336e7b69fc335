#!/usr/bin/env python
"""Benchmark of ActivityNet detection evaluation of a results file on one H100 (ops/detection_eval.py,
csrc/detection_ap.cu ssnb_detection_ap_rows); prints ONE JSON line.

  python tools/bench_anet_detection.py [--windows 7] [--calls 5] [--oracle-videos 300]
                                       [--toolkit DIR --toolkit-videos 300] [--no-gpu]

Two seeded synthetic sets at ActivityNet-1.3 validation shape: 4926 videos, 200 classes, 1..3 instances per video, 100 and
1000 result rows per video (0.49 M and 4.9 M rows), 10 tIoU thresholds np.linspace(0.5, 0.95, 10); about a third of a
video's rows are jittered copies of its instances, the rest random segments of random classes.
  gpu_ms            CUDA events around `calls` back-to-back detection_ap_rows + detection_report calls, from the packed device
                    tensors to ap on the host (the report copies it back, so every call ends in a synchronisation); median
                    window / calls after a warm-up, with the range of the windows
  load_pack_s       the loaders on the results JSON text (json.loads, load_anet_detection_ground_truth /
                    load_anet_detection_predictions, pack_anet_detection to the device), once
  oracle_cpu_s      the repository's numpy oracle (oracle/anet_detection_oracle.py, one CPU core) on the first `oracle-videos`
                    videos
  toolkit_cpu_s     with --toolkit pointing at the ActivityNet toolkit's Evaluation directory: its own
                    ANETdetection.evaluate (pandas, one core, check_status=False) on the first `toolkit-videos` videos
--no-gpu measures only the CPU columns.  The card's name, power limit and clocks are read in the same run.
"""
import argparse
import importlib.util
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

V, K = 4926, 200
SETS = (("anet_100", (100, 61)), ("anet_1000", (1000, 62)))


def synth_json(rows_per_video, seed):
    """-> (ground truth JSON, results JSON) as dicts"""
    g = np.random.RandomState(seed)
    names = ["class_%03d" % c for c in range(K)]
    n_gt = g.choice([1, 2, 3], V, p=[0.6, 0.3, 0.1])
    db, res = {}, {}
    for v in range(V):
        dur = float(30 + 200 * g.rand())
        anns = []
        for k in range(n_gt[v]):
            a, b = np.sort(g.rand(2) * dur)
            anns.append({"segment": [float(a), float(b)], "label": names[v % K if k == 0 else g.randint(K)]})
        vid = "v_%05d" % v
        db[vid] = {"subset": "validation", "duration": dur, "annotations": anns}
        n_copy = rows_per_video // 3
        pick = g.randint(0, len(anns), n_copy)
        a = np.array([anns[i]["segment"] for i in pick]).reshape(-1, 2)
        j = (a[:, 1:] - a[:, :1]) * 0.3 * (g.rand(n_copy, 2) * 2 - 1)
        seg = np.concatenate([a + j, np.sort(g.rand(rows_per_video - n_copy, 2) * dur, 1)])
        lab = [anns[i]["label"] for i in pick] + [names[c] for c in g.randint(0, K, rows_per_video - n_copy)]
        sc = g.rand(rows_per_video)
        res[vid] = [{"label": l_, "score": float(s_), "segment": [float(t0), float(t1)]} for l_, s_, (t0, t1) in zip(lab, sc, seg)]
    return ({"version": "VERSION 1.3", "taxonomy": [], "database": db},
            {"version": "VERSION 1.3", "results": res, "external_data": {}})


def first_videos(gt_j, pr_j, n):
    keep = list(gt_j["database"])[:n]
    return dict(gt_j, database={k: gt_j["database"][k] for k in keep}), dict(pr_j, results={k: pr_j["results"][k] for k in keep})


def toolkit_seconds(tk_dir, gt_j, pr_j):
    """the toolkit's ANETdetection(..., check_status=False).evaluate() from JSON files in a temporary directory"""
    sys.path.insert(0, tk_dir)
    np.float = float                                                  # eval_detection.py:231-232 under numpy 2
    spec = importlib.util.spec_from_file_location("tk_eval_detection", os.path.join(tk_dir, "eval_detection.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with tempfile.TemporaryDirectory() as d:
        gf, pf = os.path.join(d, "gt.json"), os.path.join(d, "pr.json")
        with open(gf, "w") as f:
            json.dump(gt_j, f)
        with open(pf, "w") as f:
            json.dump(pr_j, f)
        t0 = time.perf_counter()
        a = mod.ANETdetection(gf, pf, check_status=False)
        a.evaluate()
        return time.perf_counter() - t0, a.mAP


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--oracle-videos", type=int, default=300)
    ap.add_argument("--toolkit", default=None, help="the ActivityNet toolkit's Evaluation directory (its CPU time on a subset)")
    ap.add_argument("--toolkit-videos", type=int, default=300)
    ap.add_argument("--no-gpu", action="store_true", help="the CPU columns only")
    args = ap.parse_args()
    from oracle import anet_detection_oracle as O
    from ops import detection_eval as E
    line = {"metric": "anet_detection_gpu_ms_anet_100", "unit": "ms", "higher_is_better": False, "windows": args.windows,
            "calls_per_window": args.calls, "videos": V, "classes": K, "tiou_thresholds": E.TIOU_THRESHOLDS.tolist()}
    if not args.no_gpu:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("tools/bench_anet_detection.py measures the H100 path and needs a CUDA device (--no-gpu: CPU columns)")
        from bench_anet_proposals import timed
        from bench_proposals import card_info
        dev = torch.device("cuda:0")
        torch.cuda.set_device(dev)
        line.update(card=card_info(), torch=torch.__version__)
    res = {}
    for name, (per_video, seed) in SETS:
        gt_j, pr_j = synth_json(per_video, seed)
        texts = json.dumps(gt_j), json.dumps(pr_j)
        row = {"rows_per_video": per_video}
        # the oracle on the first videos
        gs, ps = first_videos(gt_j, pr_j, args.oracle_videos)
        g = E.load_anet_detection_ground_truth(gs)
        p = E.load_anet_detection_predictions(ps, g)
        off = np.concatenate([g["offsets"], np.full(len(p["video_ids"]) + 1 - len(g["offsets"]), g["offsets"][-1])])
        t0 = time.perf_counter()
        o = O.detection(p["video"], p["label"], p["seg"], p["score"], off, g["cls"], g["seg"], len(g["activity_index"]), E.TIOU_THRESHOLDS)
        row["oracle_videos"] = args.oracle_videos
        row["oracle_cpu_s"] = time.perf_counter() - t0
        row["oracle_cpu_s_per_video"] = row["oracle_cpu_s"] / args.oracle_videos
        if args.toolkit:
            row["toolkit_videos"] = args.toolkit_videos
            tk_s, tk_map = toolkit_seconds(args.toolkit, *first_videos(gt_j, pr_j, args.toolkit_videos))
            row["toolkit_cpu_s"] = tk_s
            row["toolkit_cpu_s_per_video"] = tk_s / args.toolkit_videos
            if args.toolkit_videos == args.oracle_videos:
                row["oracle_vs_toolkit_max_map_diff"] = float(np.abs(o["ap"].T.mean(axis=1) - tk_map).max())
        if not args.no_gpu:
            t0 = time.perf_counter()
            gt = E.load_anet_detection_ground_truth(json.loads(texts[0]))
            pr = E.load_anet_detection_predictions(json.loads(texts[1]), gt)
            pk = E.pack_anet_detection(gt, pr, dev)
            torch.cuda.synchronize()
            row["load_pack_s"] = time.perf_counter() - t0
            row["rows"] = int(pk["score"].numel())
            a = [pk[k] for k in ("video", "label", "seg", "score", "gt_offsets", "gt_cls", "gt_seg", "num_class")]

            def call():
                return E.detection_report(E.detection_ap_rows(*a))
            row.update(timed(call, args.calls, args.windows))
            rep = call()
            row["average_map"] = rep["average_map"]
            row["rows_per_s"] = row["rows"] / row["gpu_ms"] * 1e3
            # the GPU on the oracle's videos against the oracle
            pks = E.pack_anet_detection(g, p, dev)
            sub = E.detection_ap_rows(*[pks[k] for k in ("video", "label", "seg", "score", "gt_offsets", "gt_cls", "gt_seg", "num_class")])
            row["gpu_vs_oracle_max_ap_diff_first_videos"] = float(np.nanmax(np.abs(sub["ap"].cpu().numpy() - o["ap"])))
        res[name] = row
    line["value"] = None if args.no_gpu else res["anet_100"]["gpu_ms"]
    line["datasets"] = res
    line["timing"] = ("CUDA events around `calls` back-to-back detection_ap_rows + detection_report calls (device tensors to ap "
                      "on the host) after a warm-up call; median window / calls, with the windows' range")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
