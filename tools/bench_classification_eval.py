#!/usr/bin/env python
"""Benchmark of untrimmed video classification evaluation on one H100 (ops/classification_eval.py,
csrc/classification_ap.cu); prints ONE JSON line.

  python tools/bench_classification_eval.py [--windows 7] [--calls 10] [--toolkit DIR --toolkit-videos 300] [--no-gpu]

Three seeded synthetic sets, predictions and ground truth already packed on the device:
  anet_dense      4926 videos (ActivityNet-1.3 validation) x 200 classes, every class of every video a prediction (~0.99 M
                  rows), 1..3 ground-truth labels per video; top_k 3
  kinetics_top5   19881 videos (Kinetics-400 validation) x their 5 highest of 400 classes (~0.1 M rows), one label each; top_k 1
                  and 5 (the toolkit's eval_kinetics.py error@1 and error@5)
  kinetics_dense  the same videos x all 400 classes (~8 M rows); top_k 1 and 5
Timed with CUDA events after a warm-up: a window is `calls` back-to-back classification_ap_packed + classification_report
calls per top_k (the report copies the results to the host, so every call ends in a synchronisation); the figure is the
median window / calls, for all of a set's top_k values together.  For comparison the repository's numpy oracle
(oracle/anet_classification_oracle.py, one CPU core) evaluates the whole set once per top_k, and, with --toolkit pointing at
the ActivityNet toolkit's Evaluation directory, the toolkit's own ANETclassification.evaluate (pandas, one core) evaluates
the first `toolkit-videos` videos.  --no-gpu measures only these CPU columns.  The card's name and power limit are read in
the same run.
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

SETS = (("anet_dense", (4926, 200, None, (3,), 41)), ("kinetics_top5", (19881, 400, 5, (1, 5), 42)),
        ("kinetics_dense", (19881, 400, None, (1, 5), 42)))


def synth(V, K, keep, seed):
    """-> (video, label, score, gt_video, gt_label): scores a noisy one-hot of a video's first label; keep: the top `keep`
    classes of each video only (a top-k submission), else all K"""
    g = np.random.RandomState(seed)
    n_lab = g.choice([1, 2, 3], V, p=[0.85, 0.1, 0.05]) if K == 200 else np.ones(V, np.int64)
    gv = np.repeat(np.arange(V), n_lab).astype(np.int32)
    gl = g.randint(0, K, len(gv)).astype(np.int32)
    S = g.rand(V, K)
    first = np.concatenate([[0], np.cumsum(n_lab)[:-1]])
    S[np.arange(V), gl[first]] += g.rand(V) * 1.5
    if keep is None:
        return np.repeat(np.arange(V, dtype=np.int32), K), np.tile(np.arange(K, dtype=np.int32), V), S.reshape(-1), gv, gl
    top = np.argsort(-S, 1)[:, :keep]
    return (np.repeat(np.arange(V, dtype=np.int32), keep), top.reshape(-1).astype(np.int32),
            np.take_along_axis(S, top, 1).reshape(-1), gv, gl)


def toolkit_seconds(tk_dir, video, label, score, gv, gl, n_videos, top_k):
    """the toolkit's evaluate() on the rows of the first n_videos videos, from JSON files in a temporary directory"""
    sys.path.insert(0, tk_dir)
    np.float = float                                                  # eval_classification.py:206-207 under numpy 2
    spec = importlib.util.spec_from_file_location("tk_eval_classification", os.path.join(tk_dir, "eval_classification.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    names = ["c%03d" % c for c in range(int(max(label.max(), gl.max())) + 1)]
    db = {"v%05d" % v: {"subset": "validation", "annotations": []} for v in range(n_videos)}
    for v, c in zip(gv, gl):
        if v < n_videos:
            db["v%05d" % v]["annotations"].append({"label": names[c], "segment": [0.0, 1.0]})
    res = {}
    for v, c, s in zip(video, label, score):
        if v < n_videos:
            res.setdefault("v%05d" % v, []).append({"label": names[c], "score": float(s)})
    used = {a["label"] for d in db.values() for a in d["annotations"]}
    res = {v: [r for r in rs if r["label"] in used] for v, rs in res.items()}
    with tempfile.TemporaryDirectory() as d:
        gf, pf = os.path.join(d, "gt.json"), os.path.join(d, "pr.json")
        json.dump({"database": db, "taxonomy": [], "version": ""}, open(gf, "w"))
        json.dump({"results": res, "version": "", "external_data": {}}, open(pf, "w"))
        t0 = time.perf_counter()
        a = mod.ANETclassification(gf, pf, top_k=top_k, check_status=False)
        a.evaluate()
        return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--toolkit", default=None, help="the ActivityNet toolkit's Evaluation directory (its CPU time on a subset)")
    ap.add_argument("--toolkit-videos", type=int, default=300)
    ap.add_argument("--no-gpu", action="store_true", help="the CPU columns only")
    args = ap.parse_args()
    from oracle import anet_classification_oracle as O
    line = {"metric": "anet_classification_gpu_ms_anet_dense", "unit": "ms", "higher_is_better": False, "windows": args.windows,
            "calls_per_window": args.calls}
    if not args.no_gpu:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("tools/bench_classification_eval.py measures the H100 path and needs a CUDA device (--no-gpu: CPU columns)")
        from bench_anet_proposals import timed
        from bench_proposals import card_info
        from ops import classification_eval as E
        dev = torch.device("cuda:0")
        torch.cuda.set_device(dev)
        line.update(card=card_info(), torch=torch.__version__)
    res = {}
    for name, (V, K, keep, ks, seed) in SETS:
        video, label, score, gv, gl = synth(V, K, keep, seed)
        row = {"videos": V, "classes": K, "rows": int(len(score)), "ground_truth_pairs": int(len(gv)), "top_k": list(ks)}
        t0 = time.perf_counter()
        want = {k: O.classification(video, label, score, gv, gl, V, K, k) for k in ks}
        row["oracle_cpu_s"] = time.perf_counter() - t0
        for k in ks:
            row["map"] = float(want[k]["ap"].mean())
            row["hit_at_%d" % k] = want[k]["hit_at_k"]
        if args.toolkit:
            nv = min(args.toolkit_videos, V)
            row["toolkit_videos"] = nv
            row["toolkit_cpu_s"] = sum(toolkit_seconds(args.toolkit, video, label, score, gv, gl, nv, k) for k in ks)
            row["toolkit_cpu_s_per_video"] = row["toolkit_cpu_s"] / nv
        if not args.no_gpu:
            tens = [torch.as_tensor(x).to(dev) for x in (video, label, score, gv, gl)]

            def call():
                return [E.classification_report(E.classification_ap_packed(*tens, V, K, k)) for k in ks]
            row.update(timed(call, args.calls, args.windows))
            got = call()
            row["gpu_vs_oracle_max_ap_diff"] = max(float(np.abs(r["ap"] - want[k]["ap"]).max()) for r, k in zip(got, ks))
            row["gpu_hits_equal_oracle"] = all(r["hit_at_k"] == want[k]["hit_at_k"] for r, k in zip(got, ks))
            row["rows_per_s"] = len(ks) * len(score) / row["gpu_ms"] * 1e3
            row["speedup_vs_oracle"] = row["oracle_cpu_s"] * 1e3 / row["gpu_ms"]
        res[name] = row
    line["value"] = None if args.no_gpu else res["anet_dense"]["gpu_ms"]
    line["datasets"] = res
    line["timing"] = ("CUDA events around `calls` back-to-back classification_ap_packed + classification_report calls per top_k "
                      "after a warm-up call; median window / calls")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
