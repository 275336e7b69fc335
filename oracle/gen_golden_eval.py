"""tests/golden/eval.npz from the REAL reference (build container only: python -m oracle.gen_golden_eval).

eval_detection_results.py is a script (argparse, dataset loading and a process pool at import time), so merge_scores,
gen_detection_results, perform_regression and ravel_detections are compiled from the functions' own source text with ast --
the reference's code, unedited -- in a namespace that supplies the script's globals (score_pickle_list, weights, top_k,
num_class, cls_score_dict, softmax_bf, args, dataset_detections).  temporal_nms is imported from ops/utils.py, and
compute_average_precision_detection from anet_toolkit/Evaluation/eval_detection.py, imported as a module only (with
np.float = float, which numpy 2 removed and :229 uses); nothing that reaches the network is called.  The AP jobs run the
toolkit function per (class, threshold) exactly as eval_ap does (:219-227), serially.

Weights are given as Python floats: the script's default 1/n weights are, and numpy 2 keeps the fp32 arrays fp32 under them
(an np.float64 weight array, as --score_weights builds, would promote the merged scores to float64).

Each fixture is re-seeded until no two scores of one ranked list (the top-k argsort, an NMS list, a class-wide AP list) lie
within 1e-5 relative of each other and no tIoU lies within 1e-6 of a threshold, so that the numpy sort order, which ties
leave open, is the only one."""
import ast
import os
import sys
import types

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")

# name, K, videos, N range, mode, top_k, cls_top_k, softmax_bf, nms, thresholds, sources, weights, regress, reg None
FIXTURES = (
    ("thumos", 20, 7, (4, 60), "top_k", 40, 1, True, 0.2, "thumos", 2, None, True, False),
    ("anet", 30, 6, (3, 40), "top_k", 60, 1, False, 0.6, "anet", 2, (2.0, 1.0), True, False),
    ("all", 5, 5, (2, 30), "all", 0, 1, True, 0.3, "thumos", 1, None, False, True),
    ("cls_sbf", 8, 5, (3, 30), "cls", 0, 1, True, 0.4, "thumos", 1, None, True, False),
    ("cls_raw", 8, 5, (3, 30), "cls", 0, 3, False, 0.4, "anet", 1, None, True, True),
)


def thresholds(kind):
    return np.arange(0.1, 1.0, 0.1) if kind == "thumos" else np.arange(0.5, 1.0, 0.05)


def synth(fx, seed):
    """-> (sources: list of {vid: (rel_props, act, comp, reg)}, cls_scores {path: [K]}, gt [(vid, cls, t0, t1)])"""
    name, K, V, (n_lo, n_hi), mode, _, _, _, _, _, n_src, _, _, reg_none = fx
    g = np.random.RandomState(seed)
    vids = ["video_%s_%02d" % (name, v) for v in range(V)]
    srcs = [dict() for _ in range(n_src)]
    gt = []
    for v, vid in enumerate(vids):
        n = int(g.randint(n_lo, n_hi + 1))
        c = g.rand(n)
        d = 0.02 + 0.3 * g.rand(n)
        rel = np.stack([np.clip(c - d / 2, 0, 1), np.clip(c + d / 2, 0, 1)], 1).astype(np.float32)
        if v == 2:
            rel = rel[None]                                   # 3-D rel_props (eval_detection_results.py:92-93)
        for s in range(n_src):
            act = (g.randn(n, K + 1) * 2).astype(np.float32)
            comp = g.randn(n, K).astype(np.float32)
            if mode == "top_k":
                comp[:, K - 1] -= 30.0                        # the last class never reaches the top k: 0 AP
            reg = None if reg_none else (g.randn(n, K * 2) * 0.3).astype(np.float32)
            if reg is not None and v == 1:                    # boxes regressed onto [0, 0] and [1, 1]
                reg.reshape(n, K, 2)[0, :, :] = (-60.0, 0.0)
                reg.reshape(n, K, 2)[1, :, :] = (60.0, 0.0)
            srcs[s][vid] = (rel, act, comp, reg)
        # ground truth: frame / num_frames; video 0 has none, class 0 has none anywhere (NaN AP where it has detections)
        if v != 0:
            frames = int(g.randint(300, 3000))
            for _ in range(int(g.randint(1, 8))):
                cls = int(g.randint(1, K))
                a = int(g.randint(0, frames - 10))
                b = a + int(g.randint(5, frames // 3))
                gt.append((vid, cls, a / frames, min(b, frames) / frames))
            if v == 1:                                        # zero-length ground truth at both ends: NaN tIoU
                for cls in range(1, K):
                    gt.append((vid, cls, 0.0, 0.0))
                    gt.append((vid, cls, 1.0, 1.0))
    gt.append(("video_%s_nodet" % name, 1, 0.1, 0.3))          # a video without detections: counts in npos only
    cls_scores = {"/data/%s.mp4" % vid: g.randn(K).astype(np.float32) for vid in vids}
    return srcs, cls_scores, gt


def load_reference():
    sys.path.insert(0, REF)
    sys.path.insert(0, os.path.join(REF, "anet_toolkit", "Evaluation"))
    import yaml
    _orig = yaml.load
    yaml.load = lambda s, Loader=yaml.SafeLoader: _orig(s, Loader=Loader)
    np.float = float                                           # eval_detection.py:229 (numpy 2 removed the alias)
    import pandas as pd
    from ops.utils import temporal_nms, softmax
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_eval_detection", os.path.join(REF, "anet_toolkit", "Evaluation", "eval_detection.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    src = open(os.path.join(REF, "eval_detection_results.py")).read()
    fns = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef)
           and n.name in ("merge_scores", "gen_detection_results", "perform_regression", "ravel_detections")]
    code = compile(ast.Module(body=fns, type_ignores=[]), "eval_detection_results.py", "exec")
    return pd, temporal_nms, softmax, mod.compute_average_precision_detection, code


def run_reference(fx, srcs, cls_scores, gt, ref):
    pd, temporal_nms, softmax, compute_ap, code = ref
    name, K, V, _, mode, top_k, cls_top_k, sbf, nms, thr_kind, n_src, weights, regress, _ = fx
    w = [1.0 / n_src] * n_src if weights is None else [float(x) / sum(weights) for x in weights]
    ns = {"np": np, "os": os, "pd": pd, "softmax": softmax, "score_pickle_list": srcs, "weights": w,
          "top_k": top_k if mode == "top_k" else 0, "num_class": K, "softmax_bf": sbf,
          "cls_score_dict": ({os.path.splitext(os.path.basename(k))[0]: v for k, v in cls_scores.items()} if mode == "cls" else None),
          "args": types.SimpleNamespace(cls_top_k=cls_top_k), "dataset_detections": [dict() for _ in range(K)]}
    exec(code, ns)
    detection_scores = {k: ns["merge_scores"](k) for k in srcs[0]}
    for k, v in detection_scores.items():
        ns["gen_detection_results"](k, v)
    dd = ns["dataset_detections"]
    for c in range(K):
        dd[c] = {k: temporal_nms(v, nms) for k, v in dd[c].items()}
    if regress:
        for c in range(K):
            dd[c] = {k: ns["perform_regression"](v) for k, v in dd[c].items()}
    plain = [ns["ravel_detections"](dd, c) for c in range(K)]
    all_gt = pd.DataFrame(gt, columns=["video-id", "cls", "t-start", "t-end"])
    gt_by_cls = [all_gt[all_gt.cls == c].reset_index(drop=True).drop(columns="cls") for c in range(K)]
    thr = thresholds(thr_kind)
    ap = np.empty((K, len(thr)))
    for t, min_overlap in enumerate(thr):
        for c in range(K):
            ap[c, t] = compute_ap(gt_by_cls[c], plain[c], [min_overlap])[0]
    return detection_scores, dd, plain, ap


def margins_ok(fx, srcs, dd, gt, detection_scores):
    """no two scores of a ranked list within 1e-5 relative, no tIoU within 1e-6 of a threshold"""
    from oracle import eval_oracle as D
    name, K, V, _, mode, top_k, _, sbf, _, thr_kind, *_ = fx

    def close(s):
        s = np.sort(np.asarray(s, np.float64)[np.isfinite(s)])
        return len(s) > 1 and bool((np.diff(s) <= 1e-5 * np.abs(s[1:])).any())
    for vid, (rel, act, comp, reg) in detection_scores.items():
        cb = D.branch_scores(act, comp, mode, sbf)
        if close(cb.ravel()) if mode == "top_k" else any(close(cb[:, c]) for c in range(K)):
            return False
    thr = thresholds(thr_kind)
    for c in range(K):
        rows = [r for r in dd[c].values()]
        if rows and close(np.concatenate(rows)[:, 2]):
            return False
        for vid, r in dd[c].items():
            g = np.array([(a, b) for v, k, a, b in gt if v == vid and k == c], np.float64).reshape(-1, 2)
            for x in r:
                tiou = D.segment_iou(np.asarray(x[:2], np.float64), g)
                fin = tiou[np.isfinite(tiou)]
                if len(fin) and (np.abs(fin[:, None] - thr[None]) < 1e-6).any():
                    return False
    return True


def main():
    ref = load_reference()
    out = {}
    for fi, fx in enumerate(FIXTURES):
        name = fx[0]
        seed = 100 * fi + 1
        while True:
            srcs, cls_scores, gt = synth(fx, seed)
            detection_scores, dd, plain, ap = run_reference(fx, srcs, cls_scores, gt, ref)
            if margins_ok(fx, srcs, dd, gt, detection_scores):
                break
            seed += 1000
        vids = list(srcs[0])
        pre = name + "_"
        out[pre + "seed"] = np.int64(seed)
        out[pre + "ap"] = ap
        # post-NMS / regression detections: per class, the rows of every video in video order, with the video index
        K = fx[1]
        for c in range(K):
            rows = [(vids.index(v), r) for v, r in dd[c].items()]
            out[pre + "det_%d" % c] = (np.concatenate([r for _, r in rows]).astype(np.float64) if rows else np.zeros((0, 5)))
            out[pre + "det_video_%d" % c] = np.concatenate([np.full(len(r), vi) for vi, r in rows]).astype(np.int64) if rows else np.zeros(0, np.int64)
            p = plain[c]
            out[pre + "pred_%d" % c] = p[["t-start", "t-end", "score"]].to_numpy(np.float64) if len(p) else np.zeros((0, 3))
        print("%s: seed %d, %d detections, mAP %s" % (name, seed, sum(len(r) for c in range(K) for r in dd[c].values()),
                                                     np.round(np.nanmean(ap, 0), 4)))
    np.savez_compressed(os.path.join(GOLD, "eval.npz"), **out)
    print("wrote eval.npz:", len(out), "arrays")


if __name__ == "__main__":
    main()
