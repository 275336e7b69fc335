"""tests/golden/proposals.npz from the REAL reference (build container only: python -m oracle.gen_golden_proposals), and
tests/golden/proposals_nms.npz, the reference's NMS on random box lists (python -m oracle.gen_golden_proposals nms).

ops/sequence_funcs.py imports cleanly once the reference root is on sys.path (ops/metrics.py pulls in sklearn; the
optional GPU `nms.nms_wrapper` is absent, so temporal_nms runs temporal_nms_fallback).  gen_bottom_up_proposals.py is a
script (argparse and dataset loading at import time), so gen_prop and the score-merge loop (:76-91) are compiled from the
script's own source text with ast — the reference's code, unedited — and run in a namespace that supplies the globals they
read (args, score_dict, reg_score_dict).  label_frame_by_threshold / build_box_by_search / temporal_nms are wrapped to
record what they return; the wrappers can also replace the thresholds, tolerances or bw that gen_prop hard-codes, for the
fixtures that exercise other values.

Every fixture is re-seeded until (a) no smoothed value (softmax value when bw is None) lies within 1e-6 of an fp32
threshold, so the <= 1 ulp differences between CUDA's expf and numpy's exp cannot flip a label, (b) no two distinct boxes
with bitwise-equal scores have IoU > nms threshold, so the survivor set does not depend on how ties are ordered, and
(c) the survivors have pairwise distinct scores, so their order is the reference's order whatever the tie rule.
"""
import ast
import os
import sys
import types

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
MARGIN = 1e-6


def _script_nodes():
    src = open(os.path.join(REF, "gen_bottom_up_proposals.py")).read()
    body = ast.parse(src).body
    gen_prop = [n for n in body if isinstance(n, ast.FunctionDef) and n.name == "gen_prop"][0]
    # the first module-level `for key in score_list[0].keys():` is the score merge (:79-90)
    merge = [n for n in body if isinstance(n, ast.For) and isinstance(n.target, ast.Name) and n.target.id == "key"][0]
    return gen_prop, merge


def synth_logits(T, seed, kind, K=2):
    """[T, K] fp32 crop-mean scores; column 1 is the foreground logit, the rest is background"""
    g = np.random.RandomState(seed)
    f = (g.randn(T, K) * 0.3).astype(np.float32)
    if kind == "smooth":
        walk = np.cumsum(g.randn(T)) * 0.35
        walk -= np.convolve(walk, np.ones(min(T, 301)) / min(T, 301), mode="same")
        f[:, 1] += (walk + 0.4 * g.randn(T)).astype(np.float32)
    elif kind == "noisy":
        f[:, 1] += (np.cumsum(g.randn(T)) * 0.05 + 7.0 * g.randn(T)).astype(np.float32)
    elif kind == "all_fg":
        f[:, 1] += 9.0
    elif kind == "all_bg":
        f[:, 1] -= 9.0
    elif kind == "edges":                       # foreground at the first and the last frame, background between
        x = np.linspace(-1, 1, T)
        f[:, 1] += (12 * x * x - 5).astype(np.float32)
    elif kind == "alternating":
        f[:, 1] += np.where(np.arange(T) % 2 == 0, 4.0, -4.0).astype(np.float32) + (g.randn(T) * 2.5).astype(np.float32)
    return f


def _margin_ok(sm, thresholds):
    return all(np.abs(sm.astype(np.float64) - float(np.float32(th))).min() > MARGIN for th in thresholds) if len(sm) else True


def _ties_ok(s, e, sc, thresh):
    bits = sc.view(np.uint32)
    uniq = {}
    for a, b, k in zip(s.tolist(), e.tolist(), bits.tolist()):
        uniq.setdefault(k, set()).add((a, b))
    for k, boxes in uniq.items():
        boxes = sorted(boxes)
        for i in range(len(boxes)):
            for j in range(i + 1, len(boxes)):
                (a1, b1), (a2, b2) = boxes[i], boxes[j]
                inter = min(b1, b2) - max(a1, a2) + 1
                if inter / float((b1 - a1 + 1) + (b2 - a2 + 1) - inter) > thresh:
                    return False
    return True


def main():
    sys.path.insert(0, REF)
    import ops.sequence_funcs as SF
    from ops.metrics import softmax
    from scipy.ndimage import gaussian_filter
    assert SF.nms is None, "the reference's optional GPU nms is importable; temporal_nms would not be the fallback"
    gen_prop_node, merge_node = _script_nodes()
    gen_code = compile(ast.Module(body=[gen_prop_node], type_ignores=[]), "gen_bottom_up_proposals.py", "exec")
    merge_code = compile(ast.Module(body=[merge_node], type_ignores=[]), "gen_bottom_up_proposals.py", "exec")

    def run_gen_prop(f_score, duration, bw=3, thresholds=None, tolerances=None, minimum_len=0.0):
        rec = {}

        def label_frame_by_threshold(score_mat, cls_lst, bw=None, thresh=None, multicrop=True):
            rec["thresholds"] = thresh if thresholds is None else list(thresholds)
            rec["bw"] = bw if bw_override is False else bw_override
            out = SF.label_frame_by_threshold(score_mat, cls_lst, bw=rec["bw"], thresh=rec["thresholds"], multicrop=multicrop)
            rec["labels"] = np.stack([x[1] for x in out])
            return out

        def build_box_by_search(frm_label_lst, tol, min=1):
            rec["tolerances"] = np.asarray(tol if tolerances is None else tolerances, np.float64)
            out = SF.build_box_by_search(frm_label_lst, rec["tolerances"])
            rec["raw"] = out
            return out

        def temporal_nms(bboxes, thresh):
            rec["nms_thresh"] = thresh
            out = SF.temporal_nms(bboxes, thresh)
            rec["kept"] = out
            return out
        bw_override = False if bw == 3 else bw
        ns = {"np": np, "args": types.SimpleNamespace(dataset="thumos14", minimum_len=minimum_len),
              "score_dict": {"v": f_score}, "reg_score_dict": None, "label_frame_by_threshold": label_frame_by_threshold,
              "build_box_by_search": build_box_by_search, "temporal_nms": temporal_nms}
        exec(gen_code, ns)
        vid, pr_box, scores = ns["gen_prop"](types.SimpleNamespace(id="v", duration=duration, path="v.mp4"))
        ss = softmax(f_score)
        rec["ss"] = ss
        rec["smoothed"] = ss[:, 1] if rec["bw"] is None else gaussian_filter(ss[:, 1], rec["bw"])
        rec["pr_box"] = np.array(pr_box, np.float64).reshape(-1, 2)
        rec["pr_score_ref"] = np.array(scores, np.float32)
        return rec

    def merge(streams, weights):
        ns = {"score_list": [{"v": s} for s in streams], "args": types.SimpleNamespace(score_weights=weights), "score_dict": {}}
        exec(merge_code, ns)
        return ns["score_dict"]["v"]

    fixtures = [                                   # tag, T, kind, K, bw, thresholds, tolerances, minimum_len
        ("t1", 1, "smooth", 2, 3, None, None, 0.0),
        ("t2", 2, "smooth", 2, 3, None, None, 0.0),
        ("t5", 5, "smooth", 2, 3, None, None, 0.0),
        ("t13", 13, "smooth", 2, 3, None, None, 0.0),
        ("t700", 700, "smooth", 3, 3, None, None, 0.0),
        ("t3000", 3000, "smooth", 2, 3, None, None, 0.0),
        ("noisy", 12000, "noisy", 2, 3, None, None, 0.0),
        ("all_fg", 300, "all_fg", 2, 3, None, None, 0.0),
        ("all_bg", 300, "all_bg", 2, 3, None, None, 0.0),
        ("edges", 400, "edges", 2, 3, None, None, 0.0),
        ("alt", 600, "alternating", 2, None, None, None, 0.0),
        ("custom", 900, "smooth", 2, 2, (0.3, 0.45, 0.62, 0.77), (0.15, 0.45, 0.7, 0.95, 1.3), 0.0),
        ("minlen", 1500, "smooth", 2, 3, None, None, 4.0),
    ]
    def boxes(rec):
        raw, kept = rec["raw"], rec["kept"]
        return (np.array([b[0] for b in raw], np.int64), np.array([b[1] for b in raw], np.int64), np.array([b[3] for b in raw], np.float32),
                np.array([b[0] for b in kept], np.int64), np.array([b[1] for b in kept], np.int64), np.array([b[3] for b in kept], np.float32))

    def conditions_ok(rec):
        s, e, sc, _, _, ksc = boxes(rec)
        return (_margin_ok(rec["smoothed"], rec["thresholds"]) and _ties_ok(s, e, sc, rec["nms_thresh"])
                and len(np.unique(ksc.view(np.uint32))) == len(ksc))

    def store(out, tag, f, duration, seed, rec, min_len):
        s, e, sc, ks, ke, ksc = boxes(rec)
        p = tag + "_"
        out.update({p + "f_score": f, p + "duration": np.float64(duration), p + "seed": np.int64(seed),
                    p + "bw": np.float64(-1.0 if rec["bw"] is None else rec["bw"]),
                    p + "thresholds": np.asarray(rec["thresholds"], np.float64), p + "tolerances": rec["tolerances"],
                    p + "nms_thresh": np.float64(rec["nms_thresh"]), p + "minimum_len": np.float64(min_len),
                    p + "ss": rec["ss"], p + "smoothed": np.asarray(rec["smoothed"], np.float32), p + "labels": rec["labels"],
                    p + "raw_start": s, p + "raw_end": e, p + "raw_score": sc, p + "nms_start": ks, p + "nms_end": ke,
                    p + "nms_score": ksc, p + "pr_box": rec["pr_box"], p + "pr_score_ref": rec["pr_score_ref"]})
        print("%-7s T=%-6d seed %d: %d raw boxes, %d distinct, %d kept, %d in pr_box" % (
            tag, len(f), seed, len(s), len(set(zip(s.tolist(), e.tolist(), sc.view(np.uint32).tolist()))), len(ks),
            len(rec["pr_box"])))

    out = {"tags": np.array([f[0] for f in fixtures] + ["merge"])}
    for tag, T, kind, K, bw, thr, tol, min_len in fixtures:
        for seed in range(1000, 1200):
            f = synth_logits(T, seed, kind, K)
            duration = float(np.random.RandomState(seed).uniform(0.5, 3.0) * T / 10.0)
            rec = run_gen_prop(f, duration, bw=bw, thresholds=thr, tolerances=tol, minimum_len=min_len)
            if conditions_ok(rec):
                break
        else:
            raise SystemExit("no seed satisfies the margin / tie conditions for " + tag)
        store(out, tag, f, duration, seed, rec, min_len)

    # three-stream merge: the second stream is shorter (truncation), the third longer (resampling), with weights
    for seed in range(1000, 1200):
        g = np.random.RandomState(seed)
        streams = [synth_logits(820, seed, "smooth")[:, None, :] + (g.randn(820, 4, 2) * 0.2).astype(np.float32),
                   (g.randn(800, 4, 2) * 0.5).astype(np.float32), (g.randn(1333, 3, 2) * 0.5).astype(np.float32)]
        weights = [1.0, 0.5, 0.75]
        merged = merge(streams, weights)
        rec = run_gen_prop(merged, 91.5)
        if conditions_ok(rec):
            break
    else:
        raise SystemExit("no seed satisfies the margin / tie conditions for the merge fixture")
    for i, st in enumerate(streams):
        out["merge_stream%d" % i] = st
    out["merge_weights"] = np.array(weights, np.float64)
    store(out, "merge", merged, 91.5, seed, rec, 0.0)
    np.savez_compressed(os.path.join(GOLD, "proposals.npz"), **out)
    print("wrote proposals.npz:", len(out), "arrays")


def main_nms():
    """tests/golden/proposals_nms.npz: the reference's temporal_nms_fallback on proposal_check.nms_cases(7) -- distinct
    scores with one NaN, +inf and -inf, IoU exactly at the threshold -- as kept indices, for machines without oracle/_ref
    (python -m oracle.gen_golden_proposals nms)"""
    sys.path.insert(0, REF)
    import ops.sequence_funcs as SF
    from oracle.proposal_check import nms_cases
    assert SF.nms is None, "the reference's optional GPU nms is importable; temporal_nms would not be the fallback"
    out = {}
    for c, (s, e, sc, thresh) in enumerate(nms_cases(7)):
        kept = SF.temporal_nms([(a, b, i, x) for i, (a, b, x) in enumerate(zip(s.tolist(), e.tolist(), sc))], thresh)
        out.update({"c%d_start" % c: s, "c%d_end" % c: e, "c%d_score" % c: sc, "c%d_thresh" % c: np.float64(thresh),
                    "c%d_kept" % c: np.array([k[2] for k in kept], np.int64)})
    out["n_cases"] = np.int64(len(out) // 5)
    np.savez_compressed(os.path.join(GOLD, "proposals_nms.npz"), **out)
    print("wrote proposals_nms.npz:", int(out["n_cases"]), "cases")


if __name__ == "__main__":
    main_nms() if sys.argv[1:] == ["nms"] else main()
