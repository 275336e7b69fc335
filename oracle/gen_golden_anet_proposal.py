"""tests/golden/anet_proposal.npz from the REAL ActivityNet toolkit (build container only: python -m oracle.gen_golden_anet_proposal).

anet_toolkit/Evaluation/eval_proposal.py is imported as a module with importlib (np.int = int first: numpy 2 removed the
alias :258 uses).  ANETproposal is never constructed with check_status=True and get_blocked_videos is never called (it
reaches the network): an instance is made with __new__, given the attributes __init__ sets with check_status=False and the
blocked list of the fixture, and its own _import_ground_truth / _import_proposal / evaluate run on JSON files written to a
temporary directory.  wrapper_segment_iou is wrapped from outside to record each evaluated video's kept proposals (nr_v);
the toolkit's code is unedited.

Written:
  anet_*      a real-data slice: the first 300 validation videos with annotations of the toolkit's activity_net.v1-3.min.json
              and their 100 proposals each from uniform_random_proposals.json, evaluated on their own at AN = 100, 10 and the
              default budget
  json_*      a 12-video (4 + 8 validation) ground-truth / proposal JSON text pair with one blocked video on each side, and the toolkit's data
              frames of it, for the loaders
  <fixture>_* synthetic ragged fixtures (FIXTURES below)
Each fixture holds the packed inputs (gt_seg, gt_offsets, boxes, scores, counts; stored once per data set, <fixture>_inputs
names the fixture that holds them), thresholds, max_avg (0 for the default) and the toolkit's recall, avg_recall, proposals_per_video, nr and auc / auc_percent.  Videos with more than 16 proposals never
hold two equal scores (numpy leaves the order of ties open there); smaller ones may.  numpy's portable sort orders up to 16
elements by insertion sort, which is stable, so there the toolkit's order is the rule of ops/proposal_eval.py.  On a CPU with
AVX2 or AVX-512, numpy 2 dispatches argsort of float64 to x86-simd-sort, which is not stable at any size (6 elements are
enough): the toolkit's order of tied scores, and so its result, depends on the machine.  The generator therefore runs with
that dispatch disabled (NPY_DISABLE_CPU_FEATURES, set before numpy is imported; it re-executes itself to do so).

The oracle (oracle/anet_proposal_oracle.py) is asserted bitwise equal to the toolkit on every fixture, and on the toolkit's
whole 4926-video sample at AN = 100: a check of the oracle at scale, not a test."""
import importlib.util
import json
import os
import sys
import tempfile

SIMD_SORTS = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2"
if __name__ == "__main__" and os.environ.get("NPY_DISABLE_CPU_FEATURES") != SIMD_SORTS:
    os.execve(sys.executable, [sys.executable, "-m", "oracle.gen_golden_anet_proposal"], dict(os.environ, NPY_DISABLE_CPU_FEATURES=SIMD_SORTS))

import numpy as np                                    # noqa: E402

REF = "/root/reference"
EVAL = os.path.join(REF, "anet_toolkit", "Evaluation")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import anet_proposal_oracle as O          # noqa: E402
from ops import proposal_eval as E                    # noqa: E402  (the JSON loaders only: host code)

DEFAULT_THR = np.linspace(0.5, 0.95, 10)


def load_toolkit():
    np.int = int                                       # eval_proposal.py:258
    sys.path.insert(0, EVAL)
    spec = importlib.util.spec_from_file_location("ref_eval_proposal", os.path.join(EVAL, "eval_proposal.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    original = mod.wrapper_segment_iou
    kept = []

    def recording(target_segments, candidate_segments):
        kept.append(target_segments.shape[0])
        return original(target_segments, candidate_segments)
    mod.wrapper_segment_iou = recording
    return mod, kept


def run_toolkit(tk, gt_json, pr_json, max_avg, thresholds, blocked=(), subset="validation"):
    """-> (toolkit object after evaluate(), kept proposals per evaluated video with proposals, auc, auc_percent)"""
    mod, kept = tk
    with tempfile.TemporaryDirectory() as d:
        gf, pf = os.path.join(d, "gt.json"), os.path.join(d, "pr.json")
        with open(gf, "w") as f:
            json.dump(gt_json, f)
        with open(pf, "w") as f:
            json.dump(pr_json, f)
        a = mod.ANETproposal.__new__(mod.ANETproposal)
        a.subset, a.tiou_thresholds, a.max_avg_nr_proposals, a.verbose = subset, np.asarray(thresholds, np.float64), max_avg, False
        a.gt_fields, a.pred_fields = mod.ANETproposal.GROUND_TRUTH_FIELDS, mod.ANETproposal.PROPOSAL_FIELDS
        a.recall = a.avg_recall = a.proposals_per_video = None
        a.check_status, a.blocked_videos = False, list(blocked)
        a.ground_truth, a.activity_index = a._import_ground_truth(gf)
        a.proposal = a._import_proposal(pf)
        del kept[:]
        a.evaluate()
    auc = np.trapezoid(a.avg_recall, a.proposals_per_video)      # :148, np.trapz under its numpy 2 name
    return a, list(kept), float(auc), 100. * float(auc) / a.proposals_per_video[-1]


def pack(gt_json, pr_json, blocked=(), subset="validation"):
    gt = E.load_anet_ground_truth(gt_json, subset, blocked)
    pr = E.load_anet_proposals(pr_json, gt["video_ids"], blocked)
    off = gt["gt_offsets"] + [gt["gt_offsets"][-1]] * (len(pr["video_ids"]) - len(gt["video_ids"]))
    return dict(gt_seg=gt["segments"], gt_offsets=np.array(off, np.int64), boxes=pr["boxes"], scores=pr["scores"],
                counts=np.array(pr["counts"], np.int64))


def check_and_store(out, name, tk, gt_json, pr_json, max_avg, thresholds, blocked=(), share=None):
    """share: the fixture whose packed inputs these are (stored once, under its name)"""
    a, kept, auc, pct = run_toolkit(tk, gt_json, pr_json, max_avg, thresholds, blocked)
    pk = pack(gt_json, pr_json, blocked)
    g_cnt = np.diff(pk["gt_offsets"])
    nr = np.zeros(len(pk["counts"]), np.int32)
    with_props = np.nonzero((g_cnt > 0) & (pk["counts"] > 0))[0]
    assert len(with_props) == len(kept), (name, len(with_props), len(kept))
    nr[with_props] = kept
    thr = np.asarray(thresholds, np.float64)
    o = O.average_recall(pk["boxes"], pk["scores"], pk["counts"], pk["gt_seg"], g_cnt, max_avg, thr)
    for k, ref in (("recall", a.recall), ("avg_recall", a.avg_recall), ("proposals_per_video", a.proposals_per_video), ("nr", nr)):
        assert np.asarray(ref).dtype == o[k].dtype and np.asarray(ref).tobytes() == o[k].tobytes(), (name, k)
    assert O.area(o["avg_recall"], o["proposals_per_video"]) == (auc, pct), name
    # any equal scores in a video of more than 16 proposals would leave the toolkit's order open
    for v, (f, n) in enumerate(zip(np.concatenate([[0], np.cumsum(pk["counts"])[:-1]]), pk["counts"])):
        if n > 16 and g_cnt[v] > 0:
            s = pk["scores"][f:f + n]
            assert len(np.unique(s[~np.isnan(s)])) + min(1, int(np.isnan(s).sum())) == n and np.isnan(s).sum() <= 1, (name, v)
    pre = name + "_"
    for k, x in pk.items():
        if share:
            assert out[share + "_" + k].tobytes() == x.tobytes()
        else:
            out[pre + k] = x
    out[pre + "inputs"] = np.array(share or name)
    out[pre + "thresholds"], out[pre + "max_avg"] = thr, np.float64(max_avg or 0.0)
    out.update({pre + "recall": a.recall, pre + "avg_recall": a.avg_recall, pre + "proposals_per_video": a.proposals_per_video,
                pre + "nr": nr, pre + "total_nr": np.int64(sum(kept)), pre + "auc": np.float64(auc), pre + "auc_percent": np.float64(pct)})
    print("%-16s videos %4d  rows %6d  instances %5d  total_nr %6d  AUC %.4f%%" % (name, len(pk["counts"]), len(pk["scores"]),
                                                                                len(pk["gt_seg"]), sum(kept), pct))


# ---- synthetic fixtures -------------------------------------------------------------------------------------------------------
def as_json(videos, extra_results=(), subsets=None):
    """videos: [(vid, gt [(t0, t1)], proposals [(t0, t1, score)] or None (absent from the results))]"""
    db, res = {}, {}
    for i, (vid, gt, pr) in enumerate(videos):
        db[vid] = {"subset": (subsets or {}).get(vid, "validation"), "duration": 100.0,
                   "annotations": [{"segment": [a, b], "label": "class_%d" % (k % 3)} for k, (a, b) in enumerate(gt)]}
        if pr is not None:
            res[vid] = [{"segment": [a, b], "score": s} for a, b, s in pr]
    for vid, pr in extra_results:
        res[vid] = [{"segment": [a, b], "score": s} for a, b, s in pr]
    return ({"version": "VERSION 1.3", "taxonomy": [], "database": db},
            {"version": "VERSION 1.3", "results": res, "external_data": {}})


def rand_gt(g, n, dur=100.0):
    c, d = g.uniform(0, dur, n), g.uniform(2, dur / 3, n)
    return [(float(max(0, a)), float(min(dur, b))) for a, b in zip(c - d / 2, c + d / 2)]


def rand_props(g, n, gt, dur=100.0):
    """random boxes, a third of them near a ground-truth instance; continuous scores"""
    out = []
    for i in range(n):
        if gt and i % 3 == 0:
            a, b = gt[g.randint(len(gt))]
            w = b - a
            a, b = a + g.uniform(-0.3, 0.3) * w, b + g.uniform(-0.3, 0.3) * w
        else:
            c, d = g.uniform(0, dur), g.uniform(1, dur / 2)
            a, b = c - d / 2, c + d / 2
        out.append((float(a), float(b), float(g.rand())))
    return out


def fx_noprop(g):
    vids = []
    for v in range(6):
        gt = rand_gt(g, 1 + v % 3)
        pr = None if v == 1 else [] if v == 4 else rand_props(g, 3 + v, gt)
        vids.append(("np_%d" % v, gt, pr))
    return as_json(vids)


def fx_small_counts(g):
    vids = []
    for v in range(8):
        gt = rand_gt(g, 1 + v % 2)
        vids.append(("sc_%d" % v, gt, rand_props(g, 1 + v % 3, gt)))
    return as_json(vids)


def default_ratio_below_one():
    """the smallest (P_all, V) whose default ratio float(P)/V * float(V) / P is below 1"""
    for V in range(2, 64):
        for P in range(V, 400):
            if float(P) / V * float(V) / P < 1:
                return P, V
    raise AssertionError("no pair")


def fx_ratio_lt1(g):
    P, V = default_ratio_below_one()
    counts = [1] * V
    for i in range(P - V):
        counts[i % V] += 1
    vids = []
    for v, n in enumerate(counts):
        gt = rand_gt(g, 1 + v % 2)
        vids.append(("rl_%d" % v, gt, rand_props(g, n, gt)))
    return as_json(vids)


def fx_outside(g):
    vids, subsets = [], {}
    for v in range(7):
        gt = rand_gt(g, 1 + v % 3)
        vids.append(("out_%d" % v, gt, rand_props(g, 4 + 2 * v, gt)))
    subsets["out_2"] = "training"                           # not in the subset: its proposals count in P_all only
    vids.append(("out_empty", [], rand_props(g, 5, [])))    # in the subset without annotations: the same
    extra = [("nogt_%d" % k, rand_props(g, 3 + 4 * k, [])) for k in range(3)]
    return as_json(vids, extra, subsets), ("out_4", "nogt_1")


def fx_degenerate(g):
    vids = []
    for v in range(6):
        gt = rand_gt(g, 3)
        pr = rand_props(g, 12, gt)
        pr[0] = (gt[0][0], gt[0][0], 0.9)                    # zero length
        pr[1] = (gt[1][1], gt[1][0], 0.8)                    # reversed
        pr[2] = (float("nan"), gt[0][1], 0.7)                # NaN start
        pr[3] = (gt[2][0], gt[2][0], 0.6)
        if v % 2:
            gt[2] = (gt[2][0], gt[2][0])                     # a zero-length instance: 0 / 0 against a zero-length proposal at it
            gt[1] = (gt[1][1], gt[1][0])                     # reversed instance
        if v == 3:
            gt[0] = (float("nan"), 50.0)
        vids.append(("dg_%d" % v, gt, pr))
    return as_json(vids)


def fx_on_threshold(g):
    # [0, b] against [0, a]: tIoU a / b exactly, landing on 0.5, 0.6, 0.75, 0.8, 0.9 and just below
    vids = []
    for v, (a, b) in enumerate(((1, 2), (3, 5), (3, 4), (4, 5), (9, 10), (7, 10), (2, 4), (1, 1))):
        gt = [(0.0, float(a)), (10.0, 10.0 + a)]
        pr = [(0.0, float(b), 0.5), (10.0, 10.0 + b, 0.4), (10.0 + b - a, 10.0 + b, 0.3)]
        vids.append(("th_%d" % v, gt, pr))
    return as_json(vids)


def fx_integer(g):
    vids = []
    for v in range(10):
        gt = [(int(a), int(a) + int(w)) for a, w in zip(g.randint(0, 80, 2), g.randint(1, 20, 2))]
        pr = [(int(a), int(a) + int(w), float(g.rand())) for a, w in zip(g.randint(0, 90, 12), g.randint(0, 25, 12))]
        vids.append(("int_%d" % v, gt, pr))
    return as_json(vids)


def fx_ties(g):
    vids = []
    for v in range(10):
        gt = rand_gt(g, 2)
        pr = rand_props(g, 6 + v, gt)
        choices = [float("nan"), 0.5, 0.5, -0.0, 0.0, 0.25, 1.0]
        pr = [(a, b, choices[g.randint(len(choices))]) for a, b, _ in pr]
        vids.append(("tie_%d" % v, gt, pr))
    return as_json(vids)


def fx_ragged(g):
    vids = []
    for v in range(200):
        n_gt = int(g.randint(1, 9))
        gt = rand_gt(g, n_gt, 200.0)
        n = int(g.choice([0, g.randint(1, 17), g.randint(17, 61)], p=[0.05, 0.45, 0.5]))
        vids.append(("rag_%03d" % v, gt, rand_props(g, n, gt, 200.0)))
    return as_json(vids)


# name, builder, max_avg (None: the default), thresholds
FIXTURES = (
    ("noprop_t0", fx_noprop, None, [0.0, 0.3, 0.5]),
    ("noprop", fx_noprop, None, DEFAULT_THR),
    ("nr_zero", fx_small_counts, 1.2, DEFAULT_THR),
    ("ratio_gt1", fx_small_counts, 7.0, [0.1, 0.5, 0.9]),
    ("ratio_lt1", fx_ratio_lt1, None, DEFAULT_THR),
    ("outside", fx_outside, None, DEFAULT_THR),
    ("outside_an3", fx_outside, 3, DEFAULT_THR),
    ("degenerate", fx_degenerate, 5, np.concatenate([[0.0], DEFAULT_THR])),
    ("on_threshold", fx_on_threshold, None, [0.5, 0.6, 0.75, 0.8, 0.9]),
    ("integer", fx_integer, 8, DEFAULT_THR),
    ("ties", fx_ties, 3, [0.05, 0.3, 0.5]),
    ("ragged", fx_ragged, 20, DEFAULT_THR),
)


def main():
    assert np.argsort(np.array([0.5, 0.5, 0.25, -0.0, 0.5, 0.5])).tolist() == [3, 2, 0, 1, 4, 5], "numpy's small sorts are not stable"
    tk = load_toolkit()
    out = {}
    with open(os.path.join(EVAL, "data", "activity_net.v1-3.min.json")) as f:
        gt_all = json.load(f)
    with open(os.path.join(EVAL, "data", "uniform_random_proposals.json")) as f:
        pr_all = json.load(f)
    # the real-data slice
    val = [k for k, v in gt_all["database"].items() if v["subset"] == "validation" and v["annotations"]][:300]
    gt_s = dict(gt_all, database={k: gt_all["database"][k] for k in val})
    pr_s = dict(pr_all, results={k: pr_all["results"][k] for k in val})
    for name, an in (("anet_an100", 100), ("anet_an10", 10), ("anet_default", None)):
        check_and_store(out, name, tk, gt_s, pr_s, an, DEFAULT_THR, share=None if an == 100 else "anet_an100")
    # the JSON pair for the loaders: the first 4 videos of the database (other subsets among them) and 8 validation videos, 20
    # proposals of each validation one, two videos outside the ground truth; one blocked video on each side
    first12 = list(dict.fromkeys(list(gt_all["database"])[:4] + val[:8]))
    gt_j = dict(gt_all, database={k: gt_all["database"][k] for k in first12})
    outside = [k for k in val if k not in first12][:2]
    pr_j = dict(pr_all, results={k: pr_all["results"][k][:20] for k in [k for k in first12 if k in pr_all["results"]] + outside})
    vj = [k for k in first12 if gt_all["database"][k]["subset"] == "validation" and gt_all["database"][k]["annotations"]]
    blocked = (vj[1], outside[1])
    out["json_gt_text"], out["json_pr_text"] = np.array(json.dumps(gt_j)), np.array(json.dumps(pr_j))
    out["json_blocked"] = np.array(blocked)
    a, _, _, _ = run_toolkit(tk, gt_j, pr_j, None, DEFAULT_THR, blocked)
    gdf, pdf = a.ground_truth, a.proposal
    out["json_gt_video"], out["json_gt_seg"] = gdf["video-id"].to_numpy(str), gdf[["t-start", "t-end"]].to_numpy(np.float64)
    out["json_gt_label"] = gdf["label"].to_numpy(np.int64)
    out["json_pr_video"], out["json_pr_seg"] = pdf["video-id"].to_numpy(str), pdf[["t-start", "t-end"]].to_numpy(np.float64)
    out["json_pr_score"] = pdf["score"].to_numpy(np.float64)
    check_and_store(out, "json", tk, gt_j, pr_j, None, DEFAULT_THR, blocked)
    # synthetic fixtures
    first_of = {}
    for i, (name, build, max_avg, thr) in enumerate(FIXTURES):
        made = build(np.random.RandomState(1000 + FIXTURES.index(next(f for f in FIXTURES if f[1] is build))))
        (gj, pj), blk = (made, ()) if len(made) == 2 and isinstance(made[0], dict) and "database" in made[0] else made
        check_and_store(out, name, tk, gj, pj, max_avg, thr, blk, share=first_of.get(build))
        first_of.setdefault(build, name)
    out["fixtures"] = np.array(["anet_an100", "anet_an10", "anet_default", "json"] + [f[0] for f in FIXTURES])
    np.savez_compressed(os.path.join(GOLD, "anet_proposal.npz"), **out)
    print("wrote anet_proposal.npz: %d arrays, %d bytes" % (len(out), os.path.getsize(os.path.join(GOLD, "anet_proposal.npz"))))
    # the oracle at scale: the toolkit's whole sample at AN = 100
    import time
    t0 = time.perf_counter()
    a, kept, auc, pct = run_toolkit(tk, gt_all, pr_all, 100, DEFAULT_THR)
    t1 = time.perf_counter()
    pk = pack(gt_all, pr_all)
    o = O.average_recall(pk["boxes"], pk["scores"], pk["counts"], pk["gt_seg"], np.diff(pk["gt_offsets"]), 100, DEFAULT_THR)
    t2 = time.perf_counter()
    for k, ref in (("recall", a.recall), ("avg_recall", a.avg_recall), ("proposals_per_video", a.proposals_per_video)):
        assert np.asarray(ref).tobytes() == o[k].tobytes(), ("full sample", k)
    assert O.area(o["avg_recall"], o["proposals_per_video"]) == (auc, pct)
    print("full sample: %d videos, %d proposals, AUC %.3f%%: oracle == toolkit bitwise (toolkit %.1f s, oracle %.1f s)"
          % (len(np.diff(pk["gt_offsets"])), len(pk["scores"]), pct, t1 - t0, t2 - t1))


if __name__ == "__main__":
    main()
