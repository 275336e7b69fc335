"""tests/golden/anet_classification.npz from the REAL ActivityNet toolkit (build container only:
python -m oracle.gen_golden_anet_classification).

anet_toolkit/Evaluation/eval_classification.py and eval_kinetics.py are imported as modules with importlib (np.float = float
first: numpy 2 removed the alias :206-207 use).  ANETclassification is never constructed with check_status=True and
get_blocked_videos is never called (it reaches the network): an instance is made with __new__, given the attributes __init__
sets with check_status=False and the blocked list of the fixture, and its own _import_ground_truth / _import_prediction /
evaluate run on JSON files written to a temporary directory.  The toolkit's code is unedited.

Written:
  anet_*      a real-data slice: the first 600 validation videos of the toolkit's activity_net.v1-3.min.json, the rows of its
              sample_classification_prediction.json for them (every score there is 1.0) re-scored from a seed, and four seeded
              rows of other classes per video; evaluated by eval_classification at top_k 3 and by eval_kinetics at 1 and 5
  json_*      a ground-truth / prediction JSON text pair with blocked videos on both sides (json_gt_text, json_pr_text,
              json_blocked), evaluated as a fixture
  frame_*     the toolkit's data frames of that pair and its activity_index order, for the loaders
  <fixture>_* synthetic fixtures (FIXTURES below)
Each fixture holds the packed inputs (video, label, score, gt_video, gt_label, V, K; stored once per data set, <fixture>_inputs
names the fixture that holds them), top_k, and the toolkit's ap (in activity_index order), hit_at_k and avg_hit_at_k.  numpy's
portable sort orders up to 16 elements by insertion sort, which is stable, so there the toolkit's order of tied scores is the
rule of ops/classification_eval.py; above 16 it is open, so a class's or a video's rows never hold two equal scores (NaN
among them) when there are more than 16 of them.  On a CPU with AVX2 or AVX-512, numpy 2 dispatches argsort of float64 to
x86-simd-sort, which is not stable at any size; the generator therefore runs with that dispatch disabled
(NPY_DISABLE_CPU_FEATURES, set before numpy is imported; it re-executes itself to do so).

The oracle (oracle/anet_classification_oracle.py) is asserted bitwise equal to the toolkit on every fixture, and on the whole
4926-video validation set re-scored the same way: a check of the oracle at scale, not a test."""
import importlib.util
import json
import os
import sys
import tempfile

SIMD_SORTS = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2"
if __name__ == "__main__" and os.environ.get("NPY_DISABLE_CPU_FEATURES") != SIMD_SORTS:
    os.execve(sys.executable, [sys.executable, "-m", "oracle.gen_golden_anet_classification"],
              dict(os.environ, NPY_DISABLE_CPU_FEATURES=SIMD_SORTS))

import numpy as np                                    # noqa: E402

REF = "/root/reference"
EVAL = os.path.join(REF, "anet_toolkit", "Evaluation")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import anet_classification_oracle as O    # noqa: E402
from ops import classification_eval as E              # noqa: E402  (the JSON loaders only: host code)


def load_toolkit():
    np.float = float                                   # eval_classification.py:206-207
    sys.path.insert(0, EVAL)
    mods = {}
    for name in ("eval_classification", "eval_kinetics"):
        spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(EVAL, name + ".py"))
        mods[name] = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mods[name])
    return mods


def run_toolkit(mod, gt_json, pr_json, top_k, blocked=(), subset="validation"):
    """-> the toolkit object after evaluate()"""
    with tempfile.TemporaryDirectory() as d:
        gf, pf = os.path.join(d, "gt.json"), os.path.join(d, "pr.json")
        with open(gf, "w") as f:
            json.dump(gt_json, f)
        with open(pf, "w") as f:
            json.dump(pr_json, f)
        a = mod.ANETclassification.__new__(mod.ANETclassification)
        a.subset, a.verbose, a.top_k = subset, False, top_k
        a.gt_fields, a.pred_fields = mod.ANETclassification.GROUND_TRUTH_FIELDS, mod.ANETclassification.PREDICTION_FIELDS
        a.ap = a.hit_at_k = None
        a.check_status, a.blocked_videos = False, list(blocked)
        a.ground_truth, a.activity_index = a._import_ground_truth(gf)
        a.prediction = a._import_prediction(pf)
        a.evaluate()
    return a


def pack(gt_json, pr_json, blocked=(), subset="validation"):
    gt = E.load_anet_classification_ground_truth(gt_json, subset, blocked)
    pr = E.load_anet_classification_predictions(pr_json, gt, blocked)
    return dict(video=pr["video"], label=pr["label"], score=pr["score"], gt_video=gt["video"], gt_label=gt["label"],
                V=np.int64(len(pr["video_ids"])), K=np.int64(len(gt["activity_index"])))


def ties_defined(pk):
    """every class's and every video's rows: at most 16 of them, or no two equal scores (NaN counted as one value)"""
    s = pk["score"]
    for key in (pk["label"], pk["video"]):
        for k in np.unique(key):
            x = s[key == k]
            if len(x) > 16 and len(np.unique(x[~np.isnan(x)])) + int(np.isnan(x).sum()) != len(x):
                return False
    return True


def check_and_store(out, name, mod, gt_json, pr_json, top_k, blocked=(), share=None):
    """share: the fixture whose packed inputs these are (stored once, under its name)"""
    a = run_toolkit(mod, gt_json, pr_json, top_k, blocked)
    pk = pack(gt_json, pr_json, blocked)
    assert ties_defined(pk), name
    o = O.classification(pk["video"], pk["label"], pk["score"], pk["gt_video"], pk["gt_label"], int(pk["V"]), int(pk["K"]), top_k)
    assert a.ap.dtype == o["ap"].dtype and a.ap.tobytes() == o["ap"].tobytes(), (name, "ap")
    assert (a.hit_at_k, a.avg_hit_at_k) == (o["hit_at_k"], o["avg_hit_at_k"]), (name, a.hit_at_k, o["hit_at_k"], a.avg_hit_at_k, o["avg_hit_at_k"])
    pre = name + "_"
    for k, x in pk.items():
        if share:
            assert out[share + "_" + k].tobytes() == np.asarray(x).tobytes()
        else:
            out[pre + k] = x
    out[pre + "inputs"] = np.array(share or name)
    out[pre + "top_k"] = np.int64(top_k)
    out.update({pre + "ap": a.ap, pre + "map": np.float64(a.ap.mean()), pre + "hit_at_k": np.float64(a.hit_at_k),
                pre + "avg_hit_at_k": np.float64(a.avg_hit_at_k)})
    print("%-14s videos %4d  rows %6d  pairs %5d  classes %3d  top_k %d  mAP %.6f  hit@k %.6f  avg %.6f"
          % (name, pk["V"], len(pk["score"]), len(pk["gt_video"]), pk["K"], top_k, a.ap.mean(), a.hit_at_k, a.avg_hit_at_k))


# ---- the real-data slice --------------------------------------------------------------------------------------------------
def rescored(gt_all, pr_all, vids, seed, blocked=()):
    """the sample's rows of vids with seeded scores, plus four seeded rows per video of other classes of the slice's
    validation videos that are not blocked"""
    g = np.random.RandomState(seed)
    labels = list(dict.fromkeys(a["label"] for v in vids if gt_all["database"][v]["subset"] == "validation" and v not in blocked
                                for a in gt_all["database"][v]["annotations"]))
    res = {}
    for v in vids:
        rows = [dict(r, score=float(g.rand())) for r in pr_all["results"].get(v, [])]
        have = {r["label"] for r in rows}
        for c in g.permutation(len(labels)):
            if len(rows) >= len(pr_all["results"].get(v, [])) + 4:
                break
            if labels[c] not in have:
                rows.append({"label": labels[c], "score": float(g.rand())})
        res[v] = [rows[i] for i in g.permutation(len(rows))]
    return dict(gt_all, database={k: gt_all["database"][k] for k in vids}), dict(pr_all, results=res)


# ---- synthetic fixtures -------------------------------------------------------------------------------------------------------
def as_json(videos, extra_results=(), subsets=None):
    """videos: [(vid, gt labels [str], predictions [(label, score)] or None (absent from the results))]"""
    db, res = {}, {}
    for vid, gt, pr in videos:
        db[vid] = {"subset": (subsets or {}).get(vid, "validation"), "duration": 100.0,
                   "annotations": [{"segment": [1.0 * k, 1.0 * k + 5.0], "label": c} for k, c in enumerate(gt)]}
        if pr is not None:
            res[vid] = [{"label": c, "score": s} for c, s in pr]
    for vid, pr in extra_results:
        res[vid] = [{"label": c, "score": s} for c, s in pr]
    return ({"version": "VERSION 1.3", "taxonomy": [], "database": db},
            {"version": "VERSION 1.3", "results": res, "external_data": {}})


def cls(i):
    return "class_%02d" % i


def fx_edges(g):
    """multi-label videos, repeated annotations, repeated (video, label) rows, videos without predictions (absent and empty),
    predictions for videos without ground truth and for a video of another subset, a class with no prediction, NaN scores,
    blocked videos on both sides"""
    vids, subsets = [], {}
    for v in range(14):
        gt = [cls(int(c)) for c in g.choice(6, 1 + v % 3, replace=False)]
        if v % 4 == 1:
            gt.append(gt[0])                                   # the same label annotated twice: one ground-truth row
        pr = [(cls(int(c)), float(g.rand())) for c in g.randint(0, 5, 1 + v % 6)]   # class_05: ground truth only
        if v % 5 == 2:
            pr.append((pr[0][0], float(g.rand())))              # a repeated (video, label) row
        if v % 6 == 3:
            pr[0] = (pr[0][0], float("nan"))
        vids.append(("e_%02d" % v, gt, None if v == 4 else [] if v == 9 else pr))
    subsets["e_07"] = "training"
    extra = [("nogt_%d" % k, [(cls(int(c)), float(g.rand())) for c in g.randint(0, 5, 2 + k)]) for k in range(3)]
    return as_json(vids, extra, subsets), ("e_11", "nogt_1")


def fx_ties(g):
    """tied, -0 / +0 and NaN scores; no class or video holds more than 16 rows"""
    choices = [float("nan"), 0.5, 0.5, -0.0, 0.0, 0.25, 1.0]
    vids = []
    for v in range(8):
        gt = [cls(int(c)) for c in g.choice(4, 1 + v % 2, replace=False)]
        pr = [(cls(int(c)), choices[g.randint(len(choices))]) for c in g.randint(0, 4, 2 + v % 5)]
        vids.append(("t_%d" % v, gt, pr))
    return as_json(vids), ()


def fx_ragged(g):
    """300 videos, 24 classes, 1..3 labels each, 0..30 rows per video with continuous scores (some videos unscored)"""
    vids = []
    for v in range(300):
        gt = [cls(int(c)) for c in g.choice(24, int(g.choice([1, 2, 3], p=[0.6, 0.3, 0.1])), replace=False)]
        n = int(g.choice([0, g.randint(1, 8), g.randint(8, 31)], p=[0.05, 0.55, 0.4]))
        pr = [(cls(int(c)), float(g.rand())) for c in g.randint(0, 24, n)]
        vids.append(("r_%03d" % v, gt, None if n == 0 and v % 2 else pr))
    return as_json(vids), ()


# name, builder, evaluator, top_k
FIXTURES = (
    ("edges", fx_edges, "eval_classification", 3),
    ("edges_k1", fx_edges, "eval_kinetics", 1),
    ("edges_k5", fx_edges, "eval_kinetics", 5),
    ("ties", fx_ties, "eval_classification", 3),
    ("ties_k1", fx_ties, "eval_kinetics", 1),
    ("ragged", fx_ragged, "eval_classification", 3),
    ("ragged_k1", fx_ragged, "eval_kinetics", 1),
    ("ragged_k5", fx_ragged, "eval_kinetics", 5),
)


def main():
    assert np.argsort(np.array([0.5, 0.5, 0.25, -0.0, 0.5, 0.5])).tolist() == [3, 2, 0, 1, 4, 5], "numpy's small sorts are not stable"
    tk = load_toolkit()
    out = {}
    with open(os.path.join(EVAL, "data", "activity_net.v1-3.min.json")) as f:
        gt_all = json.load(f)
    with open(os.path.join(EVAL, "data", "sample_classification_prediction.json")) as f:
        pr_all = json.load(f)
    val = [k for k, v in gt_all["database"].items() if v["subset"] == "validation"]
    gt_s, pr_s = rescored(gt_all, pr_all, val[:600], 7)
    for name, ev, k in (("anet", "eval_classification", 3), ("anet_k1", "eval_kinetics", 1), ("anet_k5", "eval_kinetics", 5)):
        check_and_store(out, name, tk[ev], gt_s, pr_s, k, share=None if name == "anet" else "anet")
    # the JSON pair for the loaders: the first 6 videos of the database (other subsets among them) and 10 validation videos;
    # two prediction-only videos; one blocked video on each side
    first = list(dict.fromkeys(list(gt_all["database"])[:6] + val[:10]))
    extra = val[10:12]
    vj = [k for k in first if gt_all["database"][k]["subset"] == "validation"]
    blocked = (vj[1], extra[1])
    gt_j, pr_j = rescored(gt_all, pr_all, first, 8, blocked)
    for v in extra:
        pr_j["results"][v] = [{"label": gt_all["database"][first[-1]]["annotations"][0]["label"], "score": 0.125}]
    out["json_gt_text"], out["json_pr_text"] = np.array(json.dumps(gt_j)), np.array(json.dumps(pr_j))
    out["json_blocked"] = np.array(blocked)
    a = run_toolkit(tk["eval_classification"], gt_j, pr_j, 3, blocked)
    out["frame_gt_video"], out["frame_gt_label"] = a.ground_truth["video-id"].to_numpy(str), a.ground_truth["label"].to_numpy(np.int64)
    out["frame_pr_video"], out["frame_pr_label"] = a.prediction["video-id"].to_numpy(str), a.prediction["label"].to_numpy(np.int64)
    out["frame_pr_score"] = a.prediction["score"].to_numpy(np.float64)
    out["frame_classes"] = np.array(list(a.activity_index))
    check_and_store(out, "json", tk["eval_classification"], gt_j, pr_j, 3, blocked)
    # synthetic fixtures
    first_of = {}
    for name, build, ev, k in FIXTURES:
        (gj, pj), blk = build(np.random.RandomState(2000 + [f[1] for f in FIXTURES].index(build)))
        check_and_store(out, name, tk[ev], gj, pj, k, blk, share=first_of.get(build))
        first_of.setdefault(build, name)
    out["fixtures"] = np.array(["anet", "anet_k1", "anet_k5", "json"] + [f[0] for f in FIXTURES])
    np.savez_compressed(os.path.join(GOLD, "anet_classification.npz"), **out)
    print("wrote anet_classification.npz: %d arrays, %d bytes" % (len(out), os.path.getsize(os.path.join(GOLD, "anet_classification.npz"))))
    # the oracle at scale: the whole validation set, re-scored the same way
    import time
    gt_f, pr_f = rescored(gt_all, pr_all, val, 7)
    t0 = time.perf_counter()
    a = run_toolkit(tk["eval_classification"], gt_f, pr_f, 3)
    t1 = time.perf_counter()
    pk = pack(gt_f, pr_f)
    o = O.classification(pk["video"], pk["label"], pk["score"], pk["gt_video"], pk["gt_label"], int(pk["V"]), int(pk["K"]), 3)
    t2 = time.perf_counter()
    assert a.ap.tobytes() == o["ap"].tobytes() and (a.hit_at_k, a.avg_hit_at_k) == (o["hit_at_k"], o["avg_hit_at_k"]), "full set"
    print("full validation set: %d videos, %d rows, mAP %.6f, hit@3 %.6f: oracle == toolkit bitwise (toolkit %.1f s, oracle %.2f s)"
          % (pk["V"], len(pk["score"]), a.ap.mean(), a.hit_at_k, t1 - t0, t2 - t1))


if __name__ == "__main__":
    main()
