"""tests/golden/anet_detection.npz from the REAL ActivityNet toolkit (build container only:
python -m oracle.gen_golden_anet_detection).

anet_toolkit/Evaluation/eval_detection.py is imported as a module with importlib (np.float = float first: numpy 2 removed the
alias :231-232 use).  ANETdetection is never constructed with check_status=True and get_blocked_videos is never called (it
reaches the network): an instance is made with __new__, given the attributes __init__ sets with check_status=False and the
blocked list of the fixture, and its own _import_ground_truth / _import_prediction / evaluate run on JSON files written to a
temporary directory.  The toolkit's code is unedited.

Written, per fixture <name> (listed in `fixtures`):
  <name>_gt_text, <name>_pr_text   the ground-truth and results JSON texts
  <name>_blocked                   the blocked videos
  <name>_ap [n_thr, K], <name>_map [n_thr], <name>_average_map   the toolkit's self.ap, self.mAP and Average-mAP
at tIoU np.linspace(0.5, 0.95, 10) (`tiou_thresholds`), and for the "edges" fixture the toolkit's data frames
(frame_gt_* / frame_pr_* columns, frame_classes in activity_index order) for the loaders.

Fixtures:
  anet     a real-data slice: the first 300 validation videos of activity_net.v1-3.min.json; its sample_detection_prediction.json
           rows for them (each a ground-truth segment with score 1.0) with seeded scores and jittered segments, plus three
           seeded rows per video of other classes and segments
  edges    predictions for videos of another subset and for videos without annotations, ground-truth videos without
           predictions, a class without predictions, blocked videos on both sides
  ties     tied, -0 / +0 and NaN scores within and across videos, two ground truths at equal tIoU to a prediction, zero-length
           and reversed segments (a NaN tIoU)
  long     one (class, video) with 700 rows: more than one CTA of the AP sum handles
  k200     200 classes at ActivityNet-1.3 shape: 400 videos, 1..3 instances each, 0..60 rows per video
numpy's portable sort orders up to 16 elements by insertion sort, which is stable, so there the toolkit's order of tied
scores and tIoU is the rule of ops/detection_eval.py; above 16 it is open.  A fixture is kept only if no class with more than
16 rows holds two equal scores (NaN counted as one value), and no (video, class) with more than 16 instances gives a row two
equal tIoU at or above the lowest threshold; otherwise it is re-drawn from the next seed.  On a CPU with AVX2 or AVX-512,
numpy 2 dispatches float64 argsort to x86-simd-sort, which is not stable at any size; the generator therefore runs with that
dispatch disabled (NPY_DISABLE_CPU_FEATURES, set before numpy is imported; it re-executes itself to do so).

The oracle (oracle/anet_detection_oracle.py) is asserted equal to the toolkit on every fixture, to the bit."""
import importlib.util
import json
import os
import sys
import tempfile

SIMD_SORTS = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2"
if __name__ == "__main__" and os.environ.get("NPY_DISABLE_CPU_FEATURES") != SIMD_SORTS:
    os.execve(sys.executable, [sys.executable, "-m", "oracle.gen_golden_anet_detection"],
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

from oracle import anet_detection_oracle as O         # noqa: E402
from ops import detection_eval as E                   # noqa: E402  (the JSON loaders only: host code)

THR = np.linspace(0.5, 0.95, 10)


def load_toolkit():
    np.float = float                                   # eval_detection.py:231-232
    sys.path.insert(0, EVAL)
    spec = importlib.util.spec_from_file_location("ref_eval_detection", os.path.join(EVAL, "eval_detection.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_toolkit(mod, gt_json, pr_json, blocked=(), subset="validation"):
    """-> the toolkit object after evaluate()"""
    with tempfile.TemporaryDirectory() as d:
        gf, pf = os.path.join(d, "gt.json"), os.path.join(d, "pr.json")
        with open(gf, "w") as f:
            json.dump(gt_json, f)
        with open(pf, "w") as f:
            json.dump(pr_json, f)
        a = mod.ANETdetection.__new__(mod.ANETdetection)
        a.subset, a.tiou_thresholds, a.verbose = subset, THR, False
        a.gt_fields, a.pred_fields = mod.ANETdetection.GROUND_TRUTH_FIELDS, mod.ANETdetection.PREDICTION_FIELDS
        a.ap = None
        a.check_status, a.blocked_videos = False, list(blocked)
        a.ground_truth, a.activity_index = a._import_ground_truth(gf)
        a.prediction = a._import_prediction(pf)
        a.evaluate()
    return a


def pack(gt_json, pr_json, blocked=()):
    gt = E.load_anet_detection_ground_truth(gt_json, "validation", blocked)
    pr = E.load_anet_detection_predictions(pr_json, gt, blocked)
    V = len(pr["video_ids"])
    off = np.concatenate([gt["offsets"], np.full(V + 1 - len(gt["offsets"]), gt["offsets"][-1])])
    return dict(video=pr["video"], label=pr["label"], seg=pr["seg"], score=pr["score"], gt_offsets=off, gt_cls=gt["cls"],
                gt_seg=gt["seg"], K=len(gt["activity_index"]))


def ties_defined(pk):
    """no class of more than 16 rows holds two equal scores (NaN as one value); no (video, class) of more than 16 instances
    gives a row two equal tIoU (NaN as one value) at or above the lowest threshold"""
    s = pk["score"]
    for c in np.unique(pk["label"]):
        x = s[pk["label"] == c]
        if len(x) > 16 and len(np.unique(x[~np.isnan(x)])) + int(np.isnan(x).sum()) != len(x):
            return False
    off, gc, gs = pk["gt_offsets"], pk["gt_cls"], pk["gt_seg"]
    for r in range(len(s)):
        v, c = pk["video"][r], pk["label"][r]
        q = gs[off[v]:off[v + 1]][gc[off[v]:off[v + 1]] == c]
        if len(q) <= 16:
            continue
        p = pk["seg"][r]
        inter = (np.minimum(p[1], q[:, 1]) - np.maximum(p[0], q[:, 0])).clip(0)
        with np.errstate(invalid="ignore", divide="ignore"):
            t = inter / ((q[:, 1] - q[:, 0]) + (p[1] - p[0]) - inter)
        t = t[(t >= THR.min()) | np.isnan(t)]
        if len(np.unique(t[~np.isnan(t)])) + int(np.isnan(t).sum()) != len(t):
            return False
    return True


def store(out, name, mod, gt_json, pr_json, blocked=()):
    """evaluate with the toolkit, check the oracle to the bit; False when a tie the toolkit leaves open decides something"""
    try:
        pk = pack(gt_json, pr_json, blocked)
    except ValueError:                                 # a predicted label the ground truth lacks: the toolkit's KeyError
        return False
    if not ties_defined(pk):
        return False
    a = run_toolkit(mod, gt_json, pr_json, blocked)
    o = O.detection(pk["video"], pk["label"], pk["seg"], pk["score"], pk["gt_offsets"], pk["gt_cls"], pk["gt_seg"], pk["K"], THR)
    assert a.ap.shape == o["ap"].T.shape and a.ap.tobytes() == np.ascontiguousarray(o["ap"].T).tobytes(), (name, np.abs(a.ap - o["ap"].T).max())
    pre = name + "_"
    out[pre + "gt_text"], out[pre + "pr_text"] = np.array(json.dumps(gt_json)), np.array(json.dumps(pr_json))
    out[pre + "blocked"] = np.array(list(blocked), dtype=str)
    out.update({pre + "ap": a.ap, pre + "map": a.mAP, pre + "average_map": np.float64(a.mAP.mean())})
    print("%-6s videos %4d  rows %6d  instances %5d  classes %3d  average mAP %.6f"
          % (name, len(pk["gt_offsets"]) - 1, len(pk["score"]), len(pk["gt_cls"]), pk["K"], a.mAP.mean()))
    return a


# ---- the real-data slice --------------------------------------------------------------------------------------------------
def real_slice(gt_all, pr_all, vids, g):
    """the sample's rows of vids with seeded scores and segments jittered by up to 10 % of their length, plus three seeded
    rows per video of the slice's classes at random segments"""
    db = {k: gt_all["database"][k] for k in vids}
    labels = list(dict.fromkeys(a["label"] for v in vids for a in db[v]["annotations"]))
    res = {}
    for v in vids:
        dur = db[v]["duration"]
        rows = []
        for r in pr_all["results"].get(v, []):
            t0, t1 = r["segment"]
            j = (t1 - t0) * 0.1 * (g.rand(2) * 2 - 1)
            rows.append({"label": r["label"], "score": float(g.rand()), "segment": [float(t0 + j[0]), float(t1 + j[1])]})
        for _ in range(3):
            a, b = np.sort(g.rand(2) * dur)
            rows.append({"label": labels[g.randint(len(labels))], "score": float(g.rand()), "segment": [float(a), float(b)]})
        res[v] = [rows[i] for i in g.permutation(len(rows))]
    return dict(gt_all, database=db), dict(pr_all, results=res)


# ---- synthetic fixtures -------------------------------------------------------------------------------------------------------
def as_json(videos, extra_results=(), subsets=None):
    """videos: [(vid, [(label, t0, t1)] ground truth, [(label, score, t0, t1)] predictions or None (absent from the results))]"""
    db, res = {}, {}
    for vid, gt, pr in videos:
        db[vid] = {"subset": (subsets or {}).get(vid, "validation"), "duration": 200.0,
                   "annotations": [{"segment": [t0, t1], "label": c} for c, t0, t1 in gt]}
        if pr is not None:
            res[vid] = [{"label": c, "score": s, "segment": [t0, t1]} for c, s, t0, t1 in pr]
    for vid, pr in extra_results:
        res[vid] = [{"label": c, "score": s, "segment": [t0, t1]} for c, s, t0, t1 in pr]
    return ({"version": "VERSION 1.3", "taxonomy": [], "database": db},
            {"version": "VERSION 1.3", "results": res, "external_data": {}})


def cls(i):
    return "class_%03d" % i


def seg_near(g, t0, t1, spread=0.2):
    j = (t1 - t0) * spread * (g.rand(2) * 2 - 1)
    return float(t0 + j[0]), float(t1 + j[1])


def rand_seg(g, dur=200.0):
    a, b = np.sort(g.rand(2) * dur)
    return float(a), float(b)


def fx_edges(g):
    vids, subsets = [], {}
    for v in range(16):
        gt = []
        for k in range(1 + v % 3):
            t0, t1 = rand_seg(g)
            gt.append((cls(v if k == 0 and v < 5 else int(g.randint(5))), t0, t1))   # class_005: ground truth only (below)
        pr = [(c, float(g.rand())) + seg_near(g, t0, t1) for c, t0, t1 in gt for _ in range(1 + g.randint(3))]
        pr += [(cls(int(g.randint(5))), float(g.rand())) + rand_seg(g) for _ in range(g.randint(4))]
        vids.append(("e_%02d" % v, gt, None if v == 4 else [] if v == 9 else pr))
    vids.append(("e_cls5", [(cls(5), 10.0, 30.0)], None))
    vids.append(("e_noann", [], [(cls(0), 0.5, 10.0, 30.0), (cls(1), 0.25, 1.0, 5.0)]))    # a subset video without annotations
    subsets["e_07"] = "training"                                                           # its predictions: false positives
    extra = [("nogt_%d" % k, [(cls(int(c)), float(g.rand())) + rand_seg(g) for c in g.randint(0, 5, 2 + k)]) for k in range(3)]
    return as_json(vids, extra, subsets), ("e_11", "nogt_1")


def fx_ties(g):
    choices = [float("nan"), 0.5, 0.5, -0.0, 0.0, 0.25, 1.0]
    vids = []
    for v in range(10):
        c = cls(v % 6)
        # two instances at equal tIoU to the prediction (2, 18): (0, 12) and (8, 20) both give 10 / 18; a zero-length instance
        gt = [(c, 0.0, 12.0), (c, 8.0, 20.0), (c, 40.0, 40.0), (cls(int(g.randint(6))), 50.0, 70.0)]
        pr = [(c, choices[g.randint(len(choices))], 2.0, 18.0), (c, choices[g.randint(len(choices))], 2.5, 12.5),
              (c, choices[g.randint(len(choices))], 40.0, 40.0),                            # zero length on zero length: NaN tIoU
              (c, choices[g.randint(len(choices))], 12.0, 3.0),                             # reversed
              (cls(int(g.randint(6))), choices[g.randint(len(choices))], 52.0, 68.0)]
        vids.append(("t_%d" % v, gt, [pr[i] for i in g.permutation(len(pr))[:2 + v % 4]]))
    return as_json(vids), ()


def fx_long(g):
    gt = [(cls(0), 20.0 * k, 20.0 * k + 12.0) for k in range(9)] + [(cls(1), 5.0, 50.0)]
    pr = [(cls(0), float(g.rand())) + seg_near(g, *gt[g.randint(9)][1:], spread=0.5) for _ in range(700)]
    pr += [(cls(1), float(g.rand())) + seg_near(g, 5.0, 50.0) for _ in range(30)]
    other = [("l_%d" % v, [(cls(v % 2), 30.0, 60.0)], [(cls(v % 2), float(g.rand())) + seg_near(g, 30.0, 60.0)]) for v in range(4)]
    return as_json([("l_big", gt, pr)] + other), ()


def fx_k200(g):
    vids, first = [], g.permutation(200)
    for v in range(400):
        gt = []
        for k in range(int(g.choice([1, 2, 3], p=[0.6, 0.3, 0.1]))):
            t0, t1 = rand_seg(g)
            gt.append((cls(int(first[v]) if k == 0 and v < 200 else int(g.randint(200))), t0, t1))   # every class annotated
        n = int(g.choice([0, g.randint(1, 10), g.randint(10, 61)], p=[0.05, 0.45, 0.5]))
        pr = []
        for _ in range(n):
            if g.rand() < 0.4:
                c, t0, t1 = gt[g.randint(len(gt))]
                pr.append((c, float(g.rand())) + seg_near(g, t0, t1))
            else:
                pr.append((cls(int(g.randint(200))), float(g.rand())) + rand_seg(g))
        vids.append(("k_%03d" % v, gt, None if n == 0 and v % 2 else pr))
    return as_json(vids), ()


FIXTURES = (("edges", fx_edges), ("ties", fx_ties), ("long", fx_long), ("k200", fx_k200))


def main():
    assert np.argsort(np.array([0.5, 0.5, 0.25, -0.0, 0.5, 0.5])).tolist() == [3, 2, 0, 1, 4, 5], "numpy's small sorts are not stable"
    tk = load_toolkit()
    out = {"tiou_thresholds": THR}
    with open(os.path.join(EVAL, "data", "activity_net.v1-3.min.json")) as f:
        gt_all = json.load(f)
    with open(os.path.join(EVAL, "data", "sample_detection_prediction.json")) as f:
        pr_all = json.load(f)
    val = [k for k, v in gt_all["database"].items() if v["subset"] == "validation"]
    for seed in range(7, 100):
        if store(out, "anet", tk, *real_slice(gt_all, pr_all, val[:300], np.random.RandomState(seed))):
            break
    for i, (name, build) in enumerate(FIXTURES):
        for seed in range(3000 + 100 * i, 3100 + 100 * i):
            (gj, pj), blk = build(np.random.RandomState(seed))
            a = store(out, name, tk, gj, pj, blk)
            if a:
                break
        assert a, name
        if name == "edges":
            out["frame_gt_video"], out["frame_gt_label"] = a.ground_truth["video-id"].to_numpy(str), a.ground_truth["label"].to_numpy(np.int64)
            out["frame_gt_seg"] = a.ground_truth[["t-start", "t-end"]].to_numpy(np.float64)
            out["frame_pr_video"], out["frame_pr_label"] = a.prediction["video-id"].to_numpy(str), a.prediction["label"].to_numpy(np.int64)
            out["frame_pr_seg"] = a.prediction[["t-start", "t-end"]].to_numpy(np.float64)
            out["frame_pr_score"] = a.prediction["score"].to_numpy(np.float64)
            out["frame_classes"] = np.array(list(a.activity_index))
    out["fixtures"] = np.array(["anet"] + [f[0] for f in FIXTURES])
    np.savez_compressed(os.path.join(GOLD, "anet_detection.npz"), **out)
    print("wrote anet_detection.npz: %d arrays, %d bytes" % (len(out), os.path.getsize(os.path.join(GOLD, "anet_detection.npz"))))


if __name__ == "__main__":
    main()
