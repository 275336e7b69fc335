"""tests/golden/video_funcs.npz from the REAL reference functions (build container only: python -m oracle.gen_golden_video_funcs).

ops/video_funcs.py and ops/metrics.py of the reference checkout are imported unedited, as the submodules of a package made
with importlib (video_funcs imports softmax relatively).  They were written for Python 2; two of its details are supplied from
outside, into the modules' namespaces:
  xrange = range      used by sliding_window_aggregation_func, tpp_aggregation_func and video_mean_ap
  len                 returns an int whose / floors, so k = max(15, len(local_agg)/4) (video_funcs.py:49) is Python 2's
numpy's argsort of float32 / float64 is dispatched to x86-simd-sort on CPUs with AVX2 or AVX-512, which is not stable at any
size; the generator re-executes itself with that dispatch disabled, so numpy's insertion sort (stable up to 16 elements)
decides the tied fixtures, which keep K <= 16.

Written, per aggregation fixture <f>: agg_<f>_inputs (the fixture holding its agg_<src>_scores [sum T, crops, D] fp32 and
agg_<src>_offsets int64 [V+1], each score set stored once), agg_<f>_params
(JSON: mode and keyword arguments), agg_<f>_out [V, K] (the reference function per video, stacked).  Fusion: fuse_* ; softmax:
softmax_*; metrics: met_<f>_* (scores of the videos in score_dict, their label sets as (video, label) pairs, the ids missing
from score_dict, and the reference's top_k_acc / top_k_hit per video, top_k_accuracy, video_mean_ap); mca_<f>_* (scores,
labels, mean_class_accuracy)."""
import builtins
import importlib.util
import json
import os
import sys
import types
import warnings

SIMD_SORTS = "AVX512F AVX512CD AVX512_SKX AVX512_CLX AVX512_CNL AVX512_ICL AVX512_SPR AVX2"
if __name__ == "__main__" and os.environ.get("NPY_DISABLE_CPU_FEATURES") != SIMD_SORTS:
    os.execve(sys.executable, [sys.executable, "-m", "oracle.gen_golden_video_funcs"], dict(os.environ, NPY_DISABLE_CPU_FEATURES=SIMD_SORTS))

import numpy as np                                    # noqa: E402

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")

AGG_KW = {"default": ("normalization", "crop_agg"), "top_k": ("k", "normalization", "crop_agg"),
          "sliding_window": ("spans", "overlap", "norm", "fps"), "tpp": ("num_class",)}


class _Py2Int(int):
    def __truediv__(self, other):
        return _Py2Int(int(self) // other)


def load_reference(ops_dir=os.path.join(REF, "ops")):
    """-> (video_funcs, metrics) of the reference's ops directory (also the copy build() vendors under oracle/_ref/ops)"""
    pkg = types.ModuleType("ref_ops")
    pkg.__path__ = [ops_dir]
    sys.modules["ref_ops"] = pkg
    mods = {}
    for name in ("metrics", "video_funcs"):
        spec = importlib.util.spec_from_file_location("ref_ops." + name, os.path.join(ops_dir, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["ref_ops." + name] = m
        spec.loader.exec_module(m)
        m.xrange = range
        mods[name] = m
    mods["video_funcs"].len = lambda x: _Py2Int(builtins.len(x))
    return mods["video_funcs"], mods["metrics"]


def ragged(rng, Ts, crops, D, scale=3.0):
    off = np.r_[0, np.cumsum(Ts)].astype(np.int64)
    return (rng.standard_normal((int(off[-1]), crops, D)) * scale).astype(np.float32), off


def run_agg(vf, scores, off, mode, kw):
    fn = {"default": vf.default_aggregation_func, "top_k": vf.top_k_aggregation_func,
          "sliding_window": vf.sliding_window_aggregation_func, "tpp": vf.tpp_aggregation_func}[mode]
    call = dict(kw)
    if "crop_agg" in call:
        call["crop_agg"] = {"mean": np.mean, "max": np.max}[call["crop_agg"]]
    return np.stack([fn(scores[off[v]:off[v + 1]], **call) for v in range(len(off) - 1)])


class Inst:
    def __init__(self, c):
        self.num_label = c


class Video:
    def __init__(self, vid, labels):
        self.id, self.instances = vid, [Inst(c) for c in labels]


def main():
    vf, mt = load_reference()
    rng = np.random.default_rng(20261017)
    out = {}
    aggs, seen = [], {}

    def agg(name, scores, off, mode, **kw):
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            r = run_agg(vf, scores, off, mode, kw)
        src = seen.setdefault(id(scores), name)            # each score set is stored once, under the first fixture using it
        out["agg_%s_inputs" % name] = src
        if src == name:
            out["agg_%s_scores" % name], out["agg_%s_offsets" % name] = scores, off
        out["agg_%s_params" % name] = json.dumps(dict(mode=mode, **kw))
        out["agg_%s_out" % name] = r
        aggs.append(name)

    s, o = ragged(rng, [1, 3, 7, 25], 10, 12)
    agg("default_mean_norm", s, o, "default", normalization=True, crop_agg="mean")
    agg("default_max_raw", s, o, "default", normalization=False, crop_agg="max")
    agg("topk_k3", s, o, "top_k", k=3, normalization=True, crop_agg="mean")
    agg("topk_k40_max_raw", s, o, "top_k", k=40, normalization=False, crop_agg="max")
    s1, o1 = ragged(rng, [1, 2, 9], 1, 7)
    agg("default_one_crop", s1, o1, "default", normalization=True, crop_agg="mean")
    agg("topk_one_crop_raw", s1, o1, "top_k", k=2, normalization=False, crop_agg="mean")
    s, o = ragged(rng, [1, 5, 37, 120, 333], 10, 20)
    agg("sliding_norm", s, o, "sliding_window", spans=[1, 2, 4, 8, 16], overlap=0.2, norm=True, fps=1)
    agg("sliding_raw", s, o, "sliding_window", spans=[1, 2, 4, 8, 16], overlap=0.2, norm=False, fps=1)
    agg("sliding_fps2", s, o, "sliding_window", spans=[1, 2, 4, 8, 16], overlap=0.2, norm=False, fps=2)
    agg("sliding_spans13_half", s, o, "sliding_window", spans=[1, 3], overlap=0.5, norm=True, fps=1)
    s, o = ragged(rng, [1, 2, 7, 30], 10, 3 * 5)
    agg("tpp", s, o, "tpp", num_class=5)
    s, o = ragged(rng, [2, 3, 50], 4, 6, scale=1.0)
    s = np.round(s * 2) / 2                                # exact ties
    s[o[1]:o[2]] = 0.25                                    # a constant video
    agg("ties_default", s, o, "default", normalization=True, crop_agg="mean")
    agg("ties_topk", s, o, "top_k", k=4, normalization=False, crop_agg="max")
    agg("ties_sliding", s, o, "sliding_window", spans=[1, 2, 4, 8, 16], overlap=0.2, norm=True, fps=1)
    s, o = ragged(rng, [4, 6, 20, 3], 3, 5)
    s[1, :, 2] = np.inf                                    # +inf logits in video 0
    s[o[1] + 2, 1, 0] = -np.inf                            # -inf in video 1
    s[o[2]:o[3], :, 3] = -np.inf                           # a class at -inf all through video 2
    s[o[3] + 1, 2, 4] = np.nan                             # a NaN tick in video 3
    for mode, kw in (("default", dict(normalization=True, crop_agg="mean")), ("default", dict(normalization=False, crop_agg="max")),
                     ("top_k", dict(k=2, normalization=True, crop_agg="mean")), ("top_k", dict(k=5, normalization=False, crop_agg="max")),
                     ("sliding_window", dict(spans=[1, 2, 4, 8, 16], overlap=0.2, norm=True, fps=1)),
                     ("sliding_window", dict(spans=[1, 2], overlap=0.2, norm=False, fps=1))):
        agg("nonfinite_%s_%d" % (mode, len(aggs)), s, o, mode, **kw)
    out["agg_fixtures"] = np.array(aggs)

    # fusion of three [V, K] streams (the reference adds into its major argument: it gets a copy)
    streams = [(rng.standard_normal((6, 9)) * 2).astype(np.float32) for _ in range(3)]
    for norm in (True, False):
        r = np.stack([vf.default_fusion_func(streams[0][v].copy(), [streams[1][v], streams[2][v]], [1, 1.5], norm=norm) for v in range(6)])
        out["fuse_%s_out" % ("norm" if norm else "raw")] = r
    out["fuse_streams"], out["fuse_weights"] = np.stack(streams), np.array([1, 1.5])
    x = (rng.standard_normal((5, 400)) * 4).astype(np.float32)
    x[1, 3], x[2, 7], x[3, 0] = 80.0, -np.inf, np.nan
    with np.errstate(all="ignore"):
        out["softmax_in"], out["softmax_out"], out["softmax_t2_out"] = x, mt.softmax(x), mt.softmax(x, T=2)

    # metrics over score_dict / video_list: multi-label videos, videos missing from score_dict, a class without positives
    mets = []

    def metrics(name, scores, label_sets, missing):
        ids = ["v%03d" % i for i in range(len(scores))]
        vlist = [Video(i, ls) for i, ls in zip(ids, label_sets)] + [Video("gone%d" % j, [0]) for j in range(missing)]
        sd = dict(zip(ids, scores))
        lv = np.array([i for i, ls in enumerate(label_sets) for _ in sorted(set(ls))], np.int32)
        lab = np.array([c for ls in label_sets for c in sorted(set(ls))], np.int32)
        p = "met_%s_" % name
        out[p + "scores"], out[p + "label_video"], out[p + "label"], out[p + "missing"] = np.stack(scores), lv, lab, missing
        for k in (1, 3, 5):
            out[p + "acc_k%d" % k] = np.array([mt.top_k_acc(set(ls), s_, k=k) for ls, s_ in zip(label_sets, scores)])
            out[p + "hit_k%d" % k] = np.array([mt.top_k_hit(set(ls), s_, k=k) for ls, s_ in zip(label_sets, scores)])
            out[p + "top_k_accuracy_k%d" % k] = mt.top_k_accuracy(sd, vlist, k)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[p + "video_mean_ap"] = mt.video_mean_ap(sd, vlist)
        mets.append(name)

    K = 10
    labs = [sorted(set(rng.integers(0, K - 1, rng.integers(1, 4)).tolist())) for _ in range(40)]   # class K-1: no positive video
    metrics("basic", list((rng.standard_normal((40, K))).astype(np.float32)), labs, 3)
    q = list(np.round(rng.standard_normal((30, 8)) * 1.5).astype(np.float32))                        # quantised: ties everywhere
    q[0][:] = 0.0
    metrics("ties", q, [sorted(set(rng.integers(0, 8, rng.integers(1, 3)).tolist())) for _ in range(30)], 0)
    metrics("dense", list(rng.random((120, 16)).astype(np.float64)), [sorted(set(rng.integers(0, 16, rng.integers(1, 5)).tolist())) for _ in range(120)], 5)
    out["met_fixtures"] = np.array(mets)

    mcas = []

    def mca(name, scores, labels):
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            out["mca_%s_value" % name] = mt.mean_class_accuracy(scores, labels)
        out["mca_%s_scores" % name], out["mca_%s_labels" % name] = scores, np.asarray(labels, np.int32)
        mcas.append(name)

    sc = rng.standard_normal((50, 6)).astype(np.float32)
    lb = rng.integers(0, 6, 50)
    mca("plain", sc + np.eye(6, dtype=np.float32)[lb] * 1.5, lb)
    sc2 = sc.copy()
    sc2[0, 5] = 100.0                                      # class 5 predicted once, never labelled: NaN
    mca("unlabelled_prediction", sc2, np.where(lb == 5, 0, lb))
    sc3 = np.round(sc * 2).astype(np.float32) / 2          # argmax ties: the first maximum
    mca("ties", sc3, lb)
    out["mca_fixtures"] = np.array(mcas)

    np.savez_compressed(os.path.join(GOLD, "video_funcs.npz"), **out)
    print("wrote", os.path.join(GOLD, "video_funcs.npz"), len(aggs), "aggregation,", len(mets), "metrics,", len(mcas), "class-accuracy fixtures")


if __name__ == "__main__":
    main()
