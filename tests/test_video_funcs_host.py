"""The video-level aggregation and metrics oracle (oracle/video_funcs_oracle.py) against tests/golden/video_funcs.npz, which
holds what the reference's own ops/video_funcs.py and ops/metrics.py computed (oracle/gen_golden_video_funcs.py); the
library's argument checks, which refuse before any launch; the modules import without sklearn.  No GPU."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import video_funcs_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "video_funcs.npz"))
AGGS = [str(x) for x in GOLD["agg_fixtures"]]
METS = [str(x) for x in GOLD["met_fixtures"]]
MCAS = [str(x) for x in GOLD["mca_fixtures"]]


def agg_fixture(name):
    src = str(GOLD["agg_%s_inputs" % name])
    return GOLD["agg_%s_scores" % src], GOLD["agg_%s_offsets" % src], json.loads(str(GOLD["agg_%s_params" % name]))


def ulp_diff(a, b):
    """elementwise distance in units in the last place of the wider type; NaN positions must agree"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape
    assert (np.isnan(a) == np.isnan(b)).all()
    m = ~np.isnan(a)
    it = np.int32 if a.dtype == np.float32 else np.int64
    ia, ib = a[m].view(it).astype(np.int64), b[m].view(it).astype(np.int64)
    ia = np.where(ia < 0, np.iinfo(it).min - ia, ia)        # ordered integers: -0 and +0 one apart
    ib = np.where(ib < 0, np.iinfo(it).min - ib, ib)
    return np.abs(ia - ib).max(initial=0)


@pytest.mark.parametrize("name", AGGS)
def test_aggregation_oracle_equals_reference(name):
    scores, off, p = agg_fixture(name)
    mode = p.pop("mode")
    with np.errstate(all="ignore"):
        got = O.aggregate_packed(scores, off, mode, **p)
    want = GOLD["agg_%s_out" % name]
    assert got.dtype == want.dtype and got.shape == want.shape
    # the oracle runs numpy in the reference's order: bitwise, but for the float32 exp of the softmax (a rounded float64 exp
    # against libm's expf): 2 ulp
    norm = p.get("normalization", p.get("norm", False))
    assert ulp_diff(got, want) <= (2 if norm else 0), name


def test_fusion_and_softmax_oracle_equal_reference():
    st, w = GOLD["fuse_streams"], [float(x) for x in GOLD["fuse_weights"]]
    for norm in (True, False):
        got = O.fuse(st[0], [st[1], st[2]], w, norm)
        assert ulp_diff(got, GOLD["fuse_%s_out" % ("norm" if norm else "raw")]) <= (2 if norm else 0)
    with np.errstate(all="ignore"):
        assert ulp_diff(O.softmax(GOLD["softmax_in"]), GOLD["softmax_out"]) <= 2
        assert ulp_diff(O.softmax(GOLD["softmax_in"], 2), GOLD["softmax_t2_out"]) <= 2


def met_fixture(name):
    p = "met_%s_" % name
    sc, lv, lab = GOLD[p + "scores"], GOLD[p + "label_video"], GOLD[p + "label"]
    sets = [set(lab[lv == i].tolist()) for i in range(len(sc))]
    return sc, lv, lab, sets


@pytest.mark.parametrize("name", METS)
def test_metrics_oracle_equals_reference(name):
    sc, _, _, sets = met_fixture(name)
    p = "met_%s_" % name
    for k in (1, 3, 5):
        acc = np.array([O.top_k_acc(ls, s, k) for ls, s in zip(sets, sc)])
        assert (acc == GOLD[p + "acc_k%d" % k]).all()
        assert (np.array([O.top_k_hit(ls, s, k) for ls, s in zip(sets, sc)]) == GOLD[p + "hit_k%d" % k]).all()
        assert O.top_k_accuracy(sc, sets, k) == float(GOLD[p + "top_k_accuracy_k%d" % k])
    assert abs(O.video_mean_ap(sc, sets)[0] - float(GOLD[p + "video_mean_ap"])) <= 1e-12


@pytest.mark.parametrize("name", MCAS)
def test_mean_class_accuracy_oracle_equals_reference(name):
    got = O.mean_class_accuracy(GOLD["mca_%s_scores" % name], GOLD["mca_%s_labels" % name])
    want = float(GOLD["mca_%s_value" % name])
    assert (np.isnan(got) and np.isnan(want)) or abs(got - want) <= 1e-12


def test_fixtures_cover_the_edges():
    Ts = {n: np.diff(agg_fixture(n)[1]) for n in AGGS}
    params = {n: agg_fixture(n)[2] for n in AGGS}
    assert any(1 in t for t in Ts.values())                                                     # T = 1
    sl = [n for n in AGGS if params[n]["mode"] == "sliding_window"]
    assert any((Ts[n] < 16).any() for n in sl) and any((Ts[n] % 13).any() for n in sl)          # T < span, T % step != 0
    assert any(params[n]["mode"] == "top_k" and (Ts[n] < params[n]["k"]).any() for n in AGGS)   # k > T
    assert any(agg_fixture(n)[0].shape[1] == 1 for n in AGGS)                                   # one crop
    assert any(params[n].get("crop_agg") == "max" for n in AGGS)
    assert {params[n].get("normalization", params[n].get("norm")) for n in AGGS} >= {True, False}
    assert any(params[n].get("fps") == 2 for n in AGGS)
    tpp = [n for n in AGGS if params[n]["mode"] == "tpp"]
    assert any((Ts[n] < agg_fixture(n)[0].shape[2] // params[n]["num_class"]).any() for n in tpp)   # T < stage
    s = agg_fixture("nonfinite_default_%d" % AGGS.index([n for n in AGGS if n.startswith("nonfinite")][0]))[0]
    assert np.isposinf(s).any() and np.isneginf(s).any() and np.isnan(s).any()
    sc, _, lab, sets = met_fixture("basic")
    assert max(len(x) for x in sets) > 1 and int(GOLD["met_basic_missing"]) > 0                  # multi-label, missing videos
    assert set(range(sc.shape[1])) - set(lab.tolist())                                          # a class with no positive video
    assert np.isnan(float(GOLD["mca_unlabelled_prediction_value"]))


def test_tie_rule():
    s = np.array([0.5, np.nan, -0.0, 0.5, 0.0, 1.0, 0.5], np.float32)
    assert O.rank(s).tolist() == [1, 5, 6, 3, 0, 4, 2]       # NaN first, descending, equal scores the higher class first
    assert O.top_k_acc({0, 3}, s, 4) == (1, 2) and O.top_k_acc({0, 3}, s, 5) == (2, 2)


def test_library_refuses_before_any_launch():
    from ssn_b200._lib import lib
    off = (C.c_int64 * 3)(0, 4, 4)                                      # a video without ticks
    good = (C.c_int64 * 3)(0, 4, 9)
    sp = (C.c_int * 2)(1, 2)
    n0 = lib.ssnb_global_launch_count()
    fake = C.c_void_p(16)
    calls = [
        (off, 2, 10, 5, 0, 0, 1, sp, 2, 0.2, 1, 5),                     # T = 0
        (good, 2, 10, 5, 7, 0, 1, sp, 2, 0.2, 1, 5),                    # unknown mode
        (good, 2, 10, 5, 2, 1, 1, sp, 2, 0.2, 1, 5),                    # sliding window with the crop max
        (good, 2, 10, 5, 1, 0, 0, sp, 2, 0.2, 1, 5),                    # top_k = 0
        (good, 2, 10, 5, 2, 0, 1, sp, 2, 1.0, 1, 5),                    # overlap 1
        (good, 2, 10, 5, 2, 0, 1, sp, 2, 0.2, 0, 5),                    # fps 0
        (good, 2, 10, 6, 3, 0, 1, sp, 2, 0.2, 1, 4),                    # tpp: D not a multiple of num_class
    ]
    for a in calls:
        assert lib.ssnb_video_aggregate_workspace_bytes(*a) == 0
        assert lib.ssnb_video_aggregate(fake, a[0], fake, *a[1:6], 0, *a[6:], fake, fake, 1 << 30, None) == 1
    a = calls[0]
    assert lib.ssnb_video_aggregate(fake, good, fake, 2, 10, 6, 3, 0, 1, 1, sp, 2, 0.2, 1, 3, fake, fake, 1 << 30, None) == 1  # tpp + norm
    assert lib.ssnb_video_fuse(fake, None, None, 9, 4, 4, 1, 1.0, fake, None) == 1
    assert lib.ssnb_video_metrics_workspace_bytes(4, 2000) == 0
    ws = lib.ssnb_video_metrics_workspace_bytes(4, 10)
    assert ws > 0
    args = [fake, 0, 4, 10, fake, fake, 3, None, 3] + [fake] * 8 + [fake, ws, None]
    assert lib.ssnb_video_metrics(*args[:8], 0, *args[9:]) == 1        # top_k = 0
    assert lib.ssnb_video_metrics(*args[:-2], ws - 1, None) == 1       # workspace too small
    assert lib.ssnb_global_launch_count() == n0


def test_modules_import_without_sklearn():
    code = ("import sys; sys.modules['sklearn'] = None; sys.path[:0] = %r; import ops.video_funcs, ops.metrics; "
            "assert 'sklearn' not in [m.split('.')[0] for m in sys.modules if sys.modules[m] is not None]"
            % [ROOT, os.path.join(ROOT, "action-detection_b200")])
    subprocess.check_call([sys.executable, "-c", code])
