"""The staged proposal check (oracle/proposal_check.py) without a GPU: a numpy stand-in of the traced call passes it, and
one error planted at one stage is reported at that stage only; the oracle's NaN-first NMS rule; the oracle's box search
and NMS against the reference's own functions (vendored under oracle/_ref by build(); tests/golden/proposals_nms.npz
where they are absent)."""
import importlib
import os
import sys
import types

import numpy as np
import pytest

from oracle import proposal_check as C
from oracle import proposal_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_OPS = os.path.join(ROOT, "oracle", "_ref", "ops")


def _case():
    """K = 3, cls = 1: ties (quantised, zero foreground, regular runs), NaN and inf scores, a -inf row; minimum_len 4"""
    g = np.random.RandomState(5)
    videos = [(C.make_scores(kind, T, g, K=3, cls=1), T / 7.0) for kind, T in
              (("smooth", 300), ("quant", 257), ("zero_fg", 200), ("nan", 400), ("inf", 150), ("neginf_row", 90),
               ("runs_regular", 256), ("nan_bg", 64), ("smooth", 1))]
    f, offsets, durs = C.pack(videos)
    return f, offsets, durs, dict(cls=1, bw=3, minimum_len=4.0)


def _run(plant=None):
    f, offsets, durs, kw = _case()
    res = C.standin(f, offsets, durs, plant=plant, **kw)
    return C.check(res, f, offsets, durs, **kw), res


def test_standin_passes_and_covers_ties_and_nan():
    chk, _ = _run()
    chk.assert_ok()
    s = chk.stats
    print(chk.report())
    assert s["videos"] == 9 and s["tied_boxes"] > 1000 and s["nan_boxes"] > 100 and s["e2e_videos"] == 9
    assert not chk.failed() and {r.stage for r in chk.records} == set(C.STAGES)


def _flip_label(stage, v, x):
    if stage == "labels" and v == 0:
        k, t = 6, 150                                    # threshold 0.5, far from the smoothed value there
        x[k, t] = not x[k, t]
    return x


def _raw_end(stage, v, x):
    if stage == "raw" and v == 0:
        x[1][3] += 1
    return x


def _drop_last_of_block(stage, v, x):
    """the last box of the first (threshold, tolerance) block with boxes"""
    if stage == "raw" and v == 0:
        s, e, sc = x
        i = len(s) - 1
        return np.delete(s, i), np.delete(e, i), np.delete(sc, i)
    return x


def _swap_ties(stage, v, x):
    """video 2 scores every box 0: the first two survivors, swapped in the order NMS reads"""
    if stage == "nms" and v == 2:
        def nms(s, e, sc, thresh):
            keep = P.temporal_nms(s, e, sc, thresh)
            perm = np.arange(len(s))
            perm[[keep[0], keep[1]]] = perm[[keep[1], keep[0]]]
            return perm[P.temporal_nms(s[perm], e[perm], sc[perm], thresh)]
        return nms
    return x


def _nan_last(stage, v, x):
    if stage == "nms" and v == 3:
        def nms(s, e, sc, thresh):                      # the rule the oracle had before: NaN ranks last
            order, keep, d = np.argsort(-sc, kind="stable"), [], e - s + 1
            while order.size:
                i = order[0]
                keep.append(i)
                inter = np.minimum(e[i], e[order[1:]]) - np.maximum(s[i], s[order[1:]]) + 1
                order = order[np.where(inter / (d[i] + d[order[1:]] - inter).astype(float) <= thresh)[0] + 1]
            return np.array(keep, np.int64)
        return nms
    return x


def _seconds_ulp(stage, v, x):
    if stage == "seconds" and v == 0:
        x[0, 1] = np.nextafter(x[0, 1], np.inf)
    return x


def _keep_short(stage, v, x):
    if stage == "kept" and v == 0:
        keep, ok = x
        ok = ok.copy()
        ok[_first_false(ok)] = True
        return keep, ok
    return x


def _first_false(ok):
    assert not ok.all(), "the case needs a survivor that fails the length filter"
    return int(np.nonzero(~ok)[0][0])


@pytest.mark.parametrize("plant, stage", [(_flip_label, "labels"), (_raw_end, "raw"), (_drop_last_of_block, "raw"),
                                          (_swap_ties, "nms"), (_nan_last, "nms"), (_seconds_ulp, "filter"),
                                          (_keep_short, "filter")])
def test_planted_error_is_reported_at_its_stage_only(plant, stage):
    chk, _ = _run(plant)
    assert chk.failed() == {stage}, chk.failures()


def test_nan_scored_boxes_rank_first():
    """400 ticks, K = 2, foreground runs of 40 ticks and a NaN in the foreground column at background tick 150, gen_prop's
    defaults: the boxes that span the NaN score NaN, and the first survivors are NaN-scored, in search order"""
    t = np.arange(400)
    f = np.zeros((400, 2), np.float32)
    f[:, 1] = np.where((t // 40) % 2 == 0, 3.0, -3.0)
    f[150, 1] = np.nan
    r = P.gen_prop(f, 40.0)
    nan = np.isnan(r["raw_score"])
    assert nan.sum() > 100
    k = np.isnan(r["nms_score"])
    assert k.any() and not k[np.argmin(k):].any() and k[0]
    keep = P.temporal_nms(r["raw_start"], r["raw_end"], r["raw_score"], 0.9)
    assert (np.diff(keep[:k.sum()]) > 0).all()          # NaN survivors in search order


def test_nan_rule_ignores_the_sign():
    s, e = np.array([0, 10, 20, 30]), np.array([5, 15, 25, 35])
    sc = np.array([1.0, np.nan, np.inf, np.nan], np.float32)
    sc.view(np.uint32)[3] = 0xffc00000
    assert P.temporal_nms(s, e, sc, 0.5).tolist() == [1, 3, 2, 0]


def test_nms_matches_reference_golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "proposals_nms.npz"))
    for c in range(int(z["n_cases"])):
        p = "c%d_" % c
        keep = P.temporal_nms(z[p + "start"], z[p + "end"], z[p + "score"], float(z[p + "thresh"]))
        np.testing.assert_array_equal(keep, z[p + "kept"], err_msg=str(c))
    # the fixture's cases are still the ones nms_cases draws
    for c, (s, e, sc, th) in enumerate(C.nms_cases(7)):
        assert (s == z["c%d_start" % c]).all() and (sc.view(np.uint32) == z["c%d_score" % c].view(np.uint32)).all()


def _reference():
    """the vendored ops/sequence_funcs.py as a module of its own package (this repository's `ops` keeps its name)"""
    if not os.path.exists(os.path.join(REF_OPS, "sequence_funcs.py")):
        pytest.skip("oracle/_ref holds no vendored reference (build() vendors it where a checkout exists)")
    name = "_vendored_reference_ops"
    if name + ".sequence_funcs" not in sys.modules:
        pkg = types.ModuleType(name)
        pkg.__path__ = [REF_OPS]
        sys.modules[name] = pkg
        try:
            importlib.import_module(name + ".metrics")
        except ImportError:                             # metrics.py imports sklearn; the functions used here need none of it
            stub = types.ModuleType(name + ".metrics")
            stub.softmax = P.softmax
            sys.modules[name + ".metrics"] = stub
    sf = importlib.import_module(name + ".sequence_funcs")
    assert sf.nms is None
    return sf


def _label_rows(g):
    rows = []
    for T in (1, 2, 3, 17, 64, 255, 256, 700, 1999):
        for p in (0.0, 1.0, 0.02, 0.3):
            rows.append(np.repeat(g.rand((T + 7) // 8) < p, 8)[:T] if p not in (0.0, 1.0) else np.full(T, bool(p)))
        U = min(T // 2, 60)
        if U:
            rows.append(C.run_labels(T, U, g, regular=True))
            rows.append(C.run_labels(T, U, g, regular=True, end_fg=True))
            rows.append(C.run_labels(T, U, g))
    return rows


def test_build_boxes_matches_reference_search():
    sf = _reference()
    g = np.random.RandomState(11)
    tol = (0.0, 0.5, 1.0, 1.3, -0.2, 0.05)
    for row in _label_rows(g):
        frm = (g.randn(len(row)) * 3).astype(np.float32)
        if len(row) > 5:
            frm[::5] = np.round(frm[::5])
        ref = sf.build_box_by_search([(0, row, frm)], tol)
        s, e, sc = P.build_boxes(row, frm, tol)
        assert len(ref) == len(s), len(row)
        if ref:
            assert (np.array([b[0] for b in ref]) == s).all() and (np.array([b[1] for b in ref]) == e).all()
            assert (np.array([b[3] for b in ref], np.float32).view(np.uint32) == sc.view(np.uint32)).all()


def test_nms_matches_reference_on_random_cases():
    sf = _reference()
    for seed in (1, 2, 3):
        for s, e, sc, thresh in C.nms_cases(seed):
            kept = sf.temporal_nms_fallback([(a, b, i, x) for i, (a, b, x) in enumerate(zip(s.tolist(), e.tolist(), sc))], thresh)
            assert [k[2] for k in kept] == P.temporal_nms(s, e, sc, thresh).tolist()
