"""The AR-AN oracle (oracle/anet_proposal_oracle.py) against tests/golden/anet_proposal.npz, which holds what the real
ActivityNet toolkit computed (oracle/gen_golden_anet_proposal.py): recall, avg_recall, proposals_per_video, nr and the area,
bitwise; the JSON loaders of ops/proposal_eval.py against the toolkit's data frames; the library's argument checks.  No GPU."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from oracle import anet_proposal_oracle as O
from test_proplist_host import same

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anet_proposal.npz"))
FIXTURES = [str(x) for x in GOLD["fixtures"]]


def fixture(name):
    """-> dict(boxes, scores, counts, gt_seg, gt_offsets, gt_counts, thresholds, max_avg (None: the default))"""
    src = str(GOLD[name + "_inputs"]) + "_"
    f = {k: GOLD[src + k] for k in ("boxes", "scores", "counts", "gt_seg", "gt_offsets")}
    f["gt_counts"] = np.diff(f["gt_offsets"])
    f["thresholds"] = GOLD[name + "_thresholds"]
    f["max_avg"] = float(GOLD[name + "_max_avg"]) or None
    return f


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_toolkit(name):
    f = fixture(name)
    o = O.average_recall(f["boxes"], f["scores"], f["counts"], f["gt_seg"], f["gt_counts"], f["max_avg"], f["thresholds"])
    for k in ("recall", "avg_recall", "proposals_per_video", "nr"):
        assert same(o[k], GOLD[name + "_" + k]), k
    assert o["total_nr"] == int(GOLD[name + "_total_nr"])
    assert O.area(o["avg_recall"], o["proposals_per_video"]) == (float(GOLD[name + "_auc"]), float(GOLD[name + "_auc_percent"]))


def test_fixtures_cover_the_edges():
    f = fixture("noprop_t0")
    assert (f["counts"][f["gt_counts"] > 0] == 0).sum() == 2 and f["thresholds"][0] == 0.0
    assert GOLD["noprop_t0_recall"][0].max() > 0                    # the phantom column matches threshold 0.0
    nr, f = GOLD["nr_zero_nr"], fixture("nr_zero")
    assert (nr[f["counts"] > 0] == 0).any() and (nr > 0).any()
    f = fixture("ratio_lt1")
    p_all, V = int(f["counts"].sum()), int((f["gt_counts"] > 0).sum())
    assert float(p_all) / V * float(V) / p_all < 1 and (GOLD["ratio_lt1_nr"] == f["counts"] - 1).all()
    f = fixture("outside")
    assert (f["gt_counts"] == 0).sum() >= 3 and f["counts"][f["gt_counts"] == 0].sum() > 0
    f = fixture("degenerate")
    assert np.isnan(f["boxes"]).any() and np.isnan(f["gt_seg"]).any() and (f["boxes"][:, 1] < f["boxes"][:, 0]).any()
    f = fixture("ties")
    s = f["scores"]
    assert np.isnan(s).sum() > 1 and (s == 0).sum() > 1 and np.signbit(s[s == 0]).any() and f["counts"].max() <= 16
    f = fixture("integer")
    assert (f["boxes"] == np.round(f["boxes"])).all()


def test_tiou_on_a_threshold_matches():
    # [0, 2] against [0, 1] is 0.5 exactly, and tiou >= t matches it
    assert O.segment_iou([[0.0, 2.0]], [[0.0, 1.0]])[0, 0] == 0.5
    assert np.isnan(O.segment_iou([[3.0, 3.0]], [[3.0, 3.0]])[0, 0])     # 0 / 0
    assert GOLD["on_threshold_recall"][0, -1] == 1.0


def test_rank_rule():
    s = np.array([0.5, np.nan, -0.0, 0.5, 0.0, np.nan, 1.0])
    assert O.rank(s).tolist() == [5, 1, 6, 3, 0, 4, 2]              # NaN first, descending, ties by descending row


def test_loaders_against_the_toolkit_frames():
    from ops import proposal_eval as E
    gt_j, pr_j = json.loads(str(GOLD["json_gt_text"])), json.loads(str(GOLD["json_pr_text"]))
    blocked = [str(x) for x in GOLD["json_blocked"]]
    gt = E.load_anet_ground_truth(gt_j, "validation", blocked)
    vids = GOLD["json_gt_video"].tolist()
    assert gt["video_ids"] == list(dict.fromkeys(vids))
    assert same(gt["segments"], GOLD["json_gt_seg"]) and same(gt["labels"].astype(np.int64), GOLD["json_gt_label"])
    assert np.diff(gt["gt_offsets"]).tolist() == [vids.count(v) for v in gt["video_ids"]]
    pr = E.load_anet_proposals(pr_j, gt["video_ids"], blocked)
    pv = GOLD["json_pr_video"].tolist()
    # the toolkit's rows grouped by video: what get_group returns, in the packed order
    order = [i for v in pr["video_ids"] for i in range(len(pv)) if pv[i] == v]
    assert sorted(order) == list(range(len(pv))) and pr["counts"] == [pv.count(v) for v in pr["video_ids"]]
    assert same(pr["boxes"], GOLD["json_pr_seg"][order]) and same(pr["scores"], GOLD["json_pr_score"][order])
    assert blocked[0] not in pr["video_ids"] and blocked[1] not in pr["video_ids"] and len(pr["video_ids"]) > len(gt["video_ids"])
    with pytest.raises(IOError):
        E.load_anet_ground_truth({"database": {}})
    with pytest.raises(IOError):
        E.load_anet_proposals({"results": {}}, [])


def test_rejected_arguments_return_before_any_launch():
    """argument validation needs no device: the library returns SSNB_EINVAL (1), launches nothing, and the workspace query
    returns 0 for exactly those arguments"""
    from ssn_b200 import _lib
    lib = _lib.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(8)                                   # a non-null pointer that is never dereferenced
    ok, bad, empty = (C.c_int64 * 3)(0, 2, 3), (C.c_int64 * 3)(0, 2, 1), (C.c_int64 * 3)(0, 0, 0)
    thr = (C.c_double * 2)(0.5, 0.7)
    nan_thr = (C.c_double * 2)(0.5, math.nan)
    ws = lib.ssnb_proposal_ar_workspace_bytes(2, 10, ok, 2)
    assert ws > 0 and lib.ssnb_proposal_ar_workspace_bytes(2, 1000, ok, 2) > ws + 20000          # 24 bytes per row

    def call(V=2, rows=10, off=ok, t=thr, n_thr=2, max_avg=0.0, boxes=one, recall=one, ws_bytes=ws):
        return lib.ssnb_proposal_ar(boxes, one, rows, one, one, V, one, off, one, t, n_thr, max_avg, recall, one, one, one, None, None,
                                    one, ws_bytes, None)
    for kw, why in ((dict(V=0), "no video"), (dict(rows=-1), "negative rows"), (dict(rows=1 << 31), "rows past INT_MAX"),
                    (dict(off=bad), "descending offsets"), (dict(off=empty), "no ground truth"), (dict(n_thr=0), "no threshold"),
                    (dict(n_thr=65), "65 thresholds")):
        assert call(**kw) == 1, why
        assert lib.ssnb_proposal_ar_workspace_bytes(kw.get("V", 2), kw.get("rows", 10), kw.get("off", ok), kw.get("n_thr", 2)) == 0, why
    assert lib.ssnb_proposal_ar_workspace_bytes(2, 10, None, 2) == 0
    assert call(t=nan_thr) == 1
    assert call(max_avg=math.inf) == 1 and call(max_avg=math.nan) == 1
    assert call(boxes=None) == 1 and call(recall=None) == 1
    assert call(ws_bytes=ws - 1) == 1
    assert b"proposal_ar" in lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0


def test_cpu_tensors_are_refused():
    import torch
    from ops import proposal_eval as E
    z = torch.zeros(1, 2, dtype=torch.float64)
    with pytest.raises(RuntimeError):
        E.average_recall_packed(z, torch.zeros(1, dtype=torch.float64), [0], [1], np.zeros((1, 2)), [0, 1])
    with pytest.raises(RuntimeError):
        E.evaluate_proposals({}, {}, device="cpu")
