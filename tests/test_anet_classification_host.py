"""The classification oracle (oracle/anet_classification_oracle.py) against tests/golden/anet_classification.npz, which holds
what the real ActivityNet toolkit computed (oracle/gen_golden_anet_classification.py): per-class AP, hit@k and average
hit@k, bitwise; the JSON loaders of ops/classification_eval.py against the toolkit's data frames and its errors; the
library's argument checks.  No GPU."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import anet_classification_oracle as O
from test_proplist_host import same

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anet_classification.npz"))
FIXTURES = [str(x) for x in GOLD["fixtures"]]


def fixture(name):
    """-> dict(video, label, score, gt_video, gt_label, V, K, top_k)"""
    src = str(GOLD[name + "_inputs"]) + "_"
    f = {k: GOLD[src + k] for k in ("video", "label", "score", "gt_video", "gt_label")}
    f["V"], f["K"], f["top_k"] = int(GOLD[src + "V"]), int(GOLD[src + "K"]), int(GOLD[name + "_top_k"])
    return f


def oracle(f):
    return O.classification(f["video"], f["label"], f["score"], f["gt_video"], f["gt_label"], f["V"], f["K"], f["top_k"])


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_toolkit(name):
    o = oracle(fixture(name))
    assert same(o["ap"], GOLD[name + "_ap"])
    assert o["hit_at_k"] == float(GOLD[name + "_hit_at_k"]) and o["avg_hit_at_k"] == float(GOLD[name + "_avg_hit_at_k"])
    assert float(o["ap"].mean()) == float(GOLD[name + "_map"])


def test_fixtures_cover_the_edges():
    f = fixture("edges")
    pairs = f["label"].astype(np.int64) * f["V"] + f["video"]
    assert len(np.unique(pairs)) < len(pairs)                                   # a repeated (video, label) row
    assert np.isnan(f["score"]).any()
    gtv = set(f["gt_video"].tolist())
    assert set(f["video"].tolist()) - gtv                                       # predictions for videos without ground truth
    assert gtv - set(f["video"].tolist())                                       # ground-truth videos without a prediction
    assert (np.bincount(f["gt_video"], minlength=f["V"]) > 1).any()             # multi-label videos
    assert set(range(f["K"])) - set(f["label"].tolist())                        # a class with no prediction
    assert GOLD["edges_ap"][sorted(set(range(f["K"])) - set(f["label"].tolist()))].max() == 0.0
    f = fixture("ties")
    s = f["score"]
    assert np.isnan(s).sum() > 1 and (s == 0).sum() > 1 and np.signbit(s[s == 0]).any() and len(np.unique(s[~np.isnan(s)])) < len(s)
    assert max(np.bincount(f["label"]).max(), np.bincount(f["video"]).max()) <= 16
    assert sorted(int(GOLD[n + "_top_k"]) for n in ("anet", "anet_k1", "anet_k5")) == [1, 3, 5]
    assert len(GOLD["json_blocked"]) == 2


def test_rank_rule():
    s = np.array([0.5, np.nan, -0.0, 0.5, 0.0, np.nan, 1.0])
    assert O.rank(s).tolist() == [5, 1, 6, 3, 0, 4, 2]              # NaN first, descending, ties by descending row


def test_loaders_against_the_toolkit_frames():
    from ops import classification_eval as E
    gt_j, pr_j = json.loads(str(GOLD["json_gt_text"])), json.loads(str(GOLD["json_pr_text"]))
    blocked = [str(x) for x in GOLD["json_blocked"]]
    gt = E.load_anet_classification_ground_truth(gt_j, "validation", blocked)
    assert list(gt["activity_index"]) == GOLD["frame_classes"].tolist() and list(gt["activity_index"].values()) == list(range(len(gt["activity_index"])))
    assert gt["video_ids"] == sorted(set(GOLD["frame_gt_video"].tolist()))
    assert [gt["video_ids"][i] for i in gt["video"]] == GOLD["frame_gt_video"].tolist()
    assert same(gt["label"].astype(np.int64), GOLD["frame_gt_label"])
    pr = E.load_anet_classification_predictions(pr_j, gt, blocked)
    assert pr["video_ids"][:len(gt["video_ids"])] == gt["video_ids"]
    assert [pr["video_ids"][i] for i in pr["video"]] == GOLD["frame_pr_video"].tolist()
    assert same(pr["label"].astype(np.int64), GOLD["frame_pr_label"]) and same(pr["score"], GOLD["frame_pr_score"])
    assert blocked[0] not in gt["video_ids"] and blocked[1] not in pr["video_ids"] and len(pr["video_ids"]) > len(gt["video_ids"])
    # the packed fixture is what the loaders give
    f = fixture("json")
    assert same(pr["video"], f["video"]) and same(gt["video"], f["gt_video"]) and f["V"] == len(pr["video_ids"])


def test_loader_errors():
    from ops import classification_eval as E
    with pytest.raises(IOError, match="valid ground truth"):
        E.load_anet_classification_ground_truth({"database": {}, "version": ""})
    gt = E.load_anet_classification_ground_truth({"database": {"a": {"subset": "validation", "annotations": [{"label": "x"}]}},
                                                  "taxonomy": [], "version": ""})
    with pytest.raises(IOError, match="valid prediction"):
        E.load_anet_classification_predictions({"results": {}, "version": ""}, gt)
    with pytest.raises(ValueError, match="'y'"):
        E.load_anet_classification_predictions({"results": {"a": [{"label": "y", "score": 1}]}, "version": "", "external_data": {}}, gt)
    # a blocked video's unknown label is never looked up, as in the toolkit
    pr = E.load_anet_classification_predictions({"results": {"b": [{"label": "y", "score": 1}], "a": [{"label": "x", "score": 0.5}]},
                                                 "version": "", "external_data": {}}, gt, blocked_videos=["b"])
    assert pr["video"].tolist() == [0] and pr["label"].tolist() == [0] and pr["video_ids"] == ["a"]


def test_rejected_arguments_return_before_any_launch():
    """argument validation needs no device: the library returns SSNB_EINVAL (1), launches nothing, and the workspace query
    returns 0 for exactly those arguments"""
    from ssn_b200 import _lib
    lib = _lib.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(8)                                   # a non-null pointer that is never dereferenced
    ws = lib.ssnb_classification_ap_workspace_bytes(10, 4, 3, 5)
    assert ws > 0 and lib.ssnb_classification_ap_workspace_bytes(1010, 4, 3, 5) > ws + 60000        # about 70 bytes per row

    def call(rows=10, n_gt=4, V=3, K=5, top_k=3, score=one, ap=one, ws_bytes=ws):
        return lib.ssnb_classification_ap(one, one, score, rows, one, one, n_gt, V, K, top_k, ap, one, one, None, None, None, one,
                                          ws_bytes, None)
    for kw, why in ((dict(V=0), "no video"), (dict(K=0), "no class"), (dict(K=1025), "1025 classes"), (dict(rows=-1), "negative rows"),
                    (dict(rows=1 << 31), "rows past INT_MAX"), (dict(n_gt=-1), "negative n_gt"),
                    (dict(V=1 << 21, K=1024), "num_class * n_videos past INT_MAX")):
        assert call(**kw) == 1, why
        assert lib.ssnb_classification_ap_workspace_bytes(kw.get("rows", 10), kw.get("n_gt", 4), kw.get("V", 3), kw.get("K", 5)) == 0, why
    assert call(top_k=0) == 1
    assert call(score=None) == 1 and call(ap=None) == 1
    assert call(ws_bytes=ws - 1) == 1
    assert b"classification_ap" in lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0


def test_cpu_tensors_are_refused():
    import torch
    from ops import classification_eval as E
    with pytest.raises(RuntimeError):
        E.classification_ap_packed([0], [0], torch.zeros(1, dtype=torch.float64), [0], [0], 1, 1)
    with pytest.raises(RuntimeError):
        E.classification_ap_dense(torch.zeros(2, 3), [0], [0])
    with pytest.raises(RuntimeError):
        E.evaluate_classification({}, {}, device="cpu")
