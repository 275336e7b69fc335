"""The detection oracle (oracle/anet_detection_oracle.py) against tests/golden/anet_detection.npz, which holds what the real
ActivityNet toolkit's ANETdetection computed (oracle/gen_golden_anet_detection.py); the JSON loaders of ops/detection_eval.py
against the toolkit's data frames and its errors; the library's argument checks and the header's declarations.  No GPU."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from oracle import anet_detection_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "anet_detection.npz"))
FIXTURES = [str(x) for x in GOLD["fixtures"]]
THR = GOLD["tiou_thresholds"]


def fixture(name):
    """-> dict(video, label, seg, score, gt_offsets (padded to the prediction's videos), gt_cls, gt_seg, K, video_ids,
    activity_index) from the fixture's JSON texts through the loaders"""
    from ops import detection_eval as E
    blocked = [str(x) for x in GOLD[name + "_blocked"]]
    gt = E.load_anet_detection_ground_truth(json.loads(str(GOLD[name + "_gt_text"])), "validation", blocked)
    pr = E.load_anet_detection_predictions(json.loads(str(GOLD[name + "_pr_text"])), gt, blocked)
    V = len(pr["video_ids"])
    off = np.concatenate([gt["offsets"], np.full(V + 1 - len(gt["offsets"]), gt["offsets"][-1])])
    return dict(video=pr["video"], label=pr["label"], seg=pr["seg"], score=pr["score"], gt_offsets=off, gt_cls=gt["cls"],
                gt_seg=gt["seg"], K=len(gt["activity_index"]), video_ids=pr["video_ids"], activity_index=gt["activity_index"])


def oracle(f, thr=THR):
    return O.detection(f["video"], f["label"], f["seg"], f["score"], f["gt_offsets"], f["gt_cls"], f["gt_seg"], f["K"], thr)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_toolkit(name):
    o = oracle(fixture(name))
    ap = GOLD[name + "_ap"]
    assert ap.shape == (len(THR), o["ap"].shape[0])
    assert np.abs(o["ap"].T - ap).max() <= 1e-12
    assert np.abs(o["ap"].T.mean(axis=1) - GOLD[name + "_map"]).max() <= 1e-12
    assert abs(float(o["ap"].T.mean(axis=1).mean()) - float(GOLD[name + "_average_map"])) <= 1e-12


def test_fixtures_cover_the_edges():
    assert THR.tobytes() == np.linspace(0.5, 0.95, 10).tobytes() and (THR != np.round(THR, 2)).any()   # not the decimals
    f = fixture("ties")
    s = f["score"]
    assert np.isnan(s).sum() > 1 and (s == 0).sum() > 1 and np.signbit(s[s == 0]).any()
    assert len(np.unique(s[~np.isnan(s)])) + int(np.isnan(s).sum()) < len(s)                   # ties
    assert np.bincount(f["label"]).max() <= 16
    assert (f["seg"][:, 1] < f["seg"][:, 0]).any() and (f["seg"][:, 1] == f["seg"][:, 0]).any()  # reversed, zero length
    assert (f["gt_seg"][:, 1] == f["gt_seg"][:, 0]).any()
    f = fixture("edges")
    V_gt = int(np.searchsorted(f["gt_offsets"], f["gt_offsets"][-1]))
    assert (f["video"] >= V_gt).any()                                                           # videos without ground truth
    assert set(range(V_gt)) - set(f["video"].tolist())                                          # ground-truth videos, no rows
    assert set(range(f["K"])) - set(f["label"].tolist())                                        # a class without predictions
    missing = sorted(set(range(f["K"])) - set(f["label"].tolist()))
    assert GOLD["edges_ap"][:, missing].max() == 0.0
    assert len(GOLD["edges_blocked"]) == 2
    f = fixture("long")
    assert np.bincount(f["label"] * len(f["video_ids"]) + f["video"]).max() > 256
    assert fixture("k200")["K"] == 200 and len(fixture("anet")["video_ids"]) >= 300


def test_loaders_against_the_toolkit_frames():
    from ops import detection_eval as E
    gt_j, pr_j = json.loads(str(GOLD["edges_gt_text"])), json.loads(str(GOLD["edges_pr_text"]))
    blocked = [str(x) for x in GOLD["edges_blocked"]]
    gt = E.load_anet_detection_ground_truth(gt_j, "validation", blocked)
    assert list(gt["activity_index"]) == GOLD["frame_classes"].tolist()
    assert list(gt["activity_index"].values()) == list(range(len(gt["activity_index"])))
    vid_of_row = np.repeat(np.arange(len(gt["video_ids"])), np.diff(gt["offsets"]))
    assert [gt["video_ids"][i] for i in vid_of_row] == GOLD["frame_gt_video"].tolist()
    assert np.array_equal(gt["cls"].astype(np.int64), GOLD["frame_gt_label"])
    assert gt["seg"].tobytes() == GOLD["frame_gt_seg"].tobytes()
    pr = E.load_anet_detection_predictions(pr_j, gt, blocked)
    assert pr["video_ids"][:len(gt["video_ids"])] == gt["video_ids"]
    assert [pr["video_ids"][i] for i in pr["video"]] == GOLD["frame_pr_video"].tolist()
    assert np.array_equal(pr["label"].astype(np.int64), GOLD["frame_pr_label"])
    assert pr["seg"].tobytes() == GOLD["frame_pr_seg"].tobytes() and pr["score"].tobytes() == GOLD["frame_pr_score"].tobytes()
    assert blocked[0] not in gt["video_ids"] and blocked[1] not in pr["video_ids"] and len(pr["video_ids"]) > len(gt["video_ids"])
    assert "e_noann" not in gt["video_ids"] and "e_noann" in pr["video_ids"] and "e_07" not in gt["video_ids"]


def test_loader_errors():
    from ops import detection_eval as E
    with pytest.raises(IOError, match="valid ground truth"):
        E.load_anet_detection_ground_truth({"database": {}, "version": ""})
    gt = E.load_anet_detection_ground_truth({"database": {"a": {"subset": "validation", "annotations": [{"label": "x", "segment": [1, 2]}]}},
                                             "taxonomy": [], "version": ""})
    assert gt["offsets"].tolist() == [0, 1] and gt["seg"].tolist() == [[1.0, 2.0]] and gt["activity_index"] == {"x": 0}
    with pytest.raises(IOError, match="valid prediction"):
        E.load_anet_detection_predictions({"results": {}, "version": ""}, gt)
    with pytest.raises(ValueError, match=r"'y' of video 'a'"):
        E.load_anet_detection_predictions({"results": {"a": [{"label": "y", "score": 1, "segment": [0, 1]}]}, "version": "",
                                           "external_data": {}}, gt)
    # a blocked video's unknown label is never looked up, as in the toolkit
    pr = E.load_anet_detection_predictions({"results": {"b": [{"label": "y", "score": 1, "segment": [0, 1]}],
                                                        "a": [{"label": "x", "score": 0.5, "segment": [0, 1]}]},
                                            "version": "", "external_data": {}}, gt, blocked_videos=["b"])
    assert pr["video"].tolist() == [0] and pr["label"].tolist() == [0] and pr["video_ids"] == ["a"]


def test_oracle_rules():
    """hand-worked: equal scores rank the later row first, NaN first; equal tIoU locks the larger instance first; a row of a
    video without ground truth is a false positive; a zero-length row on a zero-length instance matches (NaN tIoU)"""
    gt_offsets, gt_cls = [0, 3, 3], [0, 0, 0]
    gt_seg = [[0.0, 12.0], [8.0, 20.0], [40.0, 40.0]]
    video, label = [0, 0, 1, 0, 0], [0, 0, 0, 0, 0]
    seg = [[2.0, 18.0], [2.0, 18.0], [0.0, 12.0], [40.0, 40.0], [0.0, 1.0]]
    score = [0.5, 0.5, 0.9, np.nan, 0.5]
    o = O.detection(video, label, seg, score, gt_offsets, gt_cls, gt_seg, 1, [0.5])
    # rank: NaN row 3 first, then 0.9 (row 2), then the 0.5 rows in descending row order 4, 1, 0
    assert o["rank"].tolist() == [4, 3, 1, 0, 2]
    assert o["tp"][0].tolist() == [1, 1, 0, 1, 0]                   # row 1 locks instance 1 (larger index), row 0 instance 0
    assert abs(o["ap"][0, 0] - (1 / 3 * 1.0 + 1 / 3 * 0.6 + 1 / 3 * 0.6)) <= 1e-15


def test_rejected_arguments_return_before_any_launch():
    """argument validation needs no device: the library returns SSNB_EINVAL (1), launches nothing, and the workspace query
    returns 0 for exactly those arguments"""
    from ssn_b200 import _lib
    lib = _lib.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(8)                                   # a non-null pointer that is never dereferenced
    thr = (C.c_double * 2)(0.5, 0.75)
    ws = lib.ssnb_detection_ap_rows_workspace_bytes(10, 3, 5, 4, 2)
    # about 40 B per row and 1 B per row and threshold
    assert ws > 0 and lib.ssnb_detection_ap_rows_workspace_bytes(1010, 3, 5, 4, 2) > ws + 1000 * 40

    def call(rows=10, V=3, K=5, n_gt=4, n_thr=2, score=one, ap=one, th=thr, ws_bytes=ws):
        return lib.ssnb_detection_ap_rows(one, one, one, score, rows, V, K, one, one, one, n_gt, th, n_thr, ap, None, None, one,
                                          ws_bytes, None)
    for kw, why in ((dict(V=0), "no video"), (dict(K=0), "no class"), (dict(K=-3), "negative K"), (dict(K=1025), "1025 classes"),
                    (dict(rows=-1), "negative rows"), (dict(rows=1 << 31), "rows past INT_MAX"), (dict(n_gt=-1), "negative n_gt"),
                    (dict(n_gt=1 << 31), "n_gt past INT_MAX"), (dict(n_thr=0), "no threshold"), (dict(n_thr=65), "65 thresholds"),
                    (dict(V=1 << 21, K=1024), "num_class * n_videos past INT_MAX")):
        assert call(**kw) == 1, why
        assert lib.ssnb_detection_ap_rows_workspace_bytes(kw.get("rows", 10), kw.get("V", 3), kw.get("K", 5), kw.get("n_gt", 4),
                                                          kw.get("n_thr", 2)) == 0, why
    assert call(score=None) == 1 and call(ap=None) == 1 and call(th=None) == 1
    assert call(th=(C.c_double * 2)(0.5, float("nan"))) == 1
    assert call(ws_bytes=ws - 1) == 1
    assert b"detection_ap_rows" in lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0


def test_header_declares_the_bound_signatures():
    from ssn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    for name, ret, n_args in (("ssnb_detection_ap_rows", "int", 19), ("ssnb_detection_ap_rows_workspace_bytes", "size_t", 5)):
        decl = re.search(r"%s %s\(([^)]*)\);" % (ret, name), hdr).group(1)
        assert len(decl.split(",")) == n_args == len(_lib.SIGNATURES[name][1]), name
    decl = re.search(r"size_t ssnb_detection_ap_rows_workspace_bytes\(([^)]*)\);", hdr).group(1)
    assert [a.split()[0] for a in decl.split(",")] == ["int64_t", "int", "int", "int64_t", "int"]
    assert _lib.SIGNATURES["ssnb_detection_ap_rows_workspace_bytes"][1] == [C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int]
    decl = re.search(r"int ssnb_detection_ap_rows\(([^)]*)\);", hdr).group(1)
    kinds = [a.strip().rsplit(" ", 1)[0] for a in decl.split(",")]
    want = {"int64_t": C.c_int64, "int": C.c_int, "size_t": C.c_size_t}
    for k, t in zip(kinds, _lib.SIGNATURES["ssnb_detection_ap_rows"][1]):
        if "*" in k:
            assert t in (C.c_void_p, C.POINTER(C.c_double)), k
        else:
            assert t == want[k], k


def test_cpu_tensors_are_refused():
    import torch
    from ops import detection_eval as E
    with pytest.raises(RuntimeError):
        E.detection_ap_rows([0], [0], [[0.0, 1.0]], torch.zeros(1, dtype=torch.float64), [0, 1], [0], [[0.0, 1.0]], 1)
    with pytest.raises(RuntimeError):
        E.evaluate_anet_detection({}, {}, device="cpu")
