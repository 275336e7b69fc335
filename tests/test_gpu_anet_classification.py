"""ActivityNet untrimmed video classification on the GPU (ops/classification_eval.py, csrc/classification_ap.cu) against the
real toolkit's results (tests/golden/anet_classification.npz) and against oracle/anet_classification_oracle.py on seeded
random ragged sets with ties, NaN scores, repeated rows and rows outside the videos / classes, and on a dense ActivityNet-sized
score matrix: AP within 1e-12 (the bar of test_gpu_eval.py), hit counts and true positives exact.  One call against per-class
calls, a repeat and a CUDA-graph replay bitwise, the refusals.  Nothing here reads a checkout of the reference."""
import json

import numpy as np
import pytest
import torch

from oracle import anet_classification_oracle as O
from test_anet_classification_host import FIXTURES, GOLD, fixture, oracle
from test_proplist_host import same

pytestmark = pytest.mark.gpu

AP_TOL = 1e-12


def dev():
    return torch.device("cuda:0")


def T(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(dev())


def run(f, trace=True):
    from ops import classification_eval as E
    return E.classification_ap_packed(T(f["video"], torch.int32), T(f["label"], torch.int32), T(f["score"], torch.float64),
                                      T(f["gt_video"], torch.int32), T(f["gt_label"], torch.int32), f["V"], f["K"], f["top_k"], trace=trace)


def check_against(r, o):
    ap = r["ap"].cpu().numpy()
    assert ap.shape == o["ap"].shape and np.array_equal(np.isnan(ap), np.isnan(o["ap"]))
    assert np.nanmax(np.abs(ap - o["ap"]), initial=0.0) <= AP_TOL
    assert float(r["hit_at_k"]) == o["hit_at_k"] or (np.isnan(o["hit_at_k"]) and np.isnan(float(r["hit_at_k"])))
    assert abs(float(r["avg_hit_at_k"]) - o["avg_hit_at_k"]) <= 1e-12 or np.isnan(o["avg_hit_at_k"])
    for k in ("hits", "gt_labels", "tp"):
        assert same(r[k].cpu().numpy(), o[k]), k


@pytest.mark.parametrize("name", FIXTURES)
def test_golden_fixture(name):
    f = fixture(name)
    r = run(f)
    check_against(r, oracle(f))
    ap = r["ap"].cpu().numpy()
    assert np.abs(ap - GOLD[name + "_ap"]).max() <= AP_TOL
    assert abs(float(ap.mean()) - float(GOLD[name + "_map"])) <= AP_TOL
    assert float(r["hit_at_k"]) == float(GOLD[name + "_hit_at_k"])
    assert abs(float(r["avg_hit_at_k"]) - float(GOLD[name + "_avg_hit_at_k"])) <= 1e-12


def test_evaluate_classification_from_json():
    from ops import classification_eval as E
    gt_j, pr_j = json.loads(str(GOLD["json_gt_text"])), json.loads(str(GOLD["json_pr_text"]))
    for k in (1, 3, 5):
        rep = E.evaluate_classification(gt_j, pr_j, top_k=k, blocked_videos=[str(x) for x in GOLD["json_blocked"]])
        f = fixture("json") | {"top_k": k}
        o = oracle(f)
        assert np.abs(rep["ap"] - o["ap"]).max() <= AP_TOL and abs(rep["map"] - float(o["ap"].mean())) <= AP_TOL
        assert rep["hit_at_k"] == o["hit_at_k"] and rep["error_at_k"] == 1.0 - o["hit_at_k"] and rep["top_k"] == k
        assert abs(rep["avg_hit_at_k"] - o["avg_hit_at_k"]) <= 1e-12
        if k == 3:
            assert rep["hit_at_k"] == float(GOLD["json_hit_at_k"]) and abs(rep["map"] - float(GOLD["json_map"])) <= AP_TOL
    with pytest.raises(ValueError):
        E.evaluate_classification(gt_j, pr_j, subset="no such subset")


def random_set(seed, V=2500, K=150):
    """ragged: 0..60 rows per video, 0..4 ground-truth labels (repeats among them); scores continuous in some videos and drawn
    from a small set with NaN and -0 in others (ties at every size); repeated (video, label) rows"""
    g = np.random.RandomState(seed)
    video, label, score, gv, gl = [], [], [], [], []
    pool = np.array([np.nan, 0.5, 0.5, 0.25, -0.0, 0.0, 1.0, 0.75])
    for v in range(V):
        ng = int(g.choice([0, 1, 2, 4], p=[0.1, 0.6, 0.2, 0.1]))
        labs = g.randint(0, K, ng)
        gv += [v] * ng
        gl += labs.tolist()
        n = int(g.choice([0, g.randint(1, 6), g.randint(6, 61)], p=[0.08, 0.5, 0.42]))
        lab = np.where(g.rand(n) < 0.3, g.choice(labs, n) if ng else g.randint(0, K, n), g.randint(0, K, n))
        s = pool[g.randint(0, len(pool), n)] if v % 3 == 0 else g.rand(n)
        video += [v] * n
        label += lab.tolist()
        score += s.tolist()
    perm = g.permutation(len(video))                         # rows of a video are not contiguous
    return dict(video=np.array(video, np.int32)[perm], label=np.array(label, np.int32)[perm], score=np.array(score)[perm],
                gt_video=np.array(gv, np.int32), gt_label=np.array(gl, np.int32), V=V, K=K)


@pytest.mark.parametrize("seed,top_k", [(1, 1), (2, 3), (3, 5), (4, 100)])
def test_random_ragged_against_oracle(seed, top_k):
    f = random_set(seed) | {"top_k": top_k}
    assert len(np.unique(f["label"].astype(np.int64) * f["V"] + f["video"])) < len(f["video"])
    check_against(run(f), oracle(f))


def test_rows_outside_the_videos_and_classes_are_ignored():
    f = random_set(5, V=400, K=30) | {"top_k": 3}
    g = np.random.RandomState(6)
    n_bad = 80
    bad_v = np.where(np.arange(n_bad) % 2, g.choice([-1, f["V"], 1 << 30], n_bad), g.randint(0, f["V"], n_bad))
    bad_c = np.where(np.arange(n_bad) % 2, g.randint(0, f["K"], n_bad), g.choice([-1, f["K"]], n_bad))
    n = len(f["video"]) + n_bad
    perm = g.permutation(n)
    full = f | {"video": np.concatenate([f["video"], bad_v]).astype(np.int32)[perm],
                "label": np.concatenate([f["label"], bad_c]).astype(np.int32)[perm],
                "score": np.concatenate([f["score"], g.rand(n_bad)])[perm],
                "gt_video": np.concatenate([f["gt_video"], [-1, f["V"], 3]]).astype(np.int32),
                "gt_label": np.concatenate([f["gt_label"], [0, 0, f["K"]]]).astype(np.int32)}
    keep = (full["video"] >= 0) & (full["video"] < f["V"]) & (full["label"] >= 0) & (full["label"] < f["K"])
    assert (~keep).sum() == n_bad
    o = oracle(f | {k: full[k][keep] for k in ("video", "label", "score")})
    tp = np.zeros(n, np.uint8)
    tp[keep] = o["tp"]
    check_against(run(full), o | {"tp": tp})


def test_dense_matrix_activitynet_size():
    """4926 videos x 200 classes, every class of every video a prediction (cls_scores), one or two labels per video"""
    from ops import classification_eval as E
    g = np.random.RandomState(11)
    V, K = 4926, 200
    S = g.rand(V, K)
    S[g.rand(V, K) < 0.02] = 0.5                                                # ties inside classes and videos
    gv = np.concatenate([np.arange(V), g.choice(V, 300)]).astype(np.int32)
    gl = g.randint(0, K, len(gv)).astype(np.int32)
    vid, lab = np.repeat(np.arange(V, dtype=np.int32), K), np.tile(np.arange(K, dtype=np.int32), V)
    for k in (1, 3):
        r = E.classification_ap_dense(T(S), gv, gl, top_k=k, trace=True)
        check_against(r, O.classification(vid, lab, S.reshape(-1), gv, gl, V, K, k))


def test_one_call_equals_per_class_calls():
    f = random_set(7, V=800, K=40) | {"top_k": 3}
    whole = run(f)["ap"].cpu().numpy()
    for c in (0, 3, 17, 39):
        m, gm = f["label"] == c, f["gt_label"] == c
        one = run(f | {"video": f["video"][m], "label": f["label"][m], "score": f["score"][m], "gt_video": f["gt_video"][gm],
                       "gt_label": f["gt_label"][gm]})["ap"].cpu().numpy()
        assert one[c].tobytes() == whole[c].tobytes(), c


def test_repeat_and_graph_replay_bitwise():
    from ops import classification_eval as E
    f = random_set(8, V=1500, K=100) | {"top_k": 3}
    args = [T(f[k], torch.int32) for k in ("video", "label")] + [T(f["score"], torch.float64)] + \
           [T(f[k], torch.int32) for k in ("gt_video", "gt_label")]
    a = E.classification_ap_packed(*args, f["V"], f["K"], 3, trace=True)
    b = E.classification_ap_packed(*args, f["V"], f["K"], 3, trace=True)
    for k in ("ap", "hit_at_k", "avg_hit_at_k", "hits", "gt_labels", "tp"):
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.classification_ap_packed(*args, f["V"], f["K"], 3)                  # warm-up off the capture
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        c = E.classification_ap_packed(*args, f["V"], f["K"], 3, trace=True)
    gr.replay()
    torch.cuda.synchronize()
    for k in ("ap", "hit_at_k", "avg_hit_at_k", "hits", "gt_labels", "tp"):
        assert c[k].cpu().numpy().tobytes() == a[k].cpu().numpy().tobytes(), k
    # new scores written in place: the replay follows them
    new = np.random.RandomState(10).rand(len(f["score"]))
    args[2].copy_(T(new))
    gr.replay()
    torch.cuda.synchronize()
    check_against(c, oracle(f | {"score": new}))


def test_bad_arguments_are_refused_without_a_launch():
    from ops import classification_eval as E
    from ssn_b200._lib import lib
    f = random_set(12, V=50, K=8)
    args = [f["video"], f["label"], T(f["score"]), f["gt_video"], f["gt_label"]]
    torch.cuda.synchronize()
    n0 = lib.ssnb_global_launch_count()
    for V, K, k in ((0, 8, 3), (50, 0, 3), (50, 1025, 3), (50, 8, 0)):
        with pytest.raises(RuntimeError, match="classification_ap"):
            E.classification_ap_packed(*args, V, K, k)
    with pytest.raises(ValueError):
        E.classification_ap_packed(f["video"][:-1], *args[1:], 50, 8)
    assert lib.ssnb_global_launch_count() == n0
