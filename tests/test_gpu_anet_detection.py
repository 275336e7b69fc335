"""ActivityNet detection evaluation of results files on the GPU (ops/detection_eval.py, csrc/detection_ap.cu
ssnb_detection_ap_rows) against the real toolkit's results (tests/golden/anet_detection.npz) and against
oracle/anet_detection_oracle.py on seeded random ragged sets with quantised and NaN scores, grid segments (equal tIoU) and rows
outside the videos / classes: AP within 1e-12 (the bar of test_gpu_eval.py), ranks and tp flags exact.  One call against
per-class calls, a repeat, a CUDA-graph replay on new scores and a 0xFF-filled workspace bitwise, and the row path against the
slot path (ssnb_detection_ap) on the same survivors, bitwise.  Nothing here reads a checkout of the reference."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from test_anet_detection_host import FIXTURES, GOLD, THR, fixture, oracle

pytestmark = pytest.mark.gpu

AP_TOL = 1e-12


def dev():
    return torch.device("cuda:0")


def T(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(dev())


def args(f):
    return (T(f["video"], torch.int32), T(f["label"], torch.int32), T(f["seg"], torch.float64), T(f["score"], torch.float64),
            T(f["gt_offsets"], torch.int64), T(f["gt_cls"], torch.int32), T(f["gt_seg"], torch.float64), f["K"])


def run(f, thr=THR, trace=True):
    from ops import detection_eval as E
    return E.detection_ap_rows(*args(f), thr, trace=trace)


def check_against(r, o):
    ap = r["ap"].cpu().numpy()
    assert ap.shape == o["ap"].shape and np.array_equal(np.isnan(ap), np.isnan(o["ap"]))
    assert np.nanmax(np.abs(ap - o["ap"]), initial=0.0) <= AP_TOL
    assert np.array_equal(r["rank"].cpu().numpy(), o["rank"])
    assert np.array_equal(r["tp"].cpu().numpy(), o["tp"])


@pytest.mark.parametrize("name", FIXTURES)
def test_golden_fixture(name):
    f = fixture(name)
    r = run(f)
    check_against(r, oracle(f))
    ap = r["ap"].cpu().numpy().T                                   # the toolkit's [n_thr, K]
    assert np.abs(ap - GOLD[name + "_ap"]).max() <= AP_TOL
    assert np.abs(ap.mean(axis=1) - GOLD[name + "_map"]).max() <= AP_TOL
    assert abs(float(ap.mean(axis=1).mean()) - float(GOLD[name + "_average_map"])) <= AP_TOL


@pytest.mark.parametrize("name", ["anet", "edges"])
def test_evaluate_anet_detection_from_json(name):
    from ops import detection_eval as E
    gt_j, pr_j = json.loads(str(GOLD[name + "_gt_text"])), json.loads(str(GOLD[name + "_pr_text"]))
    rep = E.evaluate_anet_detection(gt_j, pr_j, blocked_videos=[str(x) for x in GOLD[name + "_blocked"]])
    assert rep["ap"].shape == GOLD[name + "_ap"].shape and np.abs(rep["ap"] - GOLD[name + "_ap"]).max() <= AP_TOL
    assert np.abs(rep["map"] - GOLD[name + "_map"]).max() <= AP_TOL
    assert abs(rep["average_map"] - float(GOLD[name + "_average_map"])) <= AP_TOL
    assert rep["lines"][-1] == "\tAverage-mAP: {}".format(rep["map"].mean()) and list(rep["activity_index"].values())[:2] == [0, 1]
    with pytest.raises(ValueError):
        E.evaluate_anet_detection(gt_j, pr_j, subset="no such subset")


def random_set(seed, V=2000, K=200, big=0.02, bad=0):
    """ragged: 0..40 rows per video, a share `big` of the videos with 300..1000; 0..4 instances per video; scores continuous in
    some videos and quantised (with NaN and -0) in others; segments near an instance or random, on a coarse grid in some videos
    (equal tIoU to two instances); `bad` rows outside the videos or classes"""
    g = np.random.RandomState(seed)
    pool = np.array([np.nan, 0.5, 0.5, 0.25, -0.0, 0.0, 1.0, 0.75, 0.125])
    off, gc, gs, video, label, seg, score = [0], [], [], [], [], [], []
    for v in range(V):
        grid = v % 4 == 1
        ng = int(g.choice([0, 1, 2, 4], p=[0.1, 0.5, 0.25, 0.15]))
        for _ in range(ng):
            a, b = np.sort(g.randint(0, 20, 2) * 10.0) if grid else np.sort(g.rand(2) * 100)
            gc.append(int(g.randint(K)) if g.rand() < 0.5 or not gc else gc[-1])
            gs.append((a, b))
        off.append(len(gc))
        n = int(g.randint(300, 1001)) if g.rand() < big else int(g.choice([0, g.randint(1, 8), g.randint(8, 41)], p=[0.1, 0.5, 0.4]))
        for _ in range(n):
            if ng and g.rand() < 0.5:
                k = off[-2] + g.randint(ng)
                c, (a, b) = gc[k], gs[k]
                j = (b - a) * 0.3 * (g.rand(2) * 2 - 1)
                a, b = (round(a + j[0], -1), round(b + j[1], -1)) if grid else (a + j[0], b + j[1])
            else:
                c = int(g.randint(K))
                a, b = np.sort(g.randint(0, 20, 2) * 10.0) if grid else np.sort(g.rand(2) * 100)
            video.append(v)
            label.append(c)
            seg.append((a, b))
        s = pool[g.randint(0, len(pool), n)] if v % 3 == 0 else g.rand(n)
        score += s.tolist()
    video, label = np.array(video, np.int32), np.array(label, np.int32)
    if bad:
        at = g.choice(len(video), bad, replace=False)
        video[at[::2]] = g.choice([-1, V, 1 << 30], len(at[::2]))
        label[at[1::2]] = g.choice([-1, K], len(at[1::2]))
    perm = g.permutation(len(video))                               # rows of a video are not contiguous
    return dict(video=video[perm], label=label[perm], seg=np.array(seg, np.float64).reshape(-1, 2)[perm], score=np.array(score)[perm],
                gt_offsets=np.array(off, np.int64), gt_cls=np.array(gc, np.int32), gt_seg=np.array(gs, np.float64).reshape(-1, 2), K=K)


@pytest.mark.parametrize("seed,V,K,big,bad", [(1, 2000, 200, 0.02, 0), (2, 3000, 200, 0.0, 500), (3, 400, 20, 0.05, 40)])
def test_random_ragged_against_oracle(seed, V, K, big, bad):
    f = random_set(seed, V, K, big, bad)
    per_video = np.bincount(f["video"][(f["video"] >= 0) & (f["video"] < V)], minlength=V)
    assert per_video.max() >= (300 if big else 1) and np.isnan(f["score"]).any()
    check_against(run(f), oracle(f))


def test_one_call_equals_per_class_calls():
    f = random_set(5, V=600, K=40, big=0.02)
    whole = run(f, trace=False)["ap"].cpu().numpy()
    for c in (0, 3, 17, 39):
        m = f["label"] == c
        one = run(f | {"video": f["video"][m], "label": f["label"][m], "seg": f["seg"][m], "score": f["score"][m]}, trace=False)
        assert one["ap"].cpu().numpy()[c].tobytes() == whole[c].tobytes(), c


def test_repeat_graph_replay_and_filled_workspace_bitwise():
    from ops import detection_eval as E
    from ssn_b200._lib import lib, check
    f = random_set(8, V=1500, K=200, big=0.01)
    a = E.detection_ap_rows(*args(f), THR, trace=True)
    b = E.detection_ap_rows(*args(f), THR, trace=True)
    for k in ("ap", "rank", "tp"):
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
    # a workspace and outputs filled with 0xFF
    v, l, sg, sc, go, gcl, gsg, K = args(f)
    rows, n_gt = sc.numel(), gcl.numel()
    wsb = lib.ssnb_detection_ap_rows_workspace_bytes(rows, go.numel() - 1, K, n_gt, len(THR))
    ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device=dev())
    ap = torch.full((K, len(THR)), float("nan"), dtype=torch.float64, device=dev())
    rank = torch.full((rows,), -1, dtype=torch.int32, device=dev())
    tp = torch.zeros(len(THR), rows, dtype=torch.uint8, device=dev())
    with torch.cuda.device(dev()):
        check(lib.ssnb_detection_ap_rows(v.data_ptr(), l.data_ptr(), sg.data_ptr(), sc.data_ptr(), rows, go.numel() - 1, K, go.data_ptr(),
                                         gcl.data_ptr(), gsg.data_ptr(), n_gt, (C.c_double * len(THR))(*THR), len(THR), ap.data_ptr(),
                                         rank.data_ptr(), tp.data_ptr(), ws.data_ptr(), wsb, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert ap.cpu().numpy().tobytes() == a["ap"].cpu().numpy().tobytes()
    assert torch.equal(rank, a["rank"]) and torch.equal(tp, a["tp"])
    # CUDA graph: capture once, replay on new scores written in place
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.detection_ap_rows(v, l, sg, sc, go, gcl, gsg, K, THR)                # warm-up off the capture
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        c = E.detection_ap_rows(v, l, sg, sc, go, gcl, gsg, K, THR, trace=True)
    gr.replay()
    torch.cuda.synchronize()
    for k in ("ap", "rank", "tp"):
        assert c[k].cpu().numpy().tobytes() == a[k].cpu().numpy().tobytes(), k
    new = np.round(np.random.RandomState(10).rand(rows) * 50) / 50          # quantised: ties
    sc.copy_(T(new))
    gr.replay()
    torch.cuda.synchronize()
    e = E.detection_ap_rows(v, l, sg, sc, go, gcl, gsg, K, THR, trace=True)
    for k in ("ap", "rank", "tp"):
        assert c[k].cpu().numpy().tobytes() == e[k].cpu().numpy().tobytes(), k
    check_against(c, oracle(f | {"score": new}))


def test_rows_of_survivors_equal_the_slot_path_bitwise():
    """detections_packed survivors written as rows in (video, class, kept position) order, fp32 widened to double: the row
    path's AP, ranks and tp flags equal the slot path's (detection_ap) on the same survivors, bitwise"""
    from ops.detection import detections_packed, detection_ap
    from ops import detection_eval as E
    from test_gpu_eval import synth_set
    for kind, seed, top_k, nms in (("anet", 51, 60, 0.6), ("ties", 52, 30, 0.4), ("thumos", 53, 300, 0.2)):
        props, act, comp, reg, offsets, K, gt = synth_set(kind, seed, V=300 if kind != "ties" else None)
        Tt = lambda x: torch.tensor(x, device=dev())                       # noqa: E731
        d = detections_packed(Tt(props), Tt(act), Tt(comp), Tt(reg), offsets, nms, mode="top_k", top_k=top_k)
        thr = np.linspace(0.1, 0.9, 9)
        slot = detection_ap(d, gt, thr, trace=True)
        counts = d["counts"].cpu().numpy()
        V, S = counts.shape[0], int(d["slot0"][-1])
        video, label = np.zeros(S, np.int32), np.zeros(S, np.int32)
        used = np.zeros(S, bool)
        for v in range(V):
            at = d["slot0"][v]
            for c in range(K):
                video[at:at + counts[v, c]], label[at:at + counts[v, c]] = v, c
                used[at:at + counts[v, c]] = True
                at += counts[v, c]
        idx = np.nonzero(used)[0]
        dets = d["dets"][:S][torch.as_tensor(idx, device=dev())].double()
        goff = torch.tensor(gt["offsets"], dtype=torch.int64, device=dev())
        rows = E.detection_ap_rows(video[idx], label[idx], dets[:, :2].contiguous(), dets[:, 2].contiguous(), goff, gt["cls"], gt["seg"],
                                   K, thr, trace=True)
        assert len(idx) > 100
        assert rows["ap"].cpu().numpy().tobytes() == slot["ap"].cpu().numpy().tobytes(), kind
        assert np.array_equal(rows["rank"].cpu().numpy(), slot["rank"].cpu().numpy()[idx]), kind
        assert np.array_equal(rows["tp"].cpu().numpy(), slot["tp"].cpu().numpy()[:, idx]), kind


def test_bad_arguments_are_refused_without_a_launch():
    from ops import detection_eval as E
    from ssn_b200._lib import lib
    f = random_set(12, V=50, K=8)
    v, l, sg, sc, go, gcl, gsg, K = args(f)
    torch.cuda.synchronize()
    n0 = lib.ssnb_global_launch_count()
    for kk, thr in ((0, THR), (-1, THR), (1025, THR), (8, []), (8, [0.5, float("nan")]), (8, np.linspace(0.1, 0.9, 65))):
        with pytest.raises(RuntimeError, match="detection_ap_rows"):
            E.detection_ap_rows(v, l, sg, sc, go, gcl, gsg, kk, thr)
    with pytest.raises(ValueError):
        E.detection_ap_rows(v[:-1], l, sg, sc, go, gcl, gsg, K, THR)
    assert lib.ssnb_global_launch_count() == n0
