"""Detection evaluation on the GPU (ops/detection.py: detections_packed / detection_ap / evaluate_detections; csrc/detect.cu
ssnb_detect_batch, csrc/detection_ap.cu ssnb_detection_ap):
  - against tests/golden/eval.npz (the real reference's functions and the toolkit's AP): survivors, order and counts
    exact, boxes within the regression bar, AP within 1e-12;
  - stage by stage (oracle/eval_check.py) on seeded THUMOS14-like and ActivityNet1.2-like sets in one call each;
  - ties, NaN / inf logits, identical and zero-length boxes under the documented rule;
  - call properties: one call equals one call per video, repeats and CUDA-graph replays are bitwise, output memory
    pre-filled with 0xFF changes nothing, rejected arguments return before any launch."""
import ctypes as C
import os
import time

import numpy as np
import pytest
import torch

from oracle import eval_check as E
from oracle import gen_golden_eval as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda:0")


# ---- golden ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fx", G.FIXTURES, ids=[f[0] for f in G.FIXTURES])
def test_against_reference_golden(fx):
    from ops.detection import evaluate_detections, detections_packed
    from test_eval_host import fixture_inputs, GOLD
    name, K, V, _, mode, top_k, cls_top_k, sbf, nms, thr_kind, n_src, weights, regress, _ = fx
    srcs, merged, cls_scores, gt = fixture_inputs(fx)
    r = evaluate_detections(srcs, gt, weights=list(weights) if weights else None, nms_threshold=nms, top_k=top_k if mode == "top_k" else 0,
                            cls_scores=cls_scores if mode == "cls" else None, cls_top_k=cls_top_k, softmax_before_filter=sbf,
                            regress=regress, iou_range=G.thresholds(thr_kind))
    ref = GOLD[name + "_ap"]
    assert np.array_equal(np.isnan(r["ap"]), np.isnan(ref))
    assert np.nanmax(np.abs(r["ap"] - ref)) <= 1e-12
    assert np.allclose(r["map"], ref.mean(0), equal_nan=True, rtol=0, atol=1e-12)
    # the survivors themselves, through the packed call on the merged scores
    vids = list(merged)
    rel = [np.squeeze(merged[v][0], 0) if merged[v][0].ndim == 3 else merged[v][0] for v in vids]
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in rel])]).tolist()
    t = lambda xs: torch.tensor(np.concatenate(xs), device=dev())
    reg = None if merged[vids[0]][3] is None else t([merged[v][3].reshape(-1, K, 2) for v in vids])
    by_name = {os.path.splitext(os.path.basename(k))[0]: v for k, v in cls_scores.items()}
    sel = np.stack([np.argsort(by_name[v], kind="stable")[-cls_top_k:] for v in vids]) if mode == "cls" else None
    d = detections_packed(t(rel), t([merged[v][1] for v in vids]), t([merged[v][2] for v in vids]), reg, offsets, nms, mode=mode,
                          top_k=top_k, cls_sel=sel, softmax_before_filter=sbf, regress=regress)
    dets, counts = d["dets"].cpu().numpy(), d["counts"].cpu().numpy()
    for c in range(K):
        want, wv = GOLD["%s_det_%d" % (name, c)], GOLD["%s_det_video_%d" % (name, c)]
        got, gv = [], []
        for v in range(len(vids)):
            pre = d["slot0"][v] + int(counts[v, :c].sum())
            got.append(dets[pre:pre + counts[v, c]])
            gv += [v] * int(counts[v, c])
        got = np.concatenate(got).astype(np.float64)
        assert got.shape == want.shape and np.array_equal(np.array(gv), wv), (name, c)
        if len(got):
            assert np.array_equal(got[:, 3:], want[:, 3:]), (name, c)                 # loc / dur: the survivor's identity
            assert np.abs(got[:, 2] - want[:, 2]).max() <= 4e-6 * np.abs(want[:, 2]).max(), (name, c)
            assert np.abs(got[:, :2] - want[:, :2]).max() <= 4e-7, (name, c)


# ---- seeded sets -------------------------------------------------------------------------------------------------------------
def synth_set(kind, seed, V=None):
    """THUMOS14-like (K 20, N median ~111, max 2914) or ActivityNet1.2-like (K 100, N median ~45, max 187) scores, proposals and
    ground truth; 'ties': quantised logits with NaN / inf rows, identical and zero-length boxes"""
    g = np.random.RandomState(seed)
    if kind == "thumos":
        V = V or 1574
        K, ns = 20, np.clip(np.exp(g.normal(np.log(111), 1.0, V)).astype(int), 1, 2914)
        ns[0] = 2914
        n_gt = np.clip(g.poisson(10, V), 0, 218)
        n_gt[1] = 218
    elif kind == "anet":
        V = V or 2383
        K, ns = 100, np.clip(np.exp(g.normal(np.log(45), 0.6, V)).astype(int), 1, 187)
        n_gt = np.clip(g.poisson(1.5, V), 0, 18)
    else:
        V = V or 12
        K, ns = 5, g.randint(0, 40, V)
        n_gt = g.randint(0, 6, V)
    N = int(ns.sum())
    c, d = g.rand(N), 0.01 + 0.3 * g.rand(N)
    props = np.stack([np.clip(c - d / 2, 0, 1), np.clip(c + d / 2, 0, 1)], 1).astype(np.float32)
    act = (g.randn(N, K + 1) * 2).astype(np.float32)
    comp = g.randn(N, K).astype(np.float32)
    reg = (g.randn(N, K, 2) * 0.2).astype(np.float32)
    if kind == "ties":
        act = np.round(act)
        comp = np.round(comp * 2) / 2
        rows = g.choice(N, 8, replace=False)
        act[rows[0], 2] = np.nan
        act[rows[1], 0] = np.inf
        act[rows[2], 3] = -np.inf
        act[rows[3], :] = -np.inf
        comp[rows[4], 1] = np.inf
        props[rows[5]] = props[rows[6]]                     # identical boxes
        props[rows[7]] = (0.5, 0.5)                         # zero-length box
        reg[rows[:3], :, 0] = -60.0                         # regressed onto [0, 0]
    offsets = np.concatenate([[0], np.cumsum(ns)]).tolist()
    gv, gc, gs = [], [], []
    for v in range(V):
        for _ in range(int(n_gt[v])):
            a = g.rand() * 0.9
            gv.append(v); gc.append(int(g.randint(0, K))); gs.append((a, min(1.0, a + 0.02 + 0.2 * g.rand())))
    if kind == "ties":
        gv += [0, 0, 1]; gc += [1, 1, 2]; gs += [(0.0, 0.0), (0.0, 0.0), (0.5, 0.5)]
    order = np.argsort(np.array(gv), kind="stable")
    gv, gc, gs = np.array(gv)[order], np.array(gc, np.int32)[order], np.array(gs, np.float64).reshape(-1, 2)[order]
    goff = np.searchsorted(gv, np.arange(V + 1)).tolist()
    gt = {"offsets": goff, "cls": torch.tensor(gc, device=dev()), "seg": torch.tensor(gs, device=dev())}
    return props, act, comp, reg, offsets, K, gt


def run_staged(kind, mode, top_k, nms, thr, classes, seed, sbf=True, reg_none=False):
    from ops.detection import detections_packed, detection_ap
    props, act, comp, reg, offsets, K, gt = synth_set(kind, seed)
    V = len(offsets) - 1
    sel = np.stack([np.random.RandomState(seed + v).permutation(K)[:3] for v in range(V)]) if mode == "cls" else None
    T = lambda x: torch.tensor(x, device=dev())
    t0 = time.perf_counter()
    res = detections_packed(T(props), T(act), T(comp), None if reg_none else T(reg), offsets, nms, mode=mode, top_k=top_k, cls_sel=sel,
                            softmax_before_filter=sbf, trace=True)
    ap = detection_ap(res, gt, thr, trace=True)
    torch.cuda.synchronize()
    gpu_s = time.perf_counter() - t0
    chk = E.check(res, ap, props, act, comp, None if reg_none else reg, offsets, mode, nms, gt, thr, top_k=top_k, cls_sel=sel,
                  softmax_before_filter=sbf, classes=classes)
    print("%s %s: %d videos, %d proposals, %s, gpu %.3f s (first call)" % (kind, mode, V, offsets[-1], chk.stats, gpu_s))
    chk.assert_ok()
    return chk


def test_staged_thumos_like():
    chk = run_staged("thumos", "top_k", 2000, 0.2, np.arange(0.1, 1.0, 0.1), [0, 7], seed=11)
    assert chk.stats["videos"] == 1574 and chk.stats["kept"] > 0


def test_staged_activitynet_like():
    chk = run_staged("anet", "top_k", 60, 0.6, np.arange(0.5, 1.0, 0.05), [0, 1, 2, 50], seed=12)
    assert chk.stats["videos"] == 2383 and chk.stats["kept"] > 0


@pytest.mark.parametrize("mode,sbf,reg_none", [("all", True, False), ("top_k", True, True), ("cls", True, False), ("cls", False, False)])
def test_ties_nan_inf_and_degenerate_boxes(mode, sbf, reg_none):
    chk = run_staged("ties", mode, 17, 0.3, np.arange(0.1, 1.0, 0.1), None, seed=13, sbf=sbf, reg_none=reg_none)
    assert chk.stats["selected"] > 0


# ---- call properties ---------------------------------------------------------------------------------------------------------
class Batch:
    """fixed buffers for direct library calls (graph capture, pre-filled outputs)"""

    def __init__(self, props, act, comp, reg, offsets, K, mode="top_k", top_k=25, nms=0.4, fill=0):
        from ssn_b200._lib import lib, DetectBatchCfg, DET_ALL, DET_TOPK
        from ops.detection import detection_slots
        self.lib = lib
        T = lambda x: torch.tensor(x, device=dev())
        self.props, self.act, self.comp, self.reg = T(props), T(act), T(comp), T(reg)
        self.V, self.K = len(offsets) - 1, K
        self.cfg = DetectBatchCfg(DET_TOPK if mode == "top_k" else DET_ALL, top_k, 0, 1, 1, 0, nms)
        self.offs = (C.c_int64 * (self.V + 1))(*offsets)
        self.offs_dev = torch.tensor(offsets, dtype=torch.int64, device=dev())
        S = detection_slots(offsets, K, mode, top_k)[-1]
        self.dets = torch.full((S, 5), 0, dtype=torch.float32, device=dev())
        self.counts = torch.zeros(self.V, K, dtype=torch.int32, device=dev())
        if fill:
            self.dets.view(torch.uint8).fill_(fill)
            self.counts.view(torch.uint8).fill_(fill)
        self.ws_bytes = lib.ssnb_detect_batch_workspace_bytes(C.byref(self.cfg), K, self.offs, self.V)
        self.ws = torch.full((self.ws_bytes,), fill, dtype=torch.uint8, device=dev())

    def __call__(self):
        return self.lib.ssnb_detect_batch(C.byref(self.cfg), self.props.data_ptr(), self.act.data_ptr(), self.comp.data_ptr(), self.reg.data_ptr(),
                                          self.K, self.offs, self.offs_dev.data_ptr(), self.V, None, self.dets.data_ptr(),
                                          self.counts.data_ptr(), None, None, self.ws.data_ptr(), self.ws_bytes,
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream))

    def result(self):
        torch.cuda.synchronize()
        return self.dets.clone(), self.counts.clone()


def test_one_call_equals_per_video_calls_repeat_and_prefill():
    from ops.detection import detections_packed, detection_ap, pack_ground_truth
    props, act, comp, reg, offsets, K, gt = synth_set("thumos", 21, V=40)
    T = lambda x: torch.tensor(x, device=dev())
    whole = detections_packed(T(props), T(act), T(comp), T(reg), offsets, 0.2, mode="top_k", top_k=300)
    again = detections_packed(T(props), T(act), T(comp), T(reg), offsets, 0.2, mode="top_k", top_k=300)
    assert torch.equal(whole["counts"], again["counts"])
    n = int(whole["counts"].sum())
    for v in range(len(offsets) - 1):
        lo, hi = offsets[v], offsets[v + 1]
        one = detections_packed(T(props[lo:hi]), T(act[lo:hi]), T(comp[lo:hi]), T(reg[lo:hi]), [0, hi - lo], 0.2, mode="top_k", top_k=300)
        m = int(one["counts"].sum())
        s0 = whole["slot0"][v]
        assert torch.equal(one["counts"][0], whole["counts"][v])
        assert torch.equal(one["dets"][:m].view(torch.int32), whole["dets"][s0:s0 + m].view(torch.int32))
        assert torch.equal(again["dets"][s0:s0 + m].view(torch.int32), whole["dets"][s0:s0 + m].view(torch.int32))
    # AP: repeat is bitwise
    g = {"offsets": gt["offsets"], "cls": gt["cls"], "seg": gt["seg"]}
    a1, a2 = detection_ap(whole, g, np.arange(0.1, 1.0, 0.1), trace=True), detection_ap(whole, g, np.arange(0.1, 1.0, 0.1), trace=True)
    assert torch.equal(a1["ap"].view(torch.int64), a2["ap"].view(torch.int64)) and torch.equal(a1["tp"], a2["tp"])
    # pre-filled output and workspace memory
    b0, bf = Batch(props, act, comp, reg, offsets, K, top_k=300, nms=0.2), Batch(props, act, comp, reg, offsets, K, top_k=300, nms=0.2, fill=0xFF)
    assert b0() == 0 and bf() == 0
    (d0, c0), (d1, c1) = b0.result(), bf.result()
    assert torch.equal(c0, c1) and torch.equal(c0, whole["counts"])
    for v in range(len(offsets) - 1):
        s0, m = whole["slot0"][v], int(c0[v].sum())
        assert torch.equal(d0[s0:s0 + m].view(torch.int32), d1[s0:s0 + m].view(torch.int32))


def test_cuda_graph_replay_on_new_scores_equals_eager():
    props, act, comp, reg, offsets, K, _ = synth_set("anet", 31, V=50)
    b = Batch(props, act, comp, reg, offsets, K, top_k=60, nms=0.6)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert b() == 0                                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert b() == 0
    g = np.random.RandomState(32)
    act2, comp2 = (g.randn(*act.shape) * 2).astype(np.float32), g.randn(*comp.shape).astype(np.float32)
    b.act.copy_(torch.tensor(act2)); b.comp.copy_(torch.tensor(comp2))
    b.dets.fill_(0); b.counts.fill_(0)
    graph.replay()
    dg, cg = b.result()
    e = Batch(props, act2, comp2, reg, offsets, K, top_k=60, nms=0.6)
    assert e() == 0
    de, ce = e.result()
    assert torch.equal(cg, ce) and int(ce.sum()) > 0
    assert torch.equal(dg.view(torch.int32), de.view(torch.int32))


def test_rejected_arguments_return_before_any_launch():
    from ssn_b200._lib import lib, DetectBatchCfg, DET_TOPK, DET_CLS
    props, act, comp, reg, offsets, K, gt = synth_set("ties", 41, V=3)
    b = Batch(props, act, comp, reg, offsets, K, top_k=5)
    n0 = lib.ssnb_global_launch_count()
    for cfg in (DetectBatchCfg(DET_TOPK, 0, 0, 1, 1, 0, 0.4), DetectBatchCfg(DET_CLS, 0, 2, 1, 1, 0, 0.4),
                DetectBatchCfg(DET_TOPK, 5, 0, 1, 1, 0, float("nan"))):
        b.cfg = cfg
        assert b() != 0
    b.cfg = DetectBatchCfg(DET_TOPK, 5, 0, 1, 1, 0, 0.4)
    ws = b.ws_bytes
    b.ws_bytes = ws - 1
    assert b() != 0
    b.ws_bytes = ws
    S = int(b.dets.shape[0])
    thr = (C.c_double * 2)(0.5, float("nan"))
    ap = torch.empty(K, 2, dtype=torch.float64, device=dev())
    wsb = lib.ssnb_detection_ap_workspace_bytes(3, K, S, 1, 2)
    w = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev())
    slot0 = torch.zeros(4, dtype=torch.int64, device=dev())
    rc = lib.ssnb_detection_ap(b.dets.data_ptr(), b.counts.data_ptr(), slot0.data_ptr(), 3, K, S, slot0.data_ptr(), gt["cls"].data_ptr(),
                               gt["seg"].data_ptr(), 1, thr, 2, ap.data_ptr(), None, None, w.data_ptr(), wsb, None)
    assert rc != 0                                            # NaN threshold
    assert lib.ssnb_global_launch_count() == n0
