"""ActivityNet AR-AN on the GPU (ops/proposal_eval.py, csrc/proposal_ar.cu) bitwise against the real toolkit's results
(tests/golden/anet_proposal.npz) and against oracle/anet_proposal_oracle.py on a random ragged batch of 3000 videos with
ties, NaN scores and coordinates, videos without proposals and videos outside the ground truth, read from a gapped slot
layout; TAG proposals evaluated where bottom_up_proposals_packed left them; CUDA-graph replay; the refusals.
Nothing here reads a checkout of the reference."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from oracle import anet_proposal_oracle as O
from test_anet_proposal_host import FIXTURES, GOLD, fixture
from test_proplist_host import same

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def T(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(dev())


def npy(t):
    return t.cpu().numpy()


def run(f, trace=True, first=None, boxes=None, scores=None):
    from ops import proposal_eval as E
    from ops.proposal_lists import compact_layout
    if first is None:
        first, count = compact_layout(f["counts"], dev())
    else:
        count = T(f["counts"], torch.int32)
    return E.average_recall_packed(T(f["boxes"] if boxes is None else boxes), T(f["scores"] if scores is None else scores), first, count,
                                   f["gt_seg"], f["gt_offsets"], f["max_avg"], f["thresholds"], trace=trace)


def check_against(r, want, first_hit=None):
    for k in ("recall", "avg_recall", "proposals_per_video"):
        assert same(npy(r[k]), want[k]), k
    assert int(r["total_nr"]) == int(want["total_nr"])
    assert same(npy(r["nr"]), want["nr"])
    if first_hit is not None:
        assert same(npy(r["first_hit"]), first_hit)


@pytest.mark.parametrize("name", FIXTURES)
def test_golden_fixture_bitwise(name):
    from ops import proposal_eval as E
    f = fixture(name)
    r = run(f)
    check_against(r, {k: GOLD[name + "_" + k] for k in ("recall", "avg_recall", "proposals_per_video", "total_nr", "nr")})
    rep = E.ar_an_report(r)
    assert (rep["auc"], rep["auc_percent"]) == (float(GOLD[name + "_auc"]), float(GOLD[name + "_auc_percent"]))
    o = O.average_recall(f["boxes"], f["scores"], f["counts"], f["gt_seg"], f["gt_counts"], f["max_avg"], f["thresholds"])
    assert same(npy(r["first_hit"]), o["first_hit"])


def test_evaluate_proposals_from_json():
    from ops import proposal_eval as E
    gt_j, pr_j = json.loads(str(GOLD["json_gt_text"])), json.loads(str(GOLD["json_pr_text"]))
    rep = E.evaluate_proposals(gt_j, pr_j, blocked_videos=[str(x) for x in GOLD["json_blocked"]])
    for k in ("recall", "avg_recall", "proposals_per_video"):
        assert same(rep[k], GOLD["json_" + k]), k
    assert rep["auc_percent"] == float(GOLD["json_auc_percent"])


def random_batch(seed, V=3000):
    """ragged videos: 0..2000 proposals and 0..30 instances; scores drawn from a small set in some videos (ties, NaN, -0 at
    every size), NaN and reversed coordinates; the packed rows of video v start at a gapped slot (the TAG layout)"""
    g = np.random.RandomState(seed)
    counts, gcounts, boxes, scores, gts = [], [], [], [], []
    for v in range(V):
        n = int(g.choice([0, g.randint(1, 17), g.randint(17, 300), g.randint(300, 2001)], p=[0.04, 0.4, 0.5, 0.06]))
        ng = int(g.choice([0, g.randint(1, 4), g.randint(4, 31)], p=[0.05, 0.75, 0.2]))
        dur = float(g.uniform(10, 600))
        c, d = g.uniform(0, dur, ng), g.uniform(0.5, dur / 3, ng)
        gt = np.stack([np.clip(c - d / 2, 0, dur), np.clip(c + d / 2, 0, dur)], 1).reshape(-1, 2)
        pc, pd = g.uniform(0, dur, n), g.uniform(0.2, dur / 2, n)
        b = np.stack([pc - pd / 2, pc + pd / 2], 1).reshape(-1, 2)
        k = min(n, ng)
        b[:k] = gt[:k] + g.uniform(-0.1, 0.1, (k, 2)) * (gt[:k, 1:] - gt[:k, :1])
        if n > 5:
            b[2] = b[2, ::-1]
            b[3, 1] = b[3, 0]
            b[4, 0] = np.nan
        s = g.rand(n)
        if v % 4 == 0:
            s = g.choice(np.array([np.nan, 1.0, 0.5, 0.25, 0.0, -0.0]), n)
        counts.append(n), gcounts.append(ng), boxes.append(b), scores.append(s), gts.append(gt)
    return counts, gcounts, boxes, scores, gts


def gapped(counts, boxes, scores, seed):
    """rows of video v from first[v] on, with 0..7 unused rows (NaN-filled) before each video"""
    g = np.random.RandomState(seed)
    first, at = [], 0
    for n in counts:
        at += int(g.randint(0, 8))
        first.append(at)
        at += n
    B, S = np.full((at + 3, 2), np.nan), np.full(at + 3, np.nan)
    for f, n, b, s in zip(first, counts, boxes, scores):
        B[f:f + n], S[f:f + n] = b, s
    return np.array(first, np.int64), B, S


@pytest.mark.parametrize("max_avg", [None, 100, 7.5])
def test_random_ragged_batch_against_oracle(max_avg):
    counts, gcounts, boxes, scores, gts = random_batch(5)
    thr = np.linspace(0.5, 0.95, 10) if max_avg != 7.5 else np.array([0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 1.0])
    f = {"counts": np.array(counts), "gt_seg": np.concatenate(gts), "gt_offsets": np.concatenate([[0], np.cumsum(gcounts)]),
         "max_avg": max_avg, "thresholds": thr}
    first, B, S = gapped(counts, boxes, scores, 6)
    r = run(f, first=T(first), boxes=B, scores=S)
    o = O.average_recall(np.concatenate(boxes), np.concatenate(scores), counts, f["gt_seg"], gcounts, max_avg, thr)
    assert (o["nr"] > 0).sum() > 1500 and o["nr"].max() > 90 and o["total_nr"] > 19000
    check_against(r, o, o["first_hit"])
    # the same batch compact: the same answer
    f.update(boxes=np.concatenate(boxes), scores=np.concatenate(scores))
    check_against(run(f), o, o["first_hit"])


def test_tag_proposals_evaluated_in_place():
    """bottom_up_proposals_packed -> average_recall_packed on its seconds / slot0 / counts, nothing copied to the host between"""
    from ops import proposal_eval as E
    from ops.proposals import bottom_up_proposals_packed
    g = torch.Generator().manual_seed(3)
    Ts = [37, 90, 160, 64, 211, 120, 75]
    durs = [12.0, 30.0, 55.5, 21.3, 70.1, 44.0, 25.0]
    sc = torch.cat([torch.randn(t, 2, generator=g) * torch.tensor([0.3, 2.0]) for t in Ts]).to(dev())
    tag = bottom_up_proposals_packed(sc, np.concatenate([[0], np.cumsum(Ts)]).tolist(), durs)
    rs = np.random.RandomState(4)
    gts = [np.sort(rs.uniform(0, d, (n, 2)), 1) for d, n in zip(durs, (2, 0, 4, 1, 3, 5, 1))]
    goff = np.concatenate([[0], np.cumsum([len(x) for x in gts])]).tolist()
    r = E.average_recall_packed(tag["seconds"], tag["scores"], tag["slot0"].to(dev()), tag["counts"], T(np.concatenate(gts)), goff,
                                max_avg_nr_proposals=50, trace=True)
    rep = E.ar_an_report(r)
    counts, slot0, sec, s32 = npy(tag["counts"]), tag["slot0"].numpy(), npy(tag["seconds"]), npy(tag["scores"])
    b = np.concatenate([sec[s:s + n] for s, n in zip(slot0, counts)])
    s = np.concatenate([s32[s:s + n] for s, n in zip(slot0, counts)]).astype(np.float64)
    o = O.average_recall(b, s, counts, np.concatenate(gts), np.diff(goff), 50, O.THRESHOLDS)
    check_against(r, o, o["first_hit"])
    assert counts.min() > 0 and o["total_nr"] > 0 and rep["auc"] == O.area(o["avg_recall"], o["proposals_per_video"])[0]


def test_cuda_graph_replay_equals_eager():
    from ops import proposal_eval as E
    from ssn_b200._lib import lib, check
    counts, gcounts, boxes, scores, gts = random_batch(8, V=300)
    B, S = T(np.concatenate(boxes)), T(np.concatenate(scores))
    first, cnt = T(np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)), T(counts, torch.int32)
    off = np.concatenate([[0], np.cumsum(gcounts)]).astype(np.int64).tolist()
    V, rows, thr = len(counts), B.shape[0], [0.3, 0.5, 0.7]
    gt, off_d = T(np.concatenate(gts)), T(off)
    off_c, thr_c = (C.c_int64 * len(off))(*off), (C.c_double * 3)(*thr)
    ws_bytes = lib.ssnb_proposal_ar_workspace_bytes(V, rows, off_c, 3)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    o = dict(recall=torch.empty(3, 100, dtype=torch.float64, device=dev()), avg=torch.empty(100, dtype=torch.float64, device=dev()),
             ppv=torch.empty(100, dtype=torch.float64, device=dev()), total=torch.empty(1, dtype=torch.int64, device=dev()),
             nr=torch.empty(V, dtype=torch.int32, device=dev()), hit=torch.empty(off[-1], 3, dtype=torch.int32, device=dev()))

    def enqueue():
        check(lib.ssnb_proposal_ar(B.data_ptr(), S.data_ptr(), rows, first.data_ptr(), cnt.data_ptr(), V, gt.data_ptr(), off_c,
                                   off_d.data_ptr(), thr_c, 3, 20.0, o["recall"].data_ptr(), o["avg"].data_ptr(), o["ppv"].data_ptr(),
                                   o["total"].data_ptr(), o["nr"].data_ptr(), o["hit"].data_ptr(), ws.data_ptr(), ws_bytes,
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "proposal_ar")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        enqueue()                                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        enqueue()
    rs = np.random.RandomState(9)
    S.copy_(T(rs.rand(rows)))                              # new scores, same shapes
    for t in o.values():
        t.view(torch.uint8).fill_(0xFF)
    graph.replay()
    torch.cuda.synchronize()
    e = E.average_recall_packed(B, S, first, cnt, gt, off, 20.0, thr, trace=True)
    for k, ek in (("recall", "recall"), ("avg", "avg_recall"), ("ppv", "proposals_per_video"), ("total", "total_nr"), ("nr", "nr"),
                  ("hit", "first_hit")):
        assert same(npy(o[k]), npy(e[ek])), k
    old = O.average_recall(np.concatenate(boxes), np.concatenate(scores), counts, np.concatenate(gts), gcounts, 20.0, thr)
    assert not same(npy(e["first_hit"]), old["first_hit"])        # the replay did see the new scores


def test_no_kept_proposal_raises_and_cpu_tensors_are_refused():
    from ops import proposal_eval as E
    f = {"boxes": np.zeros((0, 2)), "scores": np.zeros(0), "counts": [0, 0], "gt_seg": np.array([[0.0, 1.0], [2.0, 3.0]]),
         "gt_offsets": [0, 1, 2], "max_avg": None, "thresholds": [0.5]}
    r = run(f)
    assert int(r["total_nr"]) == 0 and torch.isnan(r["avg_recall"]).all()
    with pytest.raises(ValueError):
        E.ar_an_report(r)
    f.update(boxes=np.array([[0.0, 1.0]]), scores=np.array([0.3]), counts=[1, 0], max_avg=0.5)    # ratio 0.5 * 2 / 1 = 1: kept
    assert int(run(f)["total_nr"]) == 1
    f.update(max_avg=0.2)                                                                         # int(0.4) = 0: nothing kept
    with pytest.raises(ValueError):
        E.ar_an_report(run(f))
    with pytest.raises(ValueError):
        E.evaluate_proposals({"database": {"a": {"subset": "validation", "annotations": [{"segment": [0, 1], "label": "x"}]}},
                              "taxonomy": [], "version": ""}, {"results": {}, "version": "", "external_data": {}})
    with pytest.raises(ValueError):
        run(dict(f, max_avg=-1.0))
    with pytest.raises(RuntimeError):
        E.average_recall_packed(T(np.zeros((1, 2))), torch.zeros(1, dtype=torch.float64), [0], [1], np.zeros((1, 2)), [0, 1])
