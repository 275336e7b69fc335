"""Proposal labelling on the GPU (ops/proposal_lists.py, csrc/proposal_lists.cu), each stage fed what the stage before wrote:
  - against tests/golden/proplist.npz (the real reference) and against oracle/proplist_oracle.py on a random ragged batch:
    bitwise except size_reg (CUDA's log: 4 ulp) and reg_stats (another summation order: 1e-12 relative);
  - ties, NaN and +-inf coordinates; batch call == per-video calls == a repeat with outputs pre-filled with 0xFF; CUDA-graph
    replay on new boxes; the chain from actionness scores to the test-time tail.
Nothing here reads a checkout of the reference."""

import numpy as np
import pytest
import torch

from oracle import proplist_oracle as P
from test_proplist_host import GOLD, ragged, records, same

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def T(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(dev())


def npy(t):
    return t.cpu().numpy()


def offsets(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64).tolist()


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64)).max() if a.size else 0


def random_batch(seed, V=240):
    """ragged videos with durations and frame counts of both data sets; N_v from 0 to ~3000, G_v from 0 to > 256"""
    g = np.random.RandomState(seed)
    vids = []
    for v in range(V):
        duration = float(g.uniform(5, 60) if v % 2 else g.uniform(60, 900))
        fc = int(duration * g.choice([25.0, 29.97, 30.0]))
        n = int(g.choice([0, 1, g.randint(2, 200), g.randint(200, 600)], p=[0.05, 0.05, 0.8, 0.1]))
        ng = int(g.choice([0, g.randint(1, 12)], p=[0.1, 0.9]))
        if v == 7:
            n, ng = 3100, 9
        if v in (11, 12):
            n, ng = 300, (257 if v == 11 else 600)
        c, d = g.uniform(0, duration, ng), g.uniform(0.5, duration / 3, ng)
        gt = np.stack([np.clip(c - d / 2, 0, duration), np.clip(c + d / 2, 0, duration)], 1).reshape(-1, 2)
        pc, pd = g.uniform(0, duration * 1.05, n), g.uniform(0.2, duration / 2, n)
        boxes = np.stack([np.clip(pc - pd / 2, 0, None), pc + pd / 2], 1).reshape(-1, 2)
        k = min(n, ng)
        boxes[:k] = gt[:k] + g.uniform(-0.08, 0.08, (k, 2)) * (gt[:k, 1:] - gt[:k, :1])
        if n > 4:
            boxes[3] = boxes[3, ::-1]
            boxes[4, 1] = boxes[4, 0]
        vids.append(dict(duration=duration, frame_cnt=fc, boxes=boxes, gt=gt, gt_label=g.randint(0, 20, ng).astype(np.int32)))
    return vids


def pack(vids):
    cnt, gcnt = [len(v["boxes"]) for v in vids], [len(v["gt"]) for v in vids]
    from ops.proposal_lists import compact_layout
    first, count = compact_layout(cnt, dev())
    return dict(boxes=T(np.concatenate([v["boxes"] for v in vids]).reshape(-1, 2)), first=first, count=count, counts=cnt,
                gt=T(np.concatenate([v["gt"] for v in vids]).reshape(-1, 2)), gt_label=T(np.concatenate([v["gt_label"] for v in vids]).astype(np.int32)),
                gt_offsets=offsets(gcnt), duration=[v["duration"] for v in vids], frame_cnt=[v["frame_cnt"] for v in vids])


def golden_vids():
    b, g, l, dur, fc = ragged()
    return [dict(duration=float(d), frame_cnt=int(f), boxes=x, gt=y, gt_label=z) for x, y, z, d, f in zip(b, g, l, dur, fc)]


# ---- golden ------------------------------------------------------------------------------------------------------------------
def test_label_and_list_against_reference_golden(tmp_path):
    from ops import proposal_lists as L
    p = pack(golden_vids())
    r = L.label_proposals(p, p["gt"], p["gt_label"], p["gt_offsets"], p["duration"], p["frame_cnt"], GOLD["rag_thresholds"])
    for k in ("label", "max_overlap", "overlap_self"):
        assert same(npy(r[k]), GOLD["rag_" + k]), k
    assert same(npy(r["recall"]["hits"]).astype(np.int64), GOLD["rag_hits"])
    rep = L.recall_report(r["recall"], r["count"])
    assert same(np.stack([rep["per_video"], rep["per_instance"]], 1), GOLD["rag_recall"])
    assert same(rep["average"], np.mean(GOLD["rag_recall"], axis=0)) and rep["average_proposals"] == np.mean(GOLD["rag_count"])
    dirs = ["frames/video_%04d" % i for i in range(len(p["counts"]))]
    path = str(tmp_path / "list.txt")
    assert L.write_proposal_list(path, r, dirs) == str(GOLD["rag_text"]) == open(path).read()
    # the written list read back and through the data set's rules, targets and test-time inputs
    check_loaded(L, L.record_rows(L.load_proposal_list(path)), "rag_")


def check_loaded(L, rows, prefix):
    g = lambda k: GOLD[prefix + "ds_" + k]
    assert same(np.array(rows["counts"], np.int32), g("count")) and same(np.diff(rows["gt_offsets"]).astype(np.int32), g("gt_count"))
    for k in ("frames", "coverage", "best_iou", "overlap_self", "label", "gt_frames", "gt_label"):
        assert same(npy(rows[k]), g(k)), k
    t = L.proposal_targets(rows["frames"], rows["best_iou"], rows["overlap_self"], rows["coverage"], rows["first"], rows["count"],
                           rows["gt_frames"], rows["gt_offsets"])
    assert same(npy(t["tags"]), g("tags"))
    reg = npy(t["reg"])
    assert same(reg[:, 0], g("reg")[:, 0]) and ulps(reg[:, 1], g("reg")[:, 1]) <= 4
    assert same(npy(t["pool_counts"])[:, :3], g("pools"))
    tot = npy(t["totals"]).tolist()
    assert [tot[0] + tot[3], tot[1], tot[2], tot[4]] == g("pool_totals").tolist()
    assert np.abs(npy(t["reg_stats"]) - g("stats")).max() <= 1e-12 * np.abs(g("stats")).max()
    s = L.test_proposals(rows["frames"], rows["counts"], rows["frame_cnt"])
    assert same(npy(s["num_ticks"]), g("num_ticks"))
    for k, gk in (("rel_prop", "rel_prop"), ("proposal_ticks", "ticks"), ("scaling", "scaling")):
        assert same(npy(s[k]), g(gk)), k
    assert same(npy(s["ticks32"]), g("ticks").astype(np.int32)) and same(npy(s["scaling32"]), g("scaling").astype(np.float32))


def test_normalised_list_against_reference_golden(tmp_path):
    from ops import proposal_lists as L
    path = str(tmp_path / "norm.txt")
    open(path, "w").write(str(GOLD["norm_text"]))
    loaded = L.load_proposal_list(path)
    check_loaded(L, L.record_rows(loaded, GOLD["norm_frame_cnt"], mode="normalised"), "norm_")
    # process_proposal_list's text from the same loaded list
    fc = T(GOLD["norm_frame_cnt"])
    g_n = np.diff(loaded["gt_offsets"])
    g_first, g_count = L.compact_layout(g_n, dev())
    res = dict(loaded, frame_cnt=fc, frames=L.proposal_frames(loaded["boxes"], loaded["first"], loaded["count"], fc, None, "normalised")["frames"],
               gt_frames=L.proposal_frames(loaded["gt"], g_first, g_count, fc, None, "normalised")["frames"])
    assert L.format_proposal_list(res, ["frames/" + i for i in loaded["ids"]], style="processed") == str(GOLD["norm_processed_text"])


def test_sliding_windows_against_golden_and_oracle():
    from ops import proposal_lists as L
    for c, (ts, ml, ov) in enumerate(GOLD["sw_configs"]):
        r = L.sliding_window_proposals(GOLD["sw_durations"].tolist(), int(ts), int(ml), float(ov))
        assert same(npy(r["count"]), GOLD["sw%d_count" % c])
        total = int(r["total"])
        assert total == len(GOLD["sw%d_boxes" % c]) and same(npy(r["boxes"])[:total], GOLD["sw%d_boxes" % c])
        assert same(npy(r["first"]), np.cumsum(GOLD["sw%d_count" % c].astype(np.int64)) - GOLD["sw%d_count" % c])
    g = np.random.RandomState(3)
    durs = np.concatenate([g.uniform(0.2, 40, 150), g.uniform(40, 800, 150), [0.0, -3.0, 1.0, 0.9999999999999999, 2.0, 3.0000000000000004]])
    for ts, ml, ov in ((1, 8, 0.7), (3, 5, 0.25), (0.5, 7, 0.4)):
        want = [P.sliding_windows(d, ts, ml, ov) for d in durs]
        # a device tensor of durations with a capacity: no host synchronisation inside
        cap = sum(len(w) for w in want) + 5
        r = L.sliding_window_proposals(T(durs), ts, ml, ov, capacity=cap)
        assert same(npy(r["count"]), np.array([len(w) for w in want], np.int32)) and int(r["total"]) == cap - 5
        assert same(npy(r["boxes"])[:cap - 5], np.concatenate(want))
        # and they are directly an input of the naming call
        gt = T(np.array([[1.0, 4.0]] * len(durs)))
        n = L.name_proposals_packed(r["boxes"], r["first"], r["count"], gt, T(np.zeros(len(durs), np.int32)), list(range(len(durs) + 1)))
        w0 = P.name_proposals([(1.0, 4.0)], [0], want[3])
        f0 = int(r["first"][3])
        assert same(npy(n["max_overlap"])[f0:f0 + len(want[3])], w0[1])


# ---- random ragged batch vs the oracle ----------------------------------------------------------------------------------------
def oracle_name(vids):
    named = [P.name_proposals(v["gt"], v["gt_label"], v["boxes"]) for v in vids]
    return [np.concatenate([n[i] for n in named]) for i in range(3)] + [np.concatenate([P.gt_best_iou(v["gt"], v["boxes"]) for v in vids])]


def test_random_ragged_batch_against_oracle():
    from ops import proposal_lists as L
    vids = random_batch(1)
    p = pack(vids)
    thr = [0.3, 0.5, 0.7, 0.9]
    r = L.label_proposals(p, p["gt"], p["gt_label"], p["gt_offsets"], p["duration"], p["frame_cnt"], thr)
    want = oracle_name(vids)
    for k, w in zip(("label", "max_overlap", "overlap_self", "gt_best"), want):
        assert same(npy(r[k]), w), k
    hits, pv, pi = P.proposal_recall(np.split(want[3], np.cumsum([len(v["gt"]) for v in vids])[:-1]), thr)
    assert same(npy(r["recall"]["hits"]).astype(np.int64), hits)
    rep = L.recall_report(r["recall"])
    assert same(rep["per_video"], pv) and same(rep["per_instance"], pi)
    assert same(npy(r["frames"]), np.concatenate([P.seconds_to_frames(v["boxes"], v["duration"], v["frame_cnt"]) for v in vids]))
    assert same(npy(r["gt_frames"]), np.concatenate([P.seconds_to_frames(v["gt"], v["duration"], v["frame_cnt"]) for v in vids]))
    # fresh (unrounded) overlaps as best_iou / overlap_self, the data set's rules on the frame windows
    f = L.proposal_frames(p["boxes"], p["first"], p["count"], p["frame_cnt"], p["duration"], "seconds")
    g_first, g_count = L.compact_layout(np.diff(p["gt_offsets"]), dev())
    gf = L.proposal_frames(p["gt"], g_first, g_count, p["frame_cnt"], p["duration"], "seconds")
    ovids, at, gat = [], 0, 0
    for v in vids:
        n, ng = len(v["boxes"]), len(v["gt"])
        keep, valid, cov = P.record_rows(P.seconds_to_frames(v["boxes"], v["duration"], v["frame_cnt"]), v["frame_cnt"])
        gkeep, gvalid, _ = P.record_rows(P.seconds_to_frames(v["gt"], v["duration"], v["frame_cnt"]), v["frame_cnt"])
        assert same(npy(f["keep"][at:at + n]).astype(bool), keep) and same(npy(f["valid"][at:at + n]), valid) and same(npy(f["coverage"][at:at + n]), cov)
        assert same(npy(gf["keep"][gat:gat + ng]).astype(bool), gkeep)
        ovids.append(dict(frame_cnt=v["frame_cnt"], frames=valid[keep], coverage=cov[keep], best_iou=want[1][at:at + n][keep],
                          overlap_self=want[2][at:at + n][keep], gt_frames=gvalid[gkeep]))
        at, gat = at + n, gat + ng
    keep, gkeep = f["keep"].bool(), gf["keep"].bool()
    first, count = L.compact_layout([len(o["frames"]) for o in ovids], dev())
    goff = offsets([len(o["gt_frames"]) for o in ovids])
    for exclude in (True, False):
        t = L.proposal_targets(f["valid"][keep], r["max_overlap"][keep], r["overlap_self"][keep], f["coverage"][keep], first, count,
                               gf["valid"][gkeep], goff, exclude_empty=exclude)
        out, stats, totals = P.proposal_targets(ovids, exclude_empty=exclude)
        assert same(npy(t["tags"]), np.concatenate([o["tags"] for o in out]))
        reg, wreg = npy(t["reg"]), np.concatenate([o["reg"] for o in out])
        assert same(reg[:, 0], wreg[:, 0]) and ulps(reg[:, 1], wreg[:, 1]) <= 4
        assert npy(t["pool_counts"]).tolist() == [o["pools"] for o in out] and npy(t["totals"]).tolist() == totals
        assert totals[0] > 50 and np.abs(npy(t["reg_stats"]) - stats).max() <= 1e-12 * np.abs(stats).max()
        t2 = L.proposal_targets(f["valid"][keep], r["max_overlap"][keep], r["overlap_self"][keep], f["coverage"][keep], first, count,
                                gf["valid"][gkeep], goff, exclude_empty=exclude)
        assert same(npy(t["reg_stats"]), npy(t2["reg_stats"])) and same(npy(t["reg"]), npy(t2["reg"]))          # repeatable to the bit
    for nl, ti in ((1, 6), (5, 8)):
        s = L.test_proposals(f["valid"][keep], [len(o["frames"]) for o in ovids], p["frame_cnt"], nl, ti)
        w = [P.test_proposals(o["frames"], o["frame_cnt"], nl, ti) for o in ovids]
        assert same(npy(s["num_ticks"]), np.array([x[0] for x in w], np.int32))
        for i, k in ((1, "rel_prop"), (2, "proposal_ticks"), (3, "scaling")):
            assert same(npy(s[k]), np.concatenate([x[i] for x in w])), k
        assert s["offsets"] == offsets([max(len(o["frames"]), 1) for o in ovids])


def test_ties_nan_and_inf_coordinates():
    from ops import proposal_lists as L
    nan, inf = float("nan"), float("inf")
    gt = np.array([(2.0, 8.0), (4.0, 10.0), (nan, 5.0), (1.0, nan), (-inf, 3.0), (6.0, inf), (2.0, 8.0), (-inf, inf)])
    boxes = np.array([(3.0, 9.0), (2.0, 8.0), (nan, 4.0), (4.0, nan), (nan, nan), (-inf, 5.0), (0.0, inf), (-inf, inf), (9.0, 1.0)])
    lab = np.arange(len(gt), dtype=np.int32)
    vids = [dict(boxes=boxes, gt=gt, gt_label=lab), dict(boxes=boxes[::-1].copy(), gt=gt[::-1].copy(), gt_label=lab[::-1].copy()),
            dict(boxes=boxes, gt=gt[:2], gt_label=lab[:2])]
    for v in vids:
        v.update(duration=10.0, frame_cnt=300)
    p = pack(vids)
    for thresh in (0.0, 0.5, -1.0):
        r = L.name_proposals_packed(p["boxes"], p["first"], p["count"], p["gt"], p["gt_label"], p["gt_offsets"], thresh)
        named = [P.name_proposals(v["gt"], v["gt_label"], v["boxes"], thresh) for v in vids]
        for i, k in enumerate(("label", "max_overlap", "overlap_self")):
            assert same(npy(r[k]), np.concatenate([n[i] for n in named])), (k, thresh)
        assert same(npy(r["gt_best"]), np.concatenate([P.gt_best_iou(v["gt"], v["boxes"]) for v in vids]))
    # (3, 9) overlaps (2, 8) and (4, 10) by 5 / 7 each: the one that comes first in the video's ground truth is named
    lab = npy(L.name_proposals_packed(p["boxes"], p["first"], p["count"], p["gt"], p["gt_label"], p["gt_offsets"])["label"])
    assert lab[0] == 1 and lab[2 * len(boxes) - 1] == 7 and lab[2 * len(boxes)] == 1


def test_batch_equals_per_video_repeat_and_prefill():
    from ops import proposal_lists as L
    vids = random_batch(2, V=60)
    p = pack(vids)

    def run(q):
        n = L.name_proposals_packed(q["boxes"], q["first"], q["count"], q["gt"], q["gt_label"], q["gt_offsets"])
        f = L.proposal_frames(q["boxes"], q["first"], q["count"], q["frame_cnt"], q["duration"], "seconds")
        return [npy(n[k]) for k in ("label", "max_overlap", "overlap_self", "gt_best")] + [npy(f[k]) for k in ("frames", "valid", "coverage", "keep")]
    whole = run(p)
    parts = [run(pack([v])) for v in vids]
    for i in range(len(whole)):
        assert same(whole[i], np.concatenate([x[i] for x in parts])), i
    # the library calls themselves on outputs pre-filled with 0xFF, in a slot layout with gaps: rows outside every video untouched
    from ssn_b200._lib import lib, check
    import ctypes as C
    cnt = np.array(p["counts"], np.int64)
    first = np.cumsum(cnt + 3) - cnt - 3 + 2
    rows = int(first[-1] + cnt[-1] + 1)
    idx = np.concatenate([np.arange(f, f + c) for f, c in zip(first, cnt)])
    boxes = torch.full((rows, 2), -1.0, dtype=torch.float64, device=dev())
    boxes[T(idx)] = p["boxes"]
    off = p["gt_offsets"]
    outs = [torch.full((rows,), -1, dtype=torch.int32, device=dev())] + [torch.full((rows,), float("nan"), dtype=torch.float64, device=dev()) for _ in range(2)]
    best = torch.full((off[-1],), float("nan"), dtype=torch.float64, device=dev())
    for o in outs + [best]:
        o.view(torch.uint8).fill_(0xFF)
    first_d, off_d = T(first), T(off)
    for max_count in (0, 1, 100000):               # the grid hint does not change the result
        check(lib.ssnb_name_proposals(boxes.data_ptr(), first_d.data_ptr(), p["count"].data_ptr(), len(cnt), max_count, p["gt"].data_ptr(),
                                      p["gt_label"].data_ptr(), (C.c_int64 * len(off))(*off), off_d.data_ptr(), 0.0, outs[0].data_ptr(),
                                      outs[1].data_ptr(), outs[2].data_ptr(), best.data_ptr(), None), None, "name_proposals")
        torch.cuda.synchronize()
        for o, w in zip(outs, whole[:3]):
            assert same(npy(o)[idx], w)
            gap = np.ones(rows, bool)
            gap[idx] = False
            assert (npy(o.view(torch.uint8).view(rows, -1))[gap] == 0xFF).all()
        assert same(npy(best), whole[3])


def test_cuda_graph_replay_on_new_boxes():
    """the library calls captured once on fixed shapes, replayed after new boxes were written, against an eager module call"""
    import ctypes as C
    from ops import proposal_lists as L
    from ssn_b200._lib import lib, check
    a = random_batch(4, V=40)
    b = [dict(v) for v in a]
    for x, y in zip(a, b):                          # same shapes, new coordinates
        n, ng = len(x["boxes"]), len(x["gt"])
        g = np.random.RandomState(n + ng)
        y.update(boxes=np.sort(g.uniform(0, x["duration"], (n, 2)), 1), gt=np.sort(g.uniform(0, x["duration"], (ng, 2)), 1))
    pa, pb = pack(a), pack(b)
    off, V, rows, thr = pa["gt_offsets"], len(a), pa["boxes"].shape[0], [0.5, 0.7]
    off_c, off_d, thr_c = (C.c_int64 * len(off))(*off), T(off), (C.c_double * 2)(*thr)
    dur, fc = T(pa["duration"]), T(pa["frame_cnt"], torch.int32)
    o = dict(label=torch.empty(rows, dtype=torch.int32, device=dev()), max_overlap=torch.empty(rows, dtype=torch.float64, device=dev()),
             overlap_self=torch.empty(rows, dtype=torch.float64, device=dev()), gt_best=torch.empty(max(off[-1], 1), dtype=torch.float64, device=dev()),
             hits=torch.empty(V, 2, dtype=torch.int32, device=dev()), totals=torch.empty(5, dtype=torch.int64, device=dev()),
             frames=torch.empty(rows, 2, dtype=torch.int64, device=dev()))

    def enqueue():
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        check(lib.ssnb_name_proposals(pa["boxes"].data_ptr(), pa["first"].data_ptr(), pa["count"].data_ptr(), V, rows, pa["gt"].data_ptr(),
                                      pa["gt_label"].data_ptr(), off_c, off_d.data_ptr(), 0.0, o["label"].data_ptr(), o["max_overlap"].data_ptr(),
                                      o["overlap_self"].data_ptr(), o["gt_best"].data_ptr(), st), None, "name_proposals")
        check(lib.ssnb_proposal_recall(o["gt_best"].data_ptr(), off_c, off_d.data_ptr(), V, thr_c, 2, o["hits"].data_ptr(), o["totals"].data_ptr(), st),
              None, "proposal_recall")
        check(lib.ssnb_proposal_frames(pa["boxes"].data_ptr(), pa["first"].data_ptr(), pa["count"].data_ptr(), V, rows, dur.data_ptr(), fc.data_ptr(),
                                       0, o["frames"].data_ptr(), None, None, None, st), None, "proposal_frames")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        enqueue()                                   # warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        enqueue()
    pa["boxes"].copy_(pb["boxes"])
    pa["gt"].copy_(pb["gt"])
    for t in o.values():
        t.view(torch.uint8).fill_(0xFF)
    graph.replay()
    torch.cuda.synchronize()
    e = L.label_proposals(pb, pb["gt"], pb["gt_label"], pb["gt_offsets"], pb["duration"], pb["frame_cnt"], thr)
    for k in ("label", "max_overlap", "overlap_self", "frames"):
        assert same(npy(o[k]), npy(e[k])), k
    assert same(npy(o["gt_best"])[:off[-1]], npy(e["gt_best"]))
    assert same(npy(o["hits"]), npy(e["recall"]["hits"])) and same(npy(o["totals"]), npy(e["recall"]["totals"]))
    assert not same(npy(e["max_overlap"]), oracle_name(a)[1])      # the replay did see new boxes


# ---- the chain ----------------------------------------------------------------------------------------------------------------
def test_chain_from_scores_to_test_time_inputs(tmp_path):
    from ops import proposal_lists as L
    from ops.proposals import bottom_up_proposals_packed
    from ops.ssn_ops import STPPReorgainzed
    g = torch.Generator().manual_seed(0)
    Ts = [37, 90, 160, 64, 211]
    durs = [12.0, 30.0, 55.5, 21.3, 70.1]
    fcs = [int(d * 30) for d in durs]
    scores = torch.cat([torch.randn(t, 2, generator=g) * torch.tensor([0.3, 2.0]) for t in Ts]).to(dev())
    tag = bottom_up_proposals_packed(scores, offsets(Ts), durs)
    rs = np.random.RandomState(9)
    gts = [np.sort(rs.uniform(0, d, (n, 2)), 1) for d, n in zip(durs, (2, 0, 4, 1, 3))]
    glab = [rs.randint(0, 20, len(x)).astype(np.int32) for x in gts]
    goff = offsets([len(x) for x in gts])
    r = L.label_proposals(tag, T(np.concatenate(gts)), T(np.concatenate(glab)), goff, durs, fcs)      # reads the slot layout on the device
    dirs = ["frames/v%d" % i for i in range(len(Ts))]
    path = str(tmp_path / "tag_list.txt")
    text = L.write_proposal_list(path, r, dirs)
    # the oracle fed the same kept boxes
    counts, slot0, sec = npy(tag["counts"]), tag["slot0"].numpy(), npy(tag["seconds"])
    assert counts.sum() > 20
    want = ""
    for v in range(len(Ts)):
        boxes = sec[slot0[v]:slot0[v] + counts[v]]
        lab, mo, ms = P.name_proposals(gts[v], glab[v], boxes)
        want += "# {}\n".format(v + 1) + P.format_window_list(dirs[v], fcs[v], glab[v] + 1, P.seconds_to_frames(gts[v], durs[v], fcs[v]), lab, mo, ms,
                                                              P.seconds_to_frames(boxes, durs[v], fcs[v]))
    assert text == want
    rows = L.record_rows(L.load_proposal_list(path))
    ovids = records(text)
    assert rows["counts"] == [len(o["frames"]) for o in ovids] and same(npy(rows["frames"]), np.concatenate([o["frames"] for o in ovids]))
    t = L.proposal_targets(rows["frames"], rows["best_iou"], rows["overlap_self"], rows["coverage"], rows["first"], rows["count"], rows["gt_frames"],
                           rows["gt_offsets"], fg_iou_thresh=0.5)
    out, stats, totals = P.proposal_targets(ovids, fg_thresh=0.5)
    assert same(npy(t["tags"]), np.concatenate([o["tags"] for o in out])) and npy(t["totals"]).tolist() == totals
    s = L.test_proposals(rows["frames"], rows["counts"], rows["frame_cnt"])
    w = [P.test_proposals(o["frames"], o["frame_cnt"]) for o in ovids]
    assert same(npy(s["proposal_ticks"]), np.concatenate([x[2] for x in w])) and same(npy(s["scaling"]), np.concatenate([x[3] for x in w]))
    # the test-time tail takes video 2's tick / scaling tensors as produced
    v = 2
    lo, hi = s["offsets"][v], s["offsets"][v + 1]
    K = 4
    reorg = STPPReorgainzed(K + 1 + 3 * K + 3 * 2 * K, K + 1, K, 2 * K, standalong_classifier=True, with_regression=True, stpp_cfg=(1, 1, 1))
    frame_scores = torch.randn(int(s["num_ticks"][v]), reorg.feat_dim, generator=g).to(dev())
    got = reorg.forward(frame_scores, s["proposal_ticks"][lo:hi], s["scaling"][lo:hi])
    ref = reorg.forward(frame_scores, torch.from_numpy(w[v][2]), torch.from_numpy(w[v][3]))
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    assert s["ticks32"].dtype == torch.int32 and s["scaling32"].dtype == torch.float32 and s["ticks32"].is_contiguous()
    assert torch.equal(s["ticks32"], s["proposal_ticks"].to(torch.int32)) and torch.equal(s["scaling32"], s["scaling"].to(torch.float32))
