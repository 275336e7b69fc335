"""Staged check of one traced `detections_packed` + `detection_ap` result.  TEST INFRASTRUCTURE ONLY.

Each stage is fed what the kernel before it wrote, so a wrong stage is named by the first check that fails:
  1 combined  the ranked scores [sum N, K] against the branch in float64 (combined64 for softmax(act)[:, 1:] * exp(comp)),
              per proposal (row), COMBINED_BAR, NaN positions equal;
  2 select    the selected pairs of every video, in ranking order, against the oracle's selection from the GPU's own
              combined scores: exact;
  3 nms       per (video, class), nms64 over the GPU's selection of that class in its order: the survivors' (score, loc,
              dur) in kept order and the counts, exact;
  4 boxes     the survivors' boxes against regress64 of their proposals (or the proposals themselves without regression),
              REGRESS_BAR per (video, class);
  5 rank      every survivor's class-wide rank, exact      } eval_oracle.average_precision fed the GPU's survivors
  6 tp        the tp / fp flags per threshold, exact       }
  7 ap        the AP table within AP_BAR, NaN equal        }
`Checker` records (stage, where, first mismatch).  `standin` fills the same dict from the oracle, with a hook that plants an
error into one stage's output before the next stage reads it.
"""
import numpy as np
import torch

from . import eval_oracle as D
from .infer_check import combined64, nms64, regress64, nms_order, COMBINED_BAR, REGRESS_BAR

AP_BAR = 1e-12
STAGES = ("combined", "select", "nms", "boxes", "rank", "tp", "ap")


class Checker:
    def __init__(self):
        self.records = []
        self.stats = dict(videos=0, selected=0, kept=0, worst_combined=0.0, worst_boxes=0.0, worst_ap=0.0)

    def add(self, stage, where, mismatch):
        self.records.append((stage, where, mismatch))
        return mismatch is None

    def failures(self):
        return [r for r in self.records if r[2] is not None]

    def failed(self):
        return {r[0] for r in self.failures()}

    def assert_ok(self):
        bad = self.failures()
        assert not bad, "detection check failed at:\n" + "\n".join("%s %s: %s" % r for r in bad[:20])


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def combined_ref(act, comp, mode, softmax_before_filter=True):
    """float64 combined scores of a branch"""
    a, c = torch.as_tensor(np.asarray(act, np.float64)), torch.as_tensor(np.asarray(comp, np.float64))
    if mode == "top_k":
        return (torch.softmax(a[:, 1:], 1) * torch.exp(c)).numpy()
    if mode == "cls" and not softmax_before_filter:
        return (a[:, 1:] * torch.exp(c)).numpy()
    return combined64(a, c).numpy()


def selection(comb_v, row0, mode, top_k=None, classes=None):
    """the selected pairs (global row * K + class) of one video in ranking order: NaN first, descending, equal scores the
    larger candidate index first; top_k keeps the first min(top_k, N K)"""
    n, K = comb_v.shape
    if mode == "cls":
        cls = np.asarray(classes, np.int64)
        p = np.repeat(np.arange(n), len(cls))
        c = np.tile(cls, n)
    else:
        p, c = np.divmod(np.arange(n * K), K)
    order = nms_order(comb_v[p, c]) if len(p) else np.zeros(0, np.int64)
    if mode == "top_k":
        order = order[:top_k]
    return (row0 + p[order]) * K + c[order]


def check(res, ap_res, props, act, comp, reg, offsets, mode, nms_threshold, gt, thresholds, top_k=None, cls_sel=None,
          softmax_before_filter=True, regress=True, classes=None, chk=None):
    """res: detections_packed(trace=True); ap_res: detection_ap(trace=True); gt: pack_ground_truth's dict.  classes: the
    classes stages 5-7 cover (default all)."""
    chk = Checker() if chk is None else chk
    r = {k: (_np(v) if k != "slot0" else list(v)) for k, v in res.items() if k != "slot0_dev"}
    props = np.asarray(_np(props), np.float32).reshape(-1, 2)
    comp = _np(comp)
    N, K = comp.shape
    reg = np.zeros((N, K, 2), np.float32) if reg is None else _np(reg).reshape(N, K, 2)
    V = len(offsets) - 1
    comb = r["combined"][:N]
    # 1 combined
    ref = combined_ref(_np(act), comp, mode, softmax_before_filter)
    nan_ok = (np.isnan(comb) == np.isnan(ref)).all()
    chk.add("combined", "nan positions", None if nan_ok else "row %d" % np.argwhere(np.isnan(comb) != np.isnan(ref))[0][0])
    fin = np.isfinite(ref) & np.isfinite(comb)
    d = np.where(fin, np.abs(comb.astype(np.float64) - ref), 0.0).max(axis=1) if N else np.zeros(0)
    s = np.where(fin, np.abs(ref), 0.0).max(axis=1) if N else np.zeros(0)
    err = np.where(s > 0, d / np.where(s > 0, s, 1), d)
    worst = float(err.max()) if N else 0.0
    chk.stats["worst_combined"] = max(chk.stats["worst_combined"], worst)
    chk.add("combined", "value", None if worst <= COMBINED_BAR else "%.3e at row %d" % (worst, int(err.argmax())))
    slot0, counts, dets, sel = r["slot0"], r["counts"], r["dets"], r["sel"]
    for v in range(V):
        chk.stats["videos"] += 1
        lo, hi, s0, s1 = offsets[v], offsets[v + 1], slot0[v], slot0[v + 1]
        # 2 select
        want = selection(comb[lo:hi], lo, mode, top_k, None if cls_sel is None else np.asarray(cls_sel)[v])
        got = sel[s0:s1]
        chk.stats["selected"] += len(got)
        i = None if (len(got) == len(want) and (got == want).all()) else (
            int(np.argmax(got[:min(len(got), len(want))] != want[:min(len(got), len(want))])) if len(got) == len(want) else -1)
        chk.add("select", "video %d" % v, None if i is None else "pair %d: %s, oracle %s" % (
            i, got[i] if i >= 0 else len(got), want[i] if i >= 0 else len(want)))
        # 3 nms and 4 boxes on the GPU's selection
        at = s0
        for c in range(K):
            m = got[(got % K) == c] if len(got) else got
            rows = m // K
            n = int(counts[v, c])
            kept = rows[nms64(props[rows], comb[rows, c], nms_threshold, order=np.arange(len(rows)))] if len(rows) else rows
            chk.stats["kept"] += n
            out = dets[at:at + n]
            want_f = np.stack([comb[kept, c], reg[kept, c, 0], reg[kept, c, 1]], 1) if len(kept) else np.zeros((0, 3), np.float32)
            same = n == len(kept) and np.array_equal(out[:, 2:].view(np.uint32), want_f.astype(np.float32).view(np.uint32)) or (
                n == len(kept) and np.array_equal(out[:, 2:], want_f, equal_nan=True))
            chk.add("nms", "video %d class %d" % (v, c), None if same else "%d survivors, oracle %d" % (n, len(kept)))
            if same and n:
                bref = regress64(props[kept], reg[kept, c, 0], reg[kept, c, 1]).numpy() if regress else props[kept].astype(np.float64)
                e = np.abs(out[:, :2].astype(np.float64) - bref).max() / max(np.abs(bref).max(), 1e-30)
                chk.stats["worst_boxes"] = max(chk.stats["worst_boxes"], float(e))
                chk.add("boxes", "video %d class %d" % (v, c), None if e <= REGRESS_BAR else "%.3e" % e)
            at += n
    # 5-7 the AP stage on the GPU's survivors
    a = {k: _np(x) for k, x in ap_res.items()}
    goff, gcls, gseg = gt["offsets"], _np(gt["cls"]), _np(gt["seg"])
    gvid = np.full(len(gcls), -1, np.int64)
    for v in range(V):
        gvid[goff[v]:goff[v + 1]] = v
    for c in (range(K) if classes is None else classes):
        slots, pv = [], []
        for v in range(V):
            pre = slot0[v] + int(counts[v, :c].sum())
            slots += list(range(pre, pre + int(counts[v, c])))
            pv += [v] * int(counts[v, c])
        slots = np.asarray(slots, np.int64)
        g = gcls == c
        ap, rank, tp = D.average_precision(gvid[g], gseg[g], pv, dets[slots, :2].astype(np.float64), dets[slots, 2].astype(np.float64),
                                           thresholds, trace=True)
        ok = np.array_equal(a["rank"][slots], rank)
        chk.add("rank", "class %d" % c, None if ok else "first at survivor %d" % int(np.argmax(a["rank"][slots] != rank)))
        ok = np.array_equal(a["tp"][:, slots], tp)
        chk.add("tp", "class %d" % c, None if ok else "threshold / survivor %s" % (np.argwhere(a["tp"][:, slots] != tp)[0],))
        gap = a["ap"][c]
        bad = ~((np.isnan(gap) & np.isnan(ap)) | (np.abs(gap - ap) <= AP_BAR))
        diff = np.where(np.isnan(gap) | np.isnan(ap), 0.0, np.abs(gap - ap))
        chk.stats["worst_ap"] = max(chk.stats["worst_ap"], float(diff.max()) if len(diff) else 0.0)
        chk.add("ap", "class %d" % c, None if not bad.any() else "threshold %d: %r, oracle %r" % (
            int(np.argmax(bad)), gap[np.argmax(bad)], ap[np.argmax(bad)]))
    return chk


def standin(props, act, comp, reg, offsets, mode, nms_threshold, gt, thresholds, top_k=None, cls_sel=None, softmax_before_filter=True,
            regress=True, plant=None):
    """(res, ap_res) in the wrapper's layouts, computed by the numpy oracle.  plant(stage, x) -> x may alter 'combined',
    'sel', 'dets' (after NMS, before regression: the [S, 5] rows, counts), 'boxes', 'rank', 'tp' or 'ap' before the next stage
    reads it"""
    plant = plant or (lambda stage, x: x)
    props = np.asarray(props, np.float32).reshape(-1, 2)
    act, comp = np.asarray(act, np.float32), np.asarray(comp, np.float32)
    N, K = comp.shape
    regz = np.zeros((N, K, 2), np.float32) if reg is None else np.asarray(reg, np.float32).reshape(N, K, 2)
    V = len(offsets) - 1
    comb = plant("combined", np.concatenate([D.branch_scores(act[offsets[v]:offsets[v + 1]], comp[offsets[v]:offsets[v + 1]], mode,
                                                             softmax_before_filter) for v in range(V)]).astype(np.float32))
    sels = [selection(comb[offsets[v]:offsets[v + 1]], offsets[v], mode, top_k, None if cls_sel is None else np.asarray(cls_sel)[v])
            for v in range(V)]
    slot0 = [0]
    for s in sels:
        slot0.append(slot0[-1] + len(s))
    sel = plant("sel", np.concatenate(sels).astype(np.int32))
    dets = np.zeros((max(slot0[-1], 1), 5), np.float32)
    counts = np.zeros((V, K), np.int32)
    for v in range(V):
        got = sel[slot0[v]:slot0[v + 1]]
        at = slot0[v]
        for c in range(K):
            rows = got[(got % K) == c] // K
            kept = rows[nms64(props[rows], comb[rows, c], nms_threshold, order=np.arange(len(rows)))] if len(rows) else rows
            dets[at:at + len(kept)] = np.stack([props[kept, 0], props[kept, 1], comb[kept, c], regz[kept, c, 0], regz[kept, c, 1]], 1)
            counts[v, c] = len(kept)
            at += len(kept)
    dets, counts = plant("dets", (dets, counts))
    if regress:
        n = slot0[-1]
        dets[:n, :2] = D.perform_regression(dets[:n])[:, :2]
    dets = plant("boxes", dets)
    res = {"combined": comb, "sel": sel, "dets": dets, "counts": counts, "slot0": slot0}
    goff, gcls, gseg = gt["offsets"], _np(gt["cls"]), _np(gt["seg"])
    gvid = np.full(len(gcls), -1, np.int64)
    for v in range(V):
        gvid[goff[v]:goff[v + 1]] = v
    S = max(slot0[-1], 1)
    rank_all, tp_all = np.full(S, -1, np.int32), np.zeros((len(thresholds), S), np.uint8)
    ap_all = np.zeros((K, len(thresholds)))
    for c in range(K):
        slots, pv = [], []
        for v in range(V):
            pre = slot0[v] + int(counts[v, :c].sum())
            slots += list(range(pre, pre + int(counts[v, c])))
            pv += [v] * int(counts[v, c])
        slots = np.asarray(slots, np.int64)
        g = gcls == c
        ap, rank, tp = D.average_precision(gvid[g], gseg[g], pv, dets[slots, :2].astype(np.float64), dets[slots, 2].astype(np.float64),
                                           thresholds, trace=True)
        rank_all[slots], tp_all[:, slots], ap_all[c] = rank, tp, ap
    return res, {"rank": plant("rank", rank_all), "tp": plant("tp", tp_all), "ap": plant("ap", ap_all)}
