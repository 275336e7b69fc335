"""Staged check of one `bottom_up_proposals_packed(..., trace=True)` result.  TEST INFRASTRUCTURE ONLY.

For every video, each oracle stage of oracle/proposal_oracle.py is fed what the kernel before it wrote, so a wrong stage is
named by the first check that fails, not by everything downstream of it:
  1 smoothed  the softmax column smoothed by scipy's Gaussian, against a float64 restatement (float64 softmax of the fp32
              scores, float64 Gaussian with scipy's weights): 1e-6 absolute, NaN positions equal;
  2 labels    every label bit against gpu_smoothed > fp32(threshold), exactly; a tick where the GPU's label differs from
              the oracle's own fp32 label must lie within 1e-6 of its threshold (CUDA's expf and numpy's exp may differ by
              an ulp), and is counted;
  3 raw       build_boxes on the GPU's label rows and the raw column f[:, cls + 1] against raw_frames / raw_scores /
              raw_counts, in search order, bitwise (NaN scores: positions, not bits);
  4 nms       temporal_nms on the GPU's own raw boxes: the kept boxes, in order, with their scores, are the survivors
              less those that fail the minimum-length filter;
  5 filter    every kept box passes the filter, `seconds` is start / float(T) * duration in double bitwise, and counts;
  6 e2e       where no label flipped and stages 1-5 passed, gen_prop on the raw input equals the output bitwise.
`Checker` records each check as (stage, quantity, video, first mismatch).

Also here: the score generators of the GPU check (the smooth / noisy families of oracle/gen_golden_proposals.py and the
sinusoid family of tools/bench_proposals.py restated, plus exact run counts, quantised and zero foreground columns, NaN and
inf), random NMS cases for the oracle-vs-reference test, and a numpy stand-in that fills the wrapper's trace layout from
the oracle, with hooks that plant one error at one stage.
"""
import numpy as np

from . import proposal_oracle as P

SMOOTH_BAR = 1e-6        # absolute, smoothed column vs float64 (the golden bar)
LABEL_BAND = 1e-6        # a label may differ from the oracle's fp32 label only this close to its threshold
STAGES = ("smoothed", "labels", "raw", "nms", "filter", "e2e")
NAN_BITS = (0x7fc00000, 0xffc00000, 0xff800123, 0x7fffffff)     # +NaN, -NaN, a negative signalling NaN, CUDA's NaN

# 32 thresholds / tolerances with the edges the defaults never reach: 0, 1, negative values, duplicates (label bit 31);
# tolerance 0, 0.5, 1 (exact signal ties on regular runs), 1.3 and -0.2
THR32 = (0.0, 1.0, -0.25, 0.5, 0.5, 0.01, 0.95, 0.3, 0.3, 0.7, 0.05, 0.1, 0.15, 0.2, 0.25, 0.35, 0.4, 0.45, 0.55, 0.6, 0.65,
         0.75, 0.8, 0.85, 0.9, 0.99, 0.999, 1e-4, 0.125, 0.625, 0.875, 0.7)
TOL32 = (0.0, 0.5, 1.0, 1.3, -0.2, 0.05, 0.1, 0.2, 0.3, 0.4, 0.6, 0.8, 0.25, 0.75, 0.9, 1.1, 1.5, 2.0, 0.01, 0.15, 0.35,
         0.45, 0.55, 0.65, 0.7, 0.85, 0.95, 1.2, 3.0, -0.5, 0.5, 1.0)


# ---- score generators: [T, K] fp32, column fg = cls + 1 is the foreground logit ------------------------------------------
def _base(T, g, K):
    return (g.randn(T, K) * 0.3).astype(np.float32)


def _walk(T, g):
    """gen_golden_proposals.synth_logits 'smooth': a random walk less its 301-tick running mean, plus noise"""
    walk = np.cumsum(g.randn(T)) * 0.35
    walk -= np.convolve(walk, np.ones(min(T, 301)) / min(T, 301), mode="same")
    return walk + 0.4 * g.randn(T)


def run_labels(T, U, g, regular=False, end_fg=False):
    """bool [T] with exactly U foreground runs (T >= 2U - 1).  regular: runs and gaps of one length L after a leading gap,
    so that signal[up] ties at tolerance 0.5; end_fg: the last tick is foreground"""
    lab = np.zeros(T, bool)
    if U == 0:
        return lab
    if regular:
        L = max(1, T // (2 * U))
        lead = T - (2 * U - 1) * L if end_fg else max(0, T - 2 * U * L)
        for u in range(U):
            lab[lead + 2 * u * L: lead + 2 * u * L + L] = True
        return lab
    fg = int(g.randint(U, T - (U - 1) + 1))
    runs = 1 + g.multinomial(fg - U, np.ones(U) / U)
    extra = T - fg - (U - 1)
    gaps = g.multinomial(extra, np.ones(U + 1) / (U + 1))
    if end_fg:
        gaps[0] += gaps[U]
        gaps[U] = 0
    gaps[1:U] += 1
    t = 0
    for u in range(U):
        t += gaps[u]
        lab[t:t + runs[u]] = True
        t += runs[u]
    return lab


def make_scores(kind, T, g, K=2, cls=0, U=None, end_fg=False):
    f = _base(T, g, K)
    fg = cls + 1
    if kind == "smooth":
        f[:, fg] += _walk(T, g).astype(np.float32)
    elif kind == "noisy":                               # gen_golden_proposals.synth_logits 'noisy'
        f[:, fg] += (np.cumsum(g.randn(T)) * 0.05 + 7.0 * g.randn(T)).astype(np.float32)
    elif kind == "sinus":                               # tools/bench_proposals.synth_dataset, smooth
        x = np.arange(T)
        s = sum(g.uniform(1.0, 2.5) * np.sin(2 * np.pi * x / g.uniform(150, 900) + g.uniform(0, 6.3)) for _ in range(3))
        f[:, fg] += (s + g.randn(T) * 0.4).astype(np.float32)
    elif kind in ("runs", "runs_regular"):              # exactly U runs at every threshold in [0.01, 0.95] with bw None
        U = max(1, T // 16) if U is None else U
        lab = run_labels(T, U, g, regular=kind == "runs_regular", end_fg=end_fg)
        if kind == "runs_regular":                      # integer logits: box scores tie as well as signals
            f[:] = 0.0
            f[:, fg] = np.where(lab, 9.0, -9.0)
        else:
            f[:, fg] = np.where(lab, 9.0, -9.0) + (g.randn(T) * 0.5).astype(np.float32)
    elif kind == "quant":                               # multiples of 0.25, small-integer raw column: many tied boxes
        f = np.round(f * 4) / 4
        f[:, fg] = np.clip(np.round(_walk(T, g) * 1.5), -3, 3)
    elif kind == "zero_fg":                             # every box scores 0: NMS order is the search order
        f[:, fg] = 0.0
        f[:, 0] = -(_walk(T, g) * 1.5).astype(np.float32)
    elif kind in ("nan", "nan_bg", "inf", "neginf_row"):
        f[:, fg] += _walk(T, g).astype(np.float32)
        n = max(1, T // 97)
        ticks = g.choice(T, size=min(n, T), replace=False)
        if kind == "nan":                               # NaN of either sign, preferably at background ticks
            bg = np.nonzero(f[:, fg] < -0.5)[0]
            if len(bg) >= len(ticks):
                ticks = g.choice(bg, size=len(ticks), replace=False)
            bits = f.view(np.uint32)
            bits[ticks, fg] = np.array(NAN_BITS, np.uint32)[g.randint(0, len(NAN_BITS), len(ticks))]
        elif kind == "nan_bg":                          # NaN in a column that is not the foreground
            f[ticks, 0 if fg != 0 else 1] = np.float32("nan")
        elif kind == "inf":
            f[ticks, fg] = np.where(g.rand(len(ticks)) < 0.5, np.inf, -np.inf).astype(np.float32)
        else:
            f[ticks[:1], :] = -np.inf
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(f, np.float32)


def pack(videos):
    """[(f [T, K], duration)] -> (packed f, offsets, durations)"""
    offsets = [0]
    for f, _ in videos:
        offsets.append(offsets[-1] + len(f))
    return np.concatenate([f for f, _ in videos]), offsets, [float(d) for _, d in videos]


# ---- float64 restatement of stage 1 --------------------------------------------------------------------------------------
def smooth64(f, cls=0, bw=3):
    """float64 softmax column of the fp32 scores, then scipy's Gaussian ('reflect', truncate 4.0) in float64"""
    with np.errstate(invalid="ignore", over="ignore"):
        x = np.asarray(f, np.float64)
        e = np.exp(x - x.max(axis=1, keepdims=True))
        col = e[:, cls + 1] / e.sum(axis=1)
    if bw is None or len(col) == 0:
        return col
    w = P.gaussian_weights(bw)
    r = (len(w) - 1) // 2
    i = np.arange(len(col))
    acc = col * w[r]
    for j in range(r, 0, -1):
        acc = acc + (col[P.reflect_index(i - j, len(col))] + col[P.reflect_index(i + j, len(col))]) * w[r + j]
    return acc


# ---- comparator ------------------------------------------------------------------------------------------------------------
class Record:
    def __init__(self, stage, quantity, video, mismatch):
        self.stage, self.quantity, self.video, self.mismatch = stage, quantity, video, mismatch

    @property
    def ok(self):
        return self.mismatch is None

    def __repr__(self):
        return "%s %s video %d: %s" % (self.stage, self.quantity, self.video, "ok" if self.ok else self.mismatch)


class Checker:
    """records (stage, quantity, video, first mismatch or None) and the counts the GPU test prints"""

    def __init__(self):
        self.records = []
        self.stats = dict(videos=0, raw_boxes=0, tied_boxes=0, nan_boxes=0, kept=0, flips_in_band=0, e2e_videos=0,
                          worst_smoothed=0.0)

    def add(self, stage, quantity, video, mismatch):
        self.records.append(Record(stage, quantity, video, mismatch))
        return mismatch is None

    def failures(self):
        return [r for r in self.records if not r.ok]

    def failed(self):
        return {r.stage for r in self.failures()}

    def report(self):
        s = self.stats
        return ("%d videos, %d raw boxes (%d tied, %d NaN), %d kept, %d label flips inside the band, worst smoothed error "
                "%.2e, end to end on %d videos" % (s["videos"], s["raw_boxes"], s["tied_boxes"], s["nan_boxes"], s["kept"],
                                                   s["flips_in_band"], s["worst_smoothed"], s["e2e_videos"]))

    def assert_ok(self):
        bad = self.failures()
        assert not bad, "proposal check failed at:\n" + "\n".join(map(repr, bad[:20]))


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def _first(mask):
    i = np.nonzero(mask)[0]
    return int(i[0]) if len(i) else None


def _same_scores(a, b):
    """fp32 arrays equal bit for bit, a NaN equal to any NaN -> index of the first difference or None"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return _first((na != nb) | (~na & (a.view(np.uint32) != b.view(np.uint32))))


def _seconds(s, e, T, duration):
    s, e = np.asarray(s, np.int64), np.asarray(e, np.int64)
    return np.stack([s / float(T) * duration, e / float(T) * duration], axis=1) if len(s) else np.zeros((0, 2))


def check(res, f, offsets, durations, cls=0, bw=3, thresholds=P.THRESHOLDS, tolerances=P.TOLERANCES, nms_threshold=0.9,
          minimum_len=0.0, chk=None, e2e=True):
    """every video of one traced call (res: the wrapper's dict, or the stand-in's) against the oracle, stage by stage"""
    chk = Checker() if chk is None else chk
    f = _np(f)
    r = {k: _np(v) for k, v in res.items()}
    labels_all = r["labels"].view(np.uint32)
    thr32 = [np.float32(t) for t in thresholds]
    n_thr = len(thresholds)
    for v in range(len(offsets) - 1):
        lo, hi = offsets[v], offsets[v + 1]
        T, fv, dur = hi - lo, f[lo:hi], float(durations[v])
        slot0 = int(r["slot0"][v])
        chk.stats["videos"] += 1
        ok = True
        # 1 smoothed
        got_sm = r["smoothed"][lo:hi]
        ref_sm = smooth64(fv, cls, bw)
        ok &= chk.add("smoothed", "nan positions", v, None if (np.isnan(got_sm) == np.isnan(ref_sm)).all() else
                      "tick %d" % _first(np.isnan(got_sm) != np.isnan(ref_sm)))
        fin = ~np.isnan(ref_sm) & ~np.isnan(got_sm)
        err = np.abs(got_sm[fin].astype(np.float64) - ref_sm[fin])
        worst = float(err.max()) if err.size else 0.0
        chk.stats["worst_smoothed"] = max(chk.stats["worst_smoothed"], worst)
        ok &= chk.add("smoothed", "value", v, None if worst <= SMOOTH_BAR else
                      "%.3e at tick %d" % (worst, np.nonzero(fin)[0][int(err.argmax())]))
        # 2 labels
        lab = np.stack([((labels_all[lo:hi] >> k) & 1).astype(bool) for k in range(n_thr)]) if T else np.zeros((n_thr, 0), bool)
        want = np.stack([got_sm > t for t in thr32])
        bad = np.argwhere(lab != want)
        ok &= chk.add("labels", "bits", v, None if not len(bad) else "threshold %d tick %d" % tuple(bad[0]))
        own = P.frame_labels(fv, cls, bw, thresholds)[2]
        flips = np.argwhere(lab != own)
        out = [(k, t) for k, t in flips if not abs(ref_sm[t] - float(thr32[k])) <= LABEL_BAND]
        ok &= chk.add("labels", "flips outside the band", v, None if not out else "threshold %d tick %d" % out[0])
        chk.stats["flips_in_band"] += len(flips) - len(out)
        # 3 raw boxes, from the GPU's label rows
        frm = fv[:, cls + 1]
        parts = [P.build_boxes(row, frm, tolerances) for row in lab]
        s, e, sc = (np.concatenate([p[k] for p in parts]) for k in range(3))
        n_raw = int(r["raw_counts"][v])
        chk.stats["raw_boxes"] += len(s)
        nan = np.isnan(sc)
        chk.stats["nan_boxes"] += int(nan.sum())
        if len(s):                                      # boxes whose score another box with other frames shares
            key = np.where(sc[~nan] == 0, 0, sc.view(np.uint32)[~nan]).astype(np.int64)
            distinct = np.unique(np.stack([key, s[~nan], e[~nan]], axis=1), axis=0)
            k, cnt = np.unique(distinct[:, 0], return_counts=True)
            chk.stats["tied_boxes"] += int(np.isin(key, k[cnt > 1]).sum())
        if n_raw != len(s):
            ok &= chk.add("raw", "count", v, "%d boxes, oracle %d" % (n_raw, len(s)))
        else:
            rf = r["raw_frames"][slot0:slot0 + n_raw].astype(np.int64)
            i = _first((rf[:, 0] != s) | (rf[:, 1] != e)) if n_raw else None
            ok &= chk.add("raw", "frames", v, None if i is None else "box %d: (%d, %d), oracle (%d, %d)" % (
                i, rf[i, 0], rf[i, 1], s[i], e[i]))
            rs = r["raw_scores"][slot0:slot0 + n_raw]
            i = _same_scores(rs, sc)
            ok &= chk.add("raw", "scores", v, None if i is None else "box %d: %r, oracle %r" % (i, rs[i], sc[i]))
        # 4 NMS on the GPU's own raw boxes
        n_out = int(r["counts"][v])
        chk.stats["kept"] += n_out
        gs = r["raw_frames"][slot0:slot0 + n_raw].astype(np.int64)
        gsc = r["raw_scores"][slot0:slot0 + n_raw]
        keep = P.temporal_nms(gs[:, 0], gs[:, 1], gsc, nms_threshold) if n_raw else np.zeros(0, np.int64)
        ks, ke, ksc = gs[keep, 0], gs[keep, 1], gsc[keep]
        ksec = _seconds(ks, ke, T, dur)
        passes = ksec[:, 1] - ksec[:, 0] > minimum_len
        of = r["frames"][slot0:slot0 + n_out].astype(np.int64)
        osc = r["scores"][slot0:slot0 + n_out]
        where = {(a, b): j for j, (a, b) in enumerate(zip(ks.tolist(), ke.tolist()))}
        mism, last, matched = None, -1, []
        for i in range(n_out):
            j = where.get((int(of[i, 0]), int(of[i, 1])))
            if j is None or j <= last:
                mism = "kept box %d (%d, %d) is not the next survivor" % (i, of[i, 0], of[i, 1])
                break
            if _same_scores(osc[i:i + 1], ksc[j:j + 1]) is not None:
                mism = "kept box %d: score %r, oracle %r" % (i, osc[i], ksc[j])
                break
            skipped = [x for x in range(last + 1, j) if passes[x]]
            if skipped:
                mism = "survivor %d (%d, %d) is missing before kept box %d" % (skipped[0], ks[skipped[0]], ke[skipped[0]], i)
                break
            matched.append(j)
            last = j
        if mism is None:
            rest = [x for x in range(last + 1, len(ks)) if passes[x]]
            if rest:
                mism = "survivor %d (%d, %d) is missing at the end" % (rest[0], ks[rest[0]], ke[rest[0]])
        ok &= chk.add("nms", "survivors", v, mism)
        # 5 seconds, length filter, counts
        osec = r["seconds"][slot0:slot0 + n_out]
        want_sec = _seconds(of[:, 0], of[:, 1], T, dur)
        i = _first((osec.view(np.uint64) != want_sec.view(np.uint64)).any(axis=1)) if n_out else None
        ok &= chk.add("filter", "seconds", v, None if i is None else "box %d: %r, oracle %r" % (i, osec[i], want_sec[i]))
        fails = _first(~(want_sec[:, 1] - want_sec[:, 0] > minimum_len)) if n_out else None
        ok &= chk.add("filter", "kept box fails the filter", v, None if fails is None else "box %d" % fails)
        if mism is None and fails is None:
            ok &= chk.add("filter", "count", v, None if n_out == int(passes.sum()) else "%d, oracle %d" % (n_out, passes.sum()))
        # 6 end to end, where nothing flipped and nothing failed upstream
        if e2e and ok and not len(flips):
            g = P.gen_prop(fv, dur, cls, bw, thresholds, tolerances, nms_threshold, minimum_len)
            same = (len(g["pr_frames"]) == n_out and (g["pr_frames"] == of).all() and _same_scores(g["pr_score"], osc) is None
                    and (g["pr_box"].view(np.uint64) == osec.view(np.uint64)).all())
            chk.add("e2e", "gen_prop", v, None if same else "%d boxes, gen_prop %d" % (n_out, len(g["pr_frames"])))
            chk.stats["e2e_videos"] += 1
    return chk


# ---- numpy stand-in of the traced call, with planted errors --------------------------------------------------------------
def standin(f, offsets, durations, cls=0, bw=3, thresholds=P.THRESHOLDS, tolerances=P.TOLERANCES, nms_threshold=0.9,
            minimum_len=0.0, plant=None):
    """the wrapper's trace layout filled from the oracle.  plant(stage, v, x) -> x may alter one stage's output of video v
    before the next stage reads it: 'labels' (bool [n_thr, T]), 'raw' ((start, end, score)), 'nms' (the NMS function),
    'kept' ((keep indices, passes mask)), 'seconds' ([n, 2])"""
    plant = plant or (lambda stage, v, x: x)
    f = np.asarray(f, np.float32)
    V, N, n_thr, n_tol = len(offsets) - 1, offsets[-1], len(thresholds), len(tolerances)
    slots = max(n_thr * n_tol * (N + V), 1)
    out = {"frames": np.zeros((slots, 2), np.int32), "scores": np.zeros(slots, np.float32),
           "seconds": np.zeros((slots, 2), np.float64), "counts": np.zeros(V, np.int32),
           "slot0": np.array([n_thr * n_tol * (offsets[v] + v) for v in range(V)], np.int64),
           "smoothed": np.zeros(max(N, 1), np.float32), "labels": np.zeros(max(N, 1), np.uint32),
           "raw_frames": np.zeros((slots, 2), np.int32), "raw_scores": np.zeros(slots, np.float32),
           "raw_counts": np.zeros(V, np.int32)}
    for v in range(V):
        lo, hi = offsets[v], offsets[v + 1]
        T, fv, s0 = hi - lo, f[lo:hi], int(out["slot0"][v])
        _, sm, lab = P.frame_labels(fv, cls, bw, thresholds)
        lab = plant("labels", v, lab.copy())
        out["smoothed"][lo:hi] = sm
        out["labels"][lo:hi] = sum((lab[k].astype(np.uint32) << np.uint32(k)) for k in range(n_thr))
        parts = [P.build_boxes(row, fv[:, cls + 1], tolerances) for row in lab]
        s, e, sc = plant("raw", v, tuple(np.concatenate([p[k] for p in parts]) for k in range(3)))
        n = len(s)
        out["raw_counts"][v] = n
        out["raw_frames"][s0:s0 + n] = np.stack([s, e], axis=1) if n else np.zeros((0, 2))
        out["raw_scores"][s0:s0 + n] = sc
        keep = plant("nms", v, P.temporal_nms)(s, e, sc, nms_threshold) if n else np.zeros(0, np.int64)
        sec = _seconds(s[keep], e[keep], T, float(durations[v]))
        keep, ok = plant("kept", v, (keep, sec[:, 1] - sec[:, 0] > minimum_len))
        sec = plant("seconds", v, _seconds(s[keep], e[keep], T, float(durations[v]))[ok])
        k = keep[ok]
        out["counts"][v] = len(k)
        out["frames"][s0:s0 + len(k)] = np.stack([s[k], e[k]], axis=1) if len(k) else np.zeros((0, 2))
        out["scores"][s0:s0 + len(k)] = sc[k]
        out["seconds"][s0:s0 + len(k)] = sec
    out["labels"] = out["labels"].view(np.int32)
    return out


# ---- random NMS cases (oracle vs the reference's temporal_nms_fallback) --------------------------------------------------
def nms_cases(seed, n_cases=24):
    """[(start int64 [n], end int64 [n], score fp32 [n], thresh)]: pairwise distinct finite scores plus one NaN, +inf and
    -inf, and pairs of boxes whose IoU is exactly the threshold (0.5, 0.25 or 0.75, all exact in double)"""
    g = np.random.RandomState(seed)
    cases = []
    for c in range(n_cases):
        n = int(g.randint(2, 60))
        s = g.randint(0, 200, n).astype(np.int64)
        e = s + g.randint(0, 40, n)
        thresh = (0.5, 0.25, 0.75, 0.0, 0.9)[c % 5]
        if thresh in (0.5, 0.25, 0.75):          # (a, a + 4k - 1) and (a, a + 4k * thresh - 1): IoU = thresh
            for _ in range(3):
                a, k = int(g.randint(0, 200)), int(g.randint(1, 6))
                s = np.append(s, [a, a])
                e = np.append(e, [a + 4 * k - 1, a + int(4 * k * thresh) - 1])
        sc = (g.permutation(len(s) * 4)[:len(s)].astype(np.float32) - 2.0 * len(s)) / np.float32(8)
        specials = g.choice(len(s), size=min(3, len(s)), replace=False)
        sc[specials] = np.array([np.nan, np.inf, -np.inf], np.float32)[:len(specials)]
        cases.append((s, e, sc, thresh))
    return cases
