"""CPU restatement (numpy) of TAG bottom-up proposal generation — TEST INFRASTRUCTURE ONLY (tests/, smoke() and the
benchmarks may import it; the product never does).  Needs no scipy: the Gaussian is written out in scipy's own order.

Follows gen_bottom_up_proposals.py of yjxiong/action-detection and the functions it calls:
  merge_scores         gen_bottom_up_proposals.py:76-91   stream merge (crop mean, truncate / resample, weights)
  softmax              ops/metrics.py:8-11
  gaussian_filter1d    scipy.ndimage.gaussian_filter(col, bw) as ops/sequence_funcs.py:30 calls it (truncate 4.0, 'reflect')
  frame_labels         ops/sequence_funcs.py:11-34 (label_frame_by_threshold, multicrop=False)
  build_boxes          ops/sequence_funcs.py:101-136 (build_box_by_search)
  temporal_nms         ops/sequence_funcs.py:71-97 (temporal_nms_fallback)
  gen_prop             gen_bottom_up_proposals.py:116-142 (no regression branch)
Pinned by tests/golden/proposals.npz, produced by oracle/gen_golden_proposals.py from the real reference functions.

Two choices the reference leaves open are fixed here, as in csrc/proposals.cu:
  - tied scores: numpy's argsort()[::-1] does not order them; here they keep the order the search emitted them in
    (a stable sort by descending score);
  - NaN scores: argsort()[::-1] puts them first but, once there are several, in an order numpy does not promise (with
    numpy 2.3 it already differs from a stable reversed argsort at 17 elements); here every NaN-scored box comes first,
    in search order, whatever the NaN's sign, then the rest by stable descending score;
  - gen_prop returns the score of every NMS survivor next to the length-filtered boxes (the two lists disagree once
    minimum_len > 0); here every surviving box keeps its own score.
"""
import numpy as np

THRESHOLDS = (0.01, 0.05, 0.1, .15, 0.25, .4, .5, .6, .7, .8, .9, .95)      # gen_bottom_up_proposals.py:124
TOLERANCES = (0.05, .1, .2, .3, .4, .5, .6, 0.8, 1.0)                      # gen_bottom_up_proposals.py:127


def merge_scores(streams, weights=None):
    """streams: per stream an fp32 [T_i, crops, K] array of one video -> the merged [T, K] crop-mean score"""
    out = streams[0].mean(axis=1) * (1.0 if weights is None else weights[0])
    for i in range(1, len(streams)):
        add = streams[i].mean(axis=1)
        if add.shape[0] < out.shape[0]:
            out = out[:add.shape[0], :]
        elif add.shape[0] > out.shape[0]:
            tick = add.shape[0] / float(out.shape[0])
            add = add[[int(x * tick) for x in range(out.shape[0])], :]
        out += add * (1.0 if weights is None else weights[i])
    return out


def softmax(f_score):
    e = np.exp(f_score - f_score.max(axis=-1)[..., None])
    return e / e.sum(axis=-1)[..., None]


def gaussian_weights(sigma, truncate=4.0):
    """scipy.ndimage._filters._gaussian_kernel1d(sigma, 0, int(truncate * sigma + 0.5)): float64, sums to 1"""
    radius = int(truncate * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def reflect_index(i, n):
    """scipy's 'reflect' boundary (d c b a | a b c d | d c b a), repeated for reaches longer than the signal"""
    m = np.mod(i, 2 * n)
    return np.where(m < n, m, 2 * n - 1 - m)


def gaussian_filter1d(col, sigma, truncate=4.0):
    """scipy.ndimage.gaussian_filter(col, sigma) of an fp32 1-D array, bit for bit: the line is widened to double, each
    output is w0 * x[i] followed by += (x[i-j] + x[i+j]) * w_j from the far tap (j = radius) to the near one (j = 1), as
    scipy's symmetric-kernel loop does (NI_Correlate1D), and is rounded back to fp32"""
    w = gaussian_weights(sigma, truncate)
    r = (len(w) - 1) // 2
    n = len(col)
    x = col.astype(np.float64)
    i = np.arange(n)
    acc = x * w[r]
    for j in range(r, 0, -1):
        acc = acc + (x[reflect_index(i - j, n)] + x[reflect_index(i + j, n)]) * w[r + j]
    return acc.astype(np.float32)


def frame_labels(f_score, cls=0, bw=3, thresholds=THRESHOLDS):
    """-> (ss, smoothed fp32 [T], labels bool [n_thr, T]); bw None: no smoothing. The comparison is in fp32 (numpy 2 casts
    the Python threshold down to the array's dtype)."""
    ss = softmax(f_score)
    col = ss[:, cls + 1]
    sm = col if bw is None else gaussian_filter1d(col, bw)
    return ss, sm, np.stack([sm > np.float32(th) for th in thresholds]) if len(sm) else np.zeros((len(thresholds), 0), bool)


def _left_to_right_sums(frm_scores, windows):
    """sum(frm_scores[a:b]) with Python's sum over np.float32 (0 + x[a] + x[a+1] + ... in fp32), for every (a, b)"""
    out = np.empty(len(windows), np.float32)
    by_start = {}
    for k, (a, b) in enumerate(windows):
        by_start.setdefault(a, []).append((k, b))
    n = len(frm_scores)
    for a, lst in by_start.items():
        hi = min(max(b for _, b in lst), n)
        run = np.cumsum(np.concatenate((np.zeros(1, np.float32), frm_scores[a:hi])), dtype=np.float32)
        for k, b in lst:
            out[k] = run[max(min(b, n) - a, 0)]
    return out


def build_boxes(labels, frm_scores, tolerances=TOLERANCES):
    """build_box_by_search for one label row -> (start int64 [n], end int64 [n], score fp32 [n]) in the reference's order:
    per tolerance, the forward search over up[0..U-1], then the backward search over down[U-1..0].

    forward x: the first y > x with signal[up[y]] > signal[up[x]] gives (up[x], down[y-1]+1); none gives (up[x], down[-1]+1).
    backward x: the last y < x with signal[down[y]] < s_x gives (up[y+1], down[x]+1); none gives (up[0], down[x]+1) scored
    over [0, down[x]+2).  signal[i] = cs[i] - t*i in double with cs = cumsum(1 - label); s_x = signal[down[x]], or
    signal[T-1] - t when down[x] == T.  Both searches are monotonic stacks, which find the same y as the reference's scans."""
    T = len(labels)
    lab = labels.astype(np.int64)
    diff = np.empty(T + 1)
    diff[1:-1] = lab[1:] - lab[:-1]
    diff[0], diff[T] = float(lab[0]), -float(lab[-1])
    up, down = np.nonzero(diff == 1)[0], np.nonzero(diff == -1)[0]
    cs = np.cumsum(1 - lab)
    U = len(up)
    starts, ends, windows = [], [], []
    for t in tolerances:
        t = np.float64(t)
        signal = cs - t * np.arange(T)
        su = signal[up]
        sd = np.array([signal[d] if d < T else signal[-1] - t for d in down])
        nxt, stack = [-1] * U, []
        for x in range(U - 1, -1, -1):
            while stack and su[stack[-1]] <= su[x]:
                stack.pop()
            nxt[x] = stack[-1] if stack else -1
            stack.append(x)
        prv, stack = [-1] * U, []
        for x in range(U):
            while stack and sd[stack[-1]] >= sd[x]:
                stack.pop()
            prv[x] = stack[-1] if stack else -1
            stack.append(x)
        for x in range(U):
            e = down[nxt[x] - 1] + 1 if nxt[x] >= 0 else down[-1] + 1
            starts.append(up[x]); ends.append(e); windows.append((up[x], e))
        for x in range(U - 1, -1, -1):
            y = prv[x]
            if y >= 0:
                starts.append(up[y + 1]); ends.append(down[x] + 1); windows.append((up[y + 1], down[x] + 1))
            else:
                starts.append(up[0]); ends.append(down[x] + 1); windows.append((0, down[x] + 2))
    return (np.array(starts, np.int64), np.array(ends, np.int64),
            _left_to_right_sums(frm_scores, windows) if windows else np.zeros(0, np.float32))


def temporal_nms(t1, t2, scores, thresh):
    """temporal_nms_fallback: frame-inclusive durations t2 - t1 + 1, intersection min - max + 1 (negative for disjoint
    boxes, which are never suppressed), IoU divided in double, a box survives while IoU <= thresh.  NaN-scored boxes
    come first in input order, then the rest by descending score; ties in score keep their input order.  -> indices of
    the survivors, in the order they were kept"""
    t1, t2 = np.asarray(t1, np.int64), np.asarray(t2, np.int64)
    durations = t2 - t1 + 1
    scores = np.asarray(scores, np.float32)
    nan = np.isnan(scores)
    rest = np.nonzero(~nan)[0]
    order = np.concatenate([np.nonzero(nan)[0], rest[np.argsort(-scores[rest], kind="stable")]]).astype(np.int64)
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        inter = np.minimum(t2[i], t2[order[1:]]) - np.maximum(t1[i], t1[order[1:]]) + 1
        iou = inter / (durations[i] + durations[order[1:]] - inter).astype(float)
        order = order[np.where(iou <= thresh)[0] + 1]
    return np.array(keep, np.int64)


def gen_prop(f_score, duration, cls=0, bw=3, thresholds=THRESHOLDS, tolerances=TOLERANCES, nms_threshold=0.9, minimum_len=0.0):
    """one video's merged [T, K] score -> dict of every stage: ss, smoothed, labels, the raw boxes (start, end, score) in
    search order, the NMS survivors (keep order), and the length-filtered pr_box [n, 2] seconds with their own scores"""
    T = len(f_score)
    ss, sm, labels = frame_labels(f_score, cls, bw, thresholds)
    frm = f_score[:, cls + 1]
    parts = [build_boxes(row, frm, tolerances) for row in labels]
    s, e, sc = (np.concatenate([p[k] for p in parts]) for k in range(3))
    keep = temporal_nms(s, e, sc, nms_threshold)
    ks, ke, ksc = s[keep], e[keep], sc[keep]
    pr = np.stack([ks / float(T) * duration, ke / float(T) * duration], axis=1) if len(keep) else np.zeros((0, 2))
    ok = pr[:, 1] - pr[:, 0] > minimum_len
    return {"ss": ss, "smoothed": sm, "labels": labels, "raw_start": s, "raw_end": e, "raw_score": sc,
            "nms_start": ks, "nms_end": ke, "nms_score": ksc, "pr_box": pr[ok], "pr_score": ksc[ok],
            "pr_frames": np.stack([ks[ok], ke[ok]], axis=1) if len(keep) else np.zeros((0, 2), np.int64)}
