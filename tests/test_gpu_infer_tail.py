"""The test-time tail of SSN against float64 (oracle/infer_check.py): the crop-mean test FC and the plain test FC, the
re-organised STPP through its column prefix sums, and detection post-processing (combined scores, class-wise NMS,
regression), each fed what the previous kernel wrote, at the benchmarked shapes, ActivityNet's K = 200, the size limits
and the edges.  Run on an H100: pytest -m gpu -s tests/test_gpu_infer_tail.py."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import infer_check as IC
from oracle import ssn_oracle as O
from oracle import synth

NPOT_CFG = ((1, 3), (1, 2, 3, 5), (1, 6))
COURSE8_CFG = (1, (1, 2, 3, 4, 5, 6, 7, 8), 1)
SSNB_ENOSUPPORT = 4
NAN = float("nan")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _report(title, chk):
    print("\n%s:" % title, *chk.records, sep="\n  ")


def _lib():
    from ssn_b200._lib import lib, check, int_array
    from ssn_b200.engine import _stream
    return lib, check, int_array, _stream


# ---- kernel calls, outputs pre-filled with NaN so that an unwritten element shows ---------------------------------------------
def _cropmean(feat, w, b, crops):
    lib, check, _ia, _stream = _lib()
    nt = feat.shape[0] // crops
    y = torch.full((nt, w.shape[0]), NAN, device=feat.device)
    check(lib.ssnb_test_fc_cropmean(feat.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), crops, nt, feat.shape[1],
                                    w.shape[0], y.data_ptr(), _stream()), None, "test_fc_cropmean")
    return y


def _linear(x, w, b):
    lib, check, _ia, _stream = _lib()
    y = torch.full((x.shape[0], w.shape[0]), NAN, device=x.device)
    check(lib.ssnb_linear_fwd(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), x.shape[0], x.shape[1], w.shape[0],
                              y.data_ptr(), _stream()), None, "linear_fwd")
    return y


def _lens(K):
    return K + 1, K, 2 * K


def _reorg(scores, ticks, sc, K, cfg, n=None, fill=NAN):
    """one ssnb_stpp_reorg_prefix call -> (act, comp, reg, workspace, the three output buffers)"""
    lib, check, int_array, _stream = _lib()
    dev = scores.device
    parts = [O.parse_stage_config(c)[0] for c in cfg]
    n = ticks.shape[0] if n is None else n
    tk = ticks.to(device=dev, dtype=torch.int32).contiguous()
    s2 = sc.to(device=dev, dtype=torch.float32).contiguous()
    outs = [torch.full((max(n, 1), L), fill, device=dev) for L in _lens(K)]
    args = (scores.data_ptr(), scores.shape[0], scores.shape[1], tk.data_ptr(), s2.data_ptr(), n, *_lens(K),
            int_array([len(p) for p in parts]), int_array([v for p in parts for v in p]), *[o.data_ptr() for o in outs])
    ws = torch.full((lib.ssnb_stpp_reorg_workspace_bytes(scores.shape[0], scores.shape[1]),), 0xAB, dtype=torch.uint8, device=dev)
    check(lib.ssnb_stpp_reorg_prefix(*args, ws.data_ptr(), _stream()), None, "stpp_reorg_prefix")
    torch.cuda.synchronize()
    return [o[:n] for o in outs] + [ws, outs]


def _detect(props, act, comp, reg, thr, regress, scores=None, n=None):
    """one ssnb_detect_postprocess call over the first n (all) proposals -> (rc, detections [K, N, 5], counts [K], combined
    workspace [N, K]); act None: rank `scores` as they are"""
    lib, _check, _ia, _stream = _lib()
    dev = props.device
    N = props.shape[0] if n is None else n
    K = (comp if act is not None else scores).shape[1]
    det = torch.full((K, max(N, 1), 5), NAN, device=dev)
    cnt = torch.full((K,), -1, dtype=torch.int32, device=dev)
    ws = scores.clone().contiguous() if act is None else torch.full((max(N, 1), K), NAN, device=dev)
    rc = lib.ssnb_detect_postprocess(props.data_ptr(), None if act is None else act.data_ptr(), None if act is None else comp.data_ptr(),
                                     reg.data_ptr(), N, K, float(thr), int(regress), det.data_ptr(), cnt.data_ptr(), ws.data_ptr(),
                                     _stream())
    torch.cuda.synchronize()
    return rc, det, cnt, ws


def _same(a, b):
    """bitwise equal, NaN equal to NaN"""
    return a.shape == b.shape and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


# ---- (a) test FC --------------------------------------------------------------------------------------------------------------
CROPMEAN_CASES = {                      # crops, nt, in_dim, out_dim, bias
    "bench_10x40_1024_321": (10, 40, 1024, 321, True),
    "K200_10x40_1024_3201": (10, 40, 1024, 3201, True),
    "partial_chunk_nt17": (10, 17, 1024, 321, True),
    "nt1_crops1": (1, 1, 1024, 321, True),
    "in1000_lane_tails": (10, 12, 1000, 321, True),
    "in12000_smem_limit": (2, 8, 12000, 64, True),
    "no_bias": (10, 40, 1024, 321, False),
}


def test_cropmean_fc_vs_float64():
    """linear_cropmean_kernel vs b + W . mean_c(x) at the bench's chunk, K = 200, a partial chunk, one tick of one crop, lane
    tails (in_dim 1000), the shared-memory limit (in_dim 12000) and no bias"""
    dev = _cuda()
    g = torch.Generator().manual_seed(61)
    chk = IC.Checker()
    for name, (crops, nt, ind, outd, bias) in CROPMEAN_CASES.items():
        feat = torch.randn(crops * nt, ind, generator=g).relu().to(dev)
        w = (torch.randn(outd, ind, generator=g) * 0.02).to(dev)
        b = (torch.randn(outd, generator=g) * 0.1).to(dev) if bias else None
        IC.check_cropmean(chk, "cropmean " + name, feat, w, b, crops, _cropmean(feat, w, b, crops))
    _report("linear_cropmean_kernel vs float64", chk)
    chk.assert_ok()


def test_linear_fwd_vs_float64():
    """linear_fwd_kernel (SSN.test_forward / BinaryClassifier.test_forward) at n = 400, out 2 / 321 / 3201, and n = 1"""
    dev = _cuda()
    g = torch.Generator().manual_seed(62)
    chk = IC.Checker()
    for n, outd, bias in ((400, 2, True), (400, 321, True), (400, 3201, True), (1, 321, True), (400, 321, False)):
        x = torch.randn(n, 1024, generator=g).relu().to(dev)
        w = (torch.randn(outd, 1024, generator=g) * 0.02).to(dev)
        b = (torch.randn(outd, generator=g) * 0.1).to(dev) if bias else None
        IC.check_linear(chk, "linear n=%d out=%d%s" % (n, outd, "" if bias else " no bias"), x, w, b, _linear(x, w, b))
    _report("linear_fwd_kernel vs float64", chk)
    chk.assert_ok()


# ---- (b) re-organised STPP -----------------------------------------------------------------------------------------------------
def _D(K, cfg):
    mult = sum(sum(O.parse_stage_config(c)[0]) for c in cfg)
    return (K + 1) + mult * 3 * K


def _grid_ticks():
    """every course span 1..259 at left 0, 3 and 700, with starting / ending spans that run through 1..259 as well"""
    rows = []
    for span in range(1, 260):
        s0, s3 = (span * 7) % 259 + 1, (span * 13) % 259 + 1
        for left in (0, 3, 700):
            rows.append((left - s0, left, left + span, left + span + s3))
    return torch.tensor(rows)


def _reorg_case(name):
    """-> scores [T, D], ticks [N, 4], scaling [N, 2], K, stpp_cfg"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    cfg, K = (1, (1, 2), 1), 20
    if name == "bench":                          # bench.py --mode infer: T = N = 1000, ticks drawn from [0, T]
        T, N = 1000, 1000
        ticks = torch.sort(torch.randint(0, T + 1, (N, 4), generator=g), dim=1)[0]
        sc = torch.rand(N, 2, generator=g)
    elif name == "dataset_ticks":                # ssn_dataset.py's ticks of proposals, some touching 0 and 1
        T = 500
        st = torch.rand(300, generator=g) * 0.9
        ed = (st + torch.rand(300, generator=g) * 0.5 + 0.01).clamp(max=1.0)
        st[:20], ed[20:40] = 0.0, 1.0
        st[40], ed[40] = 0.0, 1.0
        ticks, sc = IC.dataset_ticks(torch.stack([st, ed], 1).double(), T)
    elif name == "K200_T3000":
        T, N, K = 3000, 300, 200
        ticks = torch.sort(torch.randint(0, T + 1, (N, 4), generator=g), dim=1)[0]
        sc = torch.rand(N, 2, generator=g)
    elif name == "T20000_offset30":
        T, N = 20000, 200
        ticks = torch.sort(torch.randint(0, T + 1, (N, 4), generator=g), dim=1)[0]
        sc = torch.rand(N, 2, generator=g)
    elif name == "T1":
        T, N, K = 1, 40, 4
        ticks = torch.sort(torch.randint(-2, 3, (N, 4), generator=g), dim=1)[0]
        sc = torch.rand(N, 2, generator=g)
    elif name == "edges":
        T, K = 50, 4
        ticks = torch.tensor([[10, 20, 20, 30],       # tk1 == tk2
                              [40, 50, 50, 60],       # tk1 == T: empty activity slice (NaN)
                              [50, 50, 50, 50], [60, 70, 80, 90],          # left >= T in every stage
                              [-9, -7, -4, 0], [-5, -1, -1, -1],           # right <= 0; raw[-1:0] (NaN)
                              [-3, 2, 5, 9], [-12, -6, 3, 8],              # negative ticks: Python slices from the end
                              [45, 49, 55, 70], [0, 0, 0, 0], [0, 0, 1, 50], [0, 25, 26, 50]])
        sc = torch.rand(ticks.shape[0], 2, generator=g)
    elif name in NPOT_CASES:
        T, K = 1300, 2
        cfg = {"npot_1_13_1": (1, (1, 3), 1), "npot_mixed": NPOT_CFG, "course_8_levels": COURSE8_CFG}[name]
        ticks = _grid_ticks()
        sc = torch.rand(ticks.shape[0], 2, generator=g)
    else:
        raise KeyError(name)
    scores = torch.randn(T, _D(K, cfg), generator=g)
    if name == "T20000_offset30":
        scores += 30
    if name in NPOT_CASES:
        scores += 1                              # K = 2: keep the 22 .. 38 summed parts of a row from cancelling
    return scores, ticks, sc, K, cfg


def _naive_ticks(left, right, n_part):
    step = (right - left) / n_part
    return [int(left + q * step) for q in range(n_part + 1)]


NPOT_CASES = ("npot_1_13_1", "npot_mixed", "course_8_levels")
REORG_CASES = ["bench", "dataset_ticks", "K200_T3000", "T20000_offset30", "T1", "edges", "npot_1_13_1", "npot_mixed",
               "course_8_levels"]


@pytest.mark.parametrize("name", REORG_CASES)
def test_stpp_reorg_vs_float64(name):
    """stpp_reorg_prefix_kernel (after colscan_f64_kernel) vs reorg64, per proposal, NaN positions included; a repeated call
    gives the same bits"""
    dev = _cuda()
    scores, ticks, sc, K, cfg = _reorg_case(name)
    sd = scores.to(dev)
    ref = IC.reorg64(scores, ticks, sc, *_lens(K), cfg)
    chk = IC.Checker()
    got = _reorg(sd, ticks, sc, K, cfg)[:3]
    IC.check_reorg(chk, "reorg prefix %s" % name, scores, ticks, sc, *_lens(K), cfg, got, ref=ref, bar=IC.REORG_BAR)
    again = _reorg(sd, ticks, sc, K, cfg)[:3]
    for q, a, b in zip(("act", "comp", "reg"), got, again):
        assert _same(a, b), (q, "repeat")
    if name == "edges":
        assert torch.isnan(got[0][1]).all() and torch.isnan(got[0][5]).all()
    if name in NPOT_CASES:
        # the grid has teeth: part boundaries at left + q * step would be off at comp / reg, and only there
        with pytest.MonkeyPatch.context() as m:
            m.setattr(IC, "reorg_ticks", _naive_ticks)
            naive = IC.reorg64(scores, ticks, sc, *_lens(K), cfg)
        c2 = IC.Checker()
        IC.check_reorg(c2, "naive", scores, ticks, sc, *_lens(K), cfg, got, ref=naive)
        assert {q for _op, q in c2.failed()} == {"comp", "reg"}, c2.report()
    _report("re-organised STPP %s (T=%d, N=%d, K=%d, %s) vs float64" % (name, scores.shape[0], ticks.shape[0], K, cfg), chk)
    chk.assert_ok()


def test_stpp_reorg_n0_writes_nothing():
    dev = _cuda()
    scores, ticks, sc, K, cfg = _reorg_case("edges")
    outs = _reorg(scores.to(dev), ticks, sc, K, cfg, n=0, fill=-7.0)
    assert all(o.shape[0] == 0 for o in outs[:3])
    assert all(bool(o.eq(-7.0).all()) for o in outs[4])
    assert bool(outs[3].eq(0xAB).all())


# ---- (c) detection --------------------------------------------------------------------------------------------------------------
def _props(N, g, dyadic=False):
    if dyadic:
        st = torch.randint(0, 48, (N,), generator=g).float() / 64
        return torch.stack([st, st + torch.randint(1, 17, (N,), generator=g).float() / 64], 1)
    c, d = torch.rand(N, generator=g), torch.rand(N, generator=g) * 0.3 + 0.005
    return torch.stack([(c - d / 2).clamp(0, 1), (c + d / 2).clamp(0, 1)], 1)


def _idx_reg(N, K, dev):
    """(loc, dur) = (proposal index, 0): an unregressed call then reports which proposal each kept row is"""
    r = torch.zeros(N, K, 2, device=dev)
    r[:, :, 0] = torch.arange(N, device=dev, dtype=torch.float32)[:, None]
    return r


def _run_detect(chk, op, props, act, comp, reg, thr):
    """an unregressed call with index-carrying regressions (the kept indices) and a regressed call, both through the C ABI;
    checks the kernel's own combined scores, survivors and order, fields and boxes -> (ws, kept, dets)"""
    N, K = comp.shape
    rcA, detA, cntA, ws = _detect(props, act, comp, _idx_reg(N, K, props.device), thr, 0)
    rcB, detB, cntB, wsB = _detect(props, act, comp, reg, thr, 1)
    assert rcA == 0 and rcB == 0
    assert _same(ws, wsB) and torch.equal(cntA, cntB)
    counts = cntA.tolist()
    kept = [detA[c, :counts[c], 3].long().cpu().numpy() for c in range(K)]
    for c in range(K):
        assert torch.equal(detA[c, :counts[c], :2], props[torch.as_tensor(kept[c], device=props.device)]), c
    dets = [detB[c, :counts[c]] for c in range(K)]
    IC.check_detect(chk, op, props, ws, thr, kept, dets, reg, act, comp)
    return ws, kept, dets, detB, cntB


DETECT_CASES = {"N1000_K20": (1000, 20, 0.6), "N8192_K200": (8192, 200, 0.4), "N5000_K20": (5000, 20, 0.7),
                "N1_K20": (1, 20, 0.6)}


@pytest.mark.parametrize("name", sorted(DETECT_CASES))
def test_detect_vs_float64(name):
    """combined scores vs combined64; survivors and order exactly nms64 of the kernel's own combined scores (read back from
    the workspace); regressed boxes vs regress64; N = 5000 sorts 3192 padding slots"""
    dev = _cuda()
    N, K, thr = DETECT_CASES[name]
    g = torch.Generator().manual_seed(N + K)
    props = _props(N, g).to(dev)
    act, comp = (torch.randn(N, K + 1, generator=g) * 2).to(dev), (torch.randn(N, K, generator=g) * 0.5).to(dev)
    reg = (torch.randn(N, K, 2, generator=g) * 0.3).to(dev)
    chk = IC.Checker()
    _ws, kept, _d, detB, cntB = _run_detect(chk, "detect " + name, props, act, comp, reg, thr)
    from ops.detection import video_detections
    det_m, cnt_m = video_detections(props, act, comp, reg, thr)
    assert torch.equal(cnt_m, cntB)
    for c in range(K):
        assert _same(det_m[c, :int(cntB[c])], detB[c, :int(cntB[c])]), c
    _report("detection %s (thr %g): %d..%d kept per class" % (name, thr, min(map(len, kept)), max(map(len, kept))), chk)
    chk.assert_ok()


def test_detect_n0_and_size_limit():
    """N = 0: every count 0.  N = 8193: SSNB_ENOSUPPORT before any launch, nothing written"""
    dev = _cuda()
    lib, _c, _ia, _s = _lib()
    K = 5
    for N in (0, 8193):
        g = torch.Generator().manual_seed(N)
        n1 = max(N, 1)                               # N = 0: one-row buffers, so that every pointer is valid
        props = _props(n1, g).to(dev)
        act, comp, reg = torch.randn(n1, K + 1, device=dev), torch.randn(n1, K, device=dev), torch.randn(n1, K, 2, device=dev)
        before = lib.ssnb_global_launch_count()
        rc, det, cnt, ws = _detect(props, act, comp, reg, 0.5, 1, n=N)
        if N == 0:
            assert rc == 0 and cnt.tolist() == [0] * K
        else:
            assert rc == SSNB_ENOSUPPORT and lib.ssnb_global_launch_count() == before
            assert cnt.tolist() == [-1] * K and bool(torch.isnan(ws).all()) and bool(torch.isnan(det).all())


def _edge_fixture(dev):
    """N = 40, K = 3, thr 0.5, dyadic boxes: exact ties, IoU exactly at the threshold, zero-duration and identical boxes,
    disjoint boxes, a NaN act row, a combined score that is 0 * inf = NaN in fp32, regressions clipped at 0 and 1"""
    g = torch.Generator().manual_seed(71)
    N, K = 40, 3
    props = _props(N, g, dyadic=True)
    props[:12] = torch.tensor([[0.25, 0.5], [0.25, 0.5], [0, 0.5], [0, 0.25], [0.75, 0.75], [0.75, 0.75],
                               [0.0, 0.125], [0.875, 1.0], [0.5, 0.75], [0.25, 0.75], [0, 0.0625], [0.9375, 1.0]])
    act = torch.randn(N, K + 1, generator=g)
    comp = torch.randn(N, K, generator=g) * 0.5
    act[1], comp[1] = act[0], comp[0]                           # rows 0 and 1: the same scores
    act[2:4] += 2
    act[8] = NAN                                                # NaN act: a NaN combined row
    act[9] = torch.tensor([0.0, 0.0, -200.0, 0.0])
    comp[9, 1] = 100.0                                          # softmax 0 in fp32 (not in float64) times exp = inf
    reg = torch.randn(N, K, 2, generator=g) * 0.3
    reg[10:12, :, 1] = 2.0                                      # widened past 0 and 1
    reg[10, :, 0], reg[11, :, 0] = -0.5, 0.5
    return props.to(dev), act.to(dev), comp.to(dev), reg.to(dev), 0.5


def test_detect_edges_vs_float64():
    """the edge fixture through ssnb_detect_postprocess and ops.detection.video_detections: NaN-scored proposals ranked
    first, exact ties larger index first, IoU == thr kept, padding never read; combined scores vs float64 off the overflow"""
    dev = _cuda()
    props, act, comp, reg, thr = _edge_fixture(dev)
    N, K = comp.shape
    chk = IC.Checker()
    rcA, detA, cntA, ws = _detect(props, act, comp, _idx_reg(N, K, dev), thr, 0)
    rc, detB, cnt, wsB = _detect(props, act, comp, reg, thr, 1)
    assert rcA == 0 and rc == 0 and _same(ws, wsB)
    assert torch.isnan(ws[8]).all() and torch.isnan(ws[9, 1]) and torch.isfinite(ws[9, [0, 2]]).all()
    assert ws[0].eq(ws[1]).all()
    off = [i for i in range(N) if i != 9]
    chk.add("detect edges", "combined", ws[off], IC.combined64(act, comp)[off], IC.COMBINED_BAR, rows=True)
    counts = cntA.tolist()
    kept = [detA[c, :counts[c], 3].long().cpu().numpy() for c in range(K)]
    IC.check_detect(chk, "detect edges", props, ws, thr, kept, [detB[c, :counts[c]] for c in range(K)], reg)
    for c in range(K):
        k = kept[c].tolist()
        # NaN first, NaN against NaN and exact ties larger index first
        assert k[:2] == [9, 8] if c == 1 else k[0] == 8, (c, k)
        assert 0 not in k or 1 not in k or k.index(1) < k.index(0)
    boxes = torch.cat([detB[c, :counts[c], :2] for c in range(K)])
    assert bool((boxes >= 0).all() and (boxes <= 1).all()) and bool((boxes == 0).any() and (boxes == 1).any())
    from ops.detection import video_detections
    det_m, cnt_m = video_detections(props, act, comp, reg, thr)
    assert torch.equal(cnt_m, cnt)
    for c in range(K):
        assert _same(det_m[c, :counts[c]], detB[c, :counts[c]]), c
    _report("detection edge fixture", chk)
    chk.assert_ok()


@pytest.mark.parametrize("n", [32, 37])
def test_temporal_nms_nan_inf_ties(n):
    """ops.detection.temporal_nms on scores with NaN, -inf and exact ties (n = 32: no padding; 37: 27 padding slots) equals
    the rows nms64 keeps, in its order"""
    dev = _cuda()
    from ops.detection import temporal_nms
    g = torch.Generator().manual_seed(n)
    props = _props(n, g, dyadic=True)
    props[:4] = torch.tensor([[0, 0.5], [0, 0.25], [0.5, 0.5], [0.5, 0.5]])
    scores = torch.randint(0, 4, (n,), generator=g).float() / 4
    scores[[1, 7]] = NAN
    scores[[2, 9, 11]] = -math.inf
    bb = torch.cat([props, scores[:, None], torch.randn(n, 2, generator=g)], 1)
    for thr in (0.5, 0.25):
        got = temporal_nms(bb.to(dev), thr).cpu()
        want = bb[torch.as_tensor(IC.nms64(props, scores, thr))]
        assert _same(got, want), (thr, got[:, 2], want[:, 2])
        assert torch.isnan(got[0, 2])


# ---- (d) the bench's inference tail, chained ---------------------------------------------------------------------------------
def test_bench_inference_tail_chained():
    """bench.py --mode infer after the backbone: 25 crop-mean calls of 40 ticks x 10 crops (1024 -> 321, SSN's folded test FC)
    -> re-organised STPP through the prefix kernels (1000 proposals, ticks from [0, T]) -> detection, each stage against
    float64 of what the previous kernel wrote"""
    dev = _cuda()
    K, T, crops, chunk, N = 20, 1000, 10, 40, 1000
    w, b = O.prepare_test_fc(synth.synth_heads(K, 5, seed=0), 5)
    w, b = w.to(dev), b.to(dev)
    g = torch.Generator().manual_seed(81)
    chk = IC.Checker()
    out = torch.full((T, w.shape[0]), NAN, device=dev)
    for c in range(T // chunk):
        feat = torch.randn(crops * chunk, 1024, generator=g).relu().to(dev)
        out[c * chunk:(c + 1) * chunk] = y = _cropmean(feat, w, b, crops)
        IC.check_cropmean(chk, "cropmean chunk %d" % c, feat, w, b, crops, y)
    worst = max((r for r in chk.records), key=lambda r: r.err)
    chk.records = [IC.Record("cropmean x25", "y", worst.err, worst.bar, "%s, %s" % (worst.op, worst.where))]
    ticks = torch.sort(torch.randint(0, T + 1, (N, 4), generator=g), dim=1)[0]
    sc = torch.rand(N, 2, generator=g)
    cfg = (1, (1, 2), 1)
    act, comp, reg = _reorg(out, ticks, sc, K, cfg)[:3]
    IC.check_reorg(chk, "reorg prefix", out, ticks, sc, *_lens(K), cfg, (act, comp, reg))
    props = (ticks[:, 1:3].float() / T).to(dev)
    _run_detect(chk, "detect", props, act, comp, reg.view(N, K, 2), 0.6)
    _report("bench inference tail, chained", chk)
    chk.assert_ok()
