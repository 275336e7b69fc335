"""Video-level aggregation, fusion and metrics on the H100 (csrc/video_agg.cu through ops/video_funcs.py and ops/metrics.py):
the golden vectors of the reference's own functions, ragged batches of about 1000 videos against the oracle in every mode,
one call against one call per video, repeats, CUDA-graph replay, poisoned outputs and workspace, the tie rule and refusals
that launch nothing."""
import ctypes as C
import json
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import video_funcs_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "video_funcs.npz"))
AGGS = [str(x) for x in GOLD["agg_fixtures"]]
METS = [str(x) for x in GOLD["met_fixtures"]]
MCAS = [str(x) for x in GOLD["mca_fixtures"]]
DEV = torch.device("cuda:0")


def agg_fixture(name):
    src = str(GOLD["agg_%s_inputs" % name])
    return GOLD["agg_%s_scores" % src], GOLD["agg_%s_offsets" % src], json.loads(str(GOLD["agg_%s_params" % name]))


def close(got, want, rel=2e-6):
    """NaN and infinities where the reference has them, finite values within rel of the reference's"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype
    assert (np.isnan(got) == np.isnan(want)).all()
    m = np.isfinite(want)
    assert (got[~m & ~np.isnan(want)] == want[~m & ~np.isnan(want)]).all()
    err = np.abs(got[m].astype(np.float64) - want[m]) / np.maximum(np.abs(want[m].astype(np.float64)), 1e-30)
    assert err.max(initial=0) <= rel, err.max()


def same(got, want):
    """bitwise, but any NaN equals any NaN (payloads are not numpy's business) and -0 equals +0: np.max of a -0 and a +0 gives
    either, by CPU"""
    got, want = np.asarray(got), np.asarray(want)
    return got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want, equal_nan=True)


def kwargs(p):
    p = dict(p)
    mode = p.pop("mode")
    if "norm" in p:
        p["normalization"] = p.pop("norm")
    return mode, p


def test_aggregation_golden_in_one_call():
    from ops.video_funcs import aggregate_packed
    for name in AGGS:
        scores, off, p = agg_fixture(name)
        mode, kw = kwargs(p)
        got = aggregate_packed(torch.from_numpy(scores).to(DEV), off, mode, **kw).cpu().numpy()
        close(got, GOLD["agg_%s_out" % name])
        if not kw.get("normalization", False):
            with np.errstate(all="ignore"):
                want = O.aggregate_packed(scores, off, mode, **{k: v for k, v in p.items() if k != "mode"})
            assert same(got, want), name                         # numpy's order: bitwise without the softmax


def test_per_video_dropins_return_what_the_reference_returns():
    import ops.video_funcs as VF
    scores, off, _ = agg_fixture("sliding_norm")
    for v in range(len(off) - 1):
        s = scores[off[v]:off[v + 1]]
        for fn, args, key in ((VF.default_aggregation_func, (), None), (VF.top_k_aggregation_func, (3,), None),
                              (VF.sliding_window_aggregation_func, (), None)):
            r = fn(s, *args)
            assert isinstance(r, np.ndarray) and r.dtype == np.float32 and r.shape == (scores.shape[2],)
        rt = VF.default_aggregation_func(torch.from_numpy(s).to(DEV), False, np.max)
        assert rt.is_cuda and rt.cpu().numpy().tobytes() == O.default_agg(s, False, "max").tobytes()
    for name in ("sliding_norm", "sliding_fps2", "tpp", "topk_k3"):
        scores, off, p = agg_fixture(name)
        mode, kw = kwargs(p)
        fn = {"sliding_window": lambda s: VF.sliding_window_aggregation_func(s, p["spans"], p["overlap"], p["norm"], p["fps"]),
              "tpp": lambda s: VF.tpp_aggregation_func(s, p["num_class"]),
              "top_k": lambda s: VF.top_k_aggregation_func(s, p["k"], p["normalization"], np.max if p["crop_agg"] == "max" else None)}[mode]
        close(np.stack([fn(scores[off[v]:off[v + 1]]) for v in range(len(off) - 1)]), GOLD["agg_%s_out" % name])
    st, w = GOLD["fuse_streams"], [float(x) for x in GOLD["fuse_weights"]]
    for norm in (True, False):
        got = np.stack([VF.default_fusion_func(st[0][v], [st[1][v], st[2][v]], w, norm) for v in range(st.shape[1])])
        close(got, GOLD["fuse_%s_out" % ("norm" if norm else "raw")])
    from ops.metrics import softmax
    close(softmax(GOLD["softmax_in"]), GOLD["softmax_out"])
    close(softmax(GOLD["softmax_in"], 2), GOLD["softmax_t2_out"])


def ragged_set(seed, V=1000, crops=4, D=24, tmax=80, quantise=False):
    rng = np.random.default_rng(seed)
    Ts = rng.integers(1, tmax, V)
    Ts[:5] = [1, 2, 5, 13, 15]
    off = np.r_[0, np.cumsum(Ts)].astype(np.int64)
    s = (rng.standard_normal((int(off[-1]), crops, D)) * 3).astype(np.float32)
    if quantise:
        s = np.round(s).astype(np.float32)
    return s, off


MODES = [("default", dict(normalization=False, crop_agg="mean")), ("default", dict(normalization=True, crop_agg="max")),
         ("top_k", dict(k=5, normalization=False, crop_agg="max")), ("top_k", dict(k=20, normalization=True, crop_agg="mean")),
         ("sliding_window", dict(spans=[1, 2, 4, 8, 16], overlap=0.2, norm=False, fps=1)),
         ("sliding_window", dict(spans=[1, 2, 4], overlap=0.2, norm=True, fps=2)), ("tpp", dict(num_class=6))]


@pytest.mark.parametrize("mode,kw", MODES, ids=["%s-%d" % (m, i) for i, (m, _) in enumerate(MODES)])
def test_ragged_batch_against_oracle_per_video_calls_and_repeats(mode, kw):
    from ops.video_funcs import aggregate_packed
    scores, off = ragged_set(1, quantise=mode != "tpp")
    _, k2 = kwargs(dict(mode=mode, **kw))
    st = torch.from_numpy(scores).to(DEV)
    got = aggregate_packed(st, off, mode, **k2)
    want = O.aggregate_packed(scores, off, mode, **kw)
    close(got.cpu().numpy(), want)
    if not k2.get("normalization", False):
        assert same(got.cpu().numpy(), want)
    again = aggregate_packed(st, off, mode, **k2)
    assert torch.equal(got.view(torch.uint8), again.view(torch.uint8))
    for v in range(0, len(off) - 1, 37):
        one = aggregate_packed(st[off[v]:off[v + 1]].contiguous(), [0, off[v + 1] - off[v]], mode, **k2)
        assert torch.equal(one[0].view(torch.uint8), got[v].view(torch.uint8)), v


def test_graph_replay_on_new_scores_and_poisoned_buffers():
    from ssn_b200._lib import lib
    from ops.video_funcs import aggregate_packed
    scores, off = ragged_set(2, V=300)
    s2 = (np.random.default_rng(3).standard_normal(scores.shape) * 3).astype(np.float32)
    D, crops, V = scores.shape[2], scores.shape[1], len(off) - 1
    offc = np.ascontiguousarray(off)
    sp = (C.c_int * 5)(1, 2, 4, 8, 16)
    op = offc.ctypes.data_as(C.POINTER(C.c_int64))
    ws_bytes = lib.ssnb_video_aggregate_workspace_bytes(op, V, crops, D, 2, 0, 1, sp, 5, 0.2, 1, D)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=DEV)
    out = torch.full((V, D), float("nan"), device=DEV)
    out.view(torch.int32).fill_(-1)
    st = torch.from_numpy(scores).to(DEV)
    off_dev = torch.from_numpy(offc).to(DEV)
    stream = torch.cuda.Stream()

    def call():
        return lib.ssnb_video_aggregate(st.data_ptr(), op, off_dev.data_ptr(), V, crops, D, 2, 0, 1, 1, sp, 5, 0.2, 1, D, out.data_ptr(),
                                        ws.data_ptr(), ws_bytes, C.c_void_p(stream.cuda_stream))
    with torch.cuda.stream(stream):
        assert call() == 0
    stream.synchronize()
    eager = aggregate_packed(st, off, "sliding_window")
    assert torch.equal(out.view(torch.uint8), eager.view(torch.uint8))              # 0xFF outputs and workspace overwritten
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        assert call() == 0
    st.copy_(torch.from_numpy(s2))
    out.fill_(0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), aggregate_packed(st, off, "sliding_window").view(torch.uint8))


def met_fixture(name):
    p = "met_%s_" % name
    return GOLD[p + "scores"], GOLD[p + "label_video"], GOLD[p + "label"]


class _Inst:
    def __init__(self, c):
        self.num_label = c


class _Video:
    def __init__(self, vid, labels):
        self.id, self.instances = vid, [_Inst(c) for c in labels]


@pytest.mark.parametrize("name", METS)
def test_metrics_golden(name):
    import ops.metrics as M
    sc, lv, lab = met_fixture(name)
    p = "met_%s_" % name
    sets = [sorted(lab[lv == i].tolist()) for i in range(len(sc))]
    for k in (1, 3, 5):
        r = M.video_metrics_packed(torch.from_numpy(sc).to(DEV), lv, lab, k)
        acc = np.stack([r["hits"].cpu().numpy(), r["label_count"].cpu().numpy()], 1)
        assert (acc == GOLD[p + "acc_k%d" % k]).all()
        assert float(r["top_k_accuracy"][0]) == float(GOLD[p + "top_k_accuracy_k%d" % k])
        assert abs(float(r["mean_ap"][0]) - float(GOLD[p + "video_mean_ap"])) <= 1e-12
        assert [M.top_k_acc(set(s_), x, k) for s_, x in zip(sets, sc)] == [tuple(a) for a in GOLD[p + "acc_k%d" % k].tolist()]
        assert [M.top_k_hit(set(s_), x, k)[0] for s_, x in zip(sets, sc)] == [bool(h[0]) for h in GOLD[p + "hit_k%d" % k]]
    ids = ["v%03d" % i for i in range(len(sc))]
    vlist = [_Video(i, s_) for i, s_ in zip(ids, sets)] + [_Video("gone%d" % j, [0]) for j in range(int(GOLD[p + "missing"]))]
    sd = dict(zip(ids, sc))
    assert M.top_3_accuracy(sd, vlist) == float(GOLD[p + "top_k_accuracy_k3"])
    assert abs(M.video_mean_ap(sd, vlist) - float(GOLD[p + "video_mean_ap"])) <= 1e-12


def test_mean_class_accuracy_golden():
    import ops.metrics as M
    for name in MCAS:
        got, want = M.mean_class_accuracy(GOLD["mca_%s_scores" % name], GOLD["mca_%s_labels" % name]), float(GOLD["mca_%s_value" % name])
        assert (np.isnan(got) and np.isnan(want)) or abs(got - want) <= 1e-12, name


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_metrics_at_scale_against_oracle_with_the_tie_rule(dtype):
    import ops.metrics as M
    rng = np.random.default_rng(5)
    V, K = 1000, 200
    sc = np.round(rng.standard_normal((V, K)) * 2).astype(dtype)            # quantised: ties at every k-th place
    sc[3, :] = 0.0
    sc[4, ::7] = -0.0
    lv = np.repeat(np.arange(V), rng.integers(0, 4, V)).astype(np.int32)
    lab = rng.integers(0, K - 3, len(lv)).astype(np.int32)                  # repeated pairs; the last classes have no positive
    cl = rng.integers(0, K - 1, V).astype(np.int32)
    r = M.video_metrics_packed(torch.from_numpy(sc).to(DEV), lv, lab, 5, class_label=cl, trace=True)
    sets = [set(lab[lv == i].tolist()) for i in range(V)]
    idx = r["top_k_idx"].cpu().numpy()
    for v in range(V):
        assert idx[v].tolist() == O.rank(sc[v])[:5].tolist(), v
    want = np.array([O.top_k_acc(s_, x, 5) for s_, x in zip(sets, sc)])
    assert (np.stack([r["hits"].cpu().numpy(), r["label_count"].cpu().numpy()], 1) == want).all()
    assert float(r["top_k_accuracy"][0]) == O.top_k_accuracy(sc, sets, 5)
    mean_ap, ap = O.video_mean_ap(sc, sets)
    assert np.abs(r["ap"].cpu().numpy() - ap).max() <= 1e-12 and abs(float(r["mean_ap"][0]) - mean_ap) <= 1e-12
    _, cf = O.confusion(sc, cl)
    assert (r["confusion"].cpu().numpy() == cf).all()
    got, want = float(r["mean_class_accuracy"][0]), O.mean_class_accuracy(sc, cl)
    assert (np.isnan(got) and np.isnan(want)) or abs(got - want) <= 1e-12
    again = M.video_metrics_packed(torch.from_numpy(sc).to(DEV), lv, lab, 5, class_label=cl, trace=True)
    for k in ("hits", "ap", "mean_ap", "confusion", "top_k_idx"):
        assert torch.equal(again[k], r[k]), k


def test_refusals_launch_nothing():
    from ssn_b200._lib import lib
    import ops.metrics as M
    from ops.video_funcs import aggregate_packed
    s = torch.zeros(10, 2, 6, device=DEV)
    torch.cuda.synchronize()
    n0 = lib.ssnb_global_launch_count()
    for call in (lambda: aggregate_packed(s, [0, 4, 4, 10]),                       # a video without ticks
                 lambda: aggregate_packed(s, [0, 10], "top_k", k=0),
                 lambda: aggregate_packed(s, [0, 10], "sliding_window", crop_agg="max"),
                 lambda: aggregate_packed(s, [0, 10], "sliding_window", fps=0),
                 lambda: aggregate_packed(s, [0, 10], "tpp", num_class=4),
                 lambda: M.video_metrics_packed(torch.zeros(3, 1025, device=DEV), [0], [0]),
                 lambda: M.video_metrics_packed(torch.zeros(3, 5, device=DEV), [0], [0], top_k=0)):
        with pytest.raises(RuntimeError):
            call()
    assert lib.ssnb_global_launch_count() == n0
