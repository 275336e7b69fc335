"""ssnb_stpp_reorg_batch / ops.ssn_ops.reorg_packed on the H100: ssn_test.py:87-92 for many ragged videos per call.  The
golden videos against the reference's float64 pooling and its fp32 de-normalisation; a ragged 500-video call bitwise against
one single-video call per video; repeats into garbage-filled buffers, a CUDA-graph replay, the refusals; and a two-stream
THUMOS14-like set from test_proposals to the AP table, bitwise against evaluate_detections fed ssn_test.py-style dicts.
Run on an H100: pytest -m gpu -s tests/test_gpu_test_tail.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import infer_check as IC
from oracle import test_tail_oracle as TO
from test_test_tail_host import GOLD, SETS, golden_set, lens

STD_CFG = (1, (1, 2), 1)
SSNB_EINVAL, SSNB_ENOSUPPORT = 1, 4


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _bits(x):
    return x.contiguous().view(torch.int32)


def _same_bits(a, b):
    return a.shape == b.shape and bool(torch.equal(_bits(a), _bits(b)))


def _levels(cfg):
    from ssn_b200.engine import parse_stage_config
    parts = [parse_stage_config(c)[0] for c in cfg]
    return [len(p) for p in parts], [v for p in parts for v in p], sum(sum(p) for p in parts)


def _D(K, cfg):
    return K + 1 + _levels(cfg)[2] * 3 * K


def _torch_denorm(reg, stats, K):
    """ssn_test.py:89-92 as the reference runs it (torch, on the kernel's raw reg)"""
    reg_scores = reg.clone().view(-1, K, 2)
    reg_scores[:, :, 0] = reg_scores[:, :, 0] * stats[1, 0] + stats[0, 0]
    reg_scores[:, :, 1] = reg_scores[:, :, 1] * stats[1, 1] + stats[0, 1]
    return reg_scores


class Batch:
    """one raw ssnb_stpp_reorg_batch call with its buffers kept (outputs and workspace pre-filled with `fill`)"""

    def __init__(self, scores, toff, ticks, scaling, off, K, cfg, stats=None, fill=0xFF, spare=0):
        from ssn_b200._lib import lib
        self.lib, dev = lib, scores.device
        self.scores, self.ticks, self.scaling = scores, ticks.to(dev, torch.int32).contiguous(), scaling.to(dev, torch.float32).contiguous()
        self.toff, self.off, self.K, self.cfg, self.stats = [int(x) for x in toff], [int(x) for x in off], K, cfg, stats
        import ctypes as C
        V = len(self.off) - 1
        self.c_toff, self.c_off = (C.c_int64 * (V + 1))(*self.toff), (C.c_int64 * (V + 1))(*self.off)
        self.c_stats = None if stats is None else (C.c_double * 4)(*np.asarray(stats, np.float64).reshape(-1).tolist())
        self.toff_dev = torch.tensor(self.toff, dtype=torch.int64, device=dev)
        self.off_dev = torch.tensor(self.off, dtype=torch.int64, device=dev)
        N = self.off[-1]
        self.outs = [torch.full((N + spare, 4 * L), fill, dtype=torch.uint8, device=dev).view(torch.float32) for L in lens(K)]
        self.ws_bytes = lib.ssnb_stpp_reorg_batch_workspace_bytes(self.c_toff, V, scores.shape[1])
        self.ws = torch.full((max(self.ws_bytes, 1),), fill, dtype=torch.uint8, device=dev)

    def __call__(self, **override):
        from ssn_b200._lib import int_array
        from ssn_b200.engine import _stream
        counts, levels, _ = _levels(self.cfg)
        a = dict(scores=self.scores.data_ptr(), D=self.scores.shape[1], toff=self.c_toff, toff_dev=self.toff_dev.data_ptr(),
                 ticks=self.ticks.data_ptr(), scaling=self.scaling.data_ptr(), off=self.c_off, off_dev=self.off_dev.data_ptr(),
                 V=len(self.off) - 1, act=self.K + 1, comp=self.K, reg=2 * self.K, counts=int_array(counts), levels=int_array(levels),
                 stats=self.c_stats, out_act=self.outs[0].data_ptr(), out_comp=self.outs[1].data_ptr(), out_reg=self.outs[2].data_ptr(),
                 ws=self.ws.data_ptr(), ws_bytes=self.ws_bytes)
        a.update(override)
        return self.lib.ssnb_stpp_reorg_batch(*a.values(), _stream())

    def rows(self):
        return [o[:self.off[-1]] for o in self.outs]


def _single(scores_v, ticks_v, sc_v, K, cfg):
    """one ssnb_stpp_reorg_prefix call (STPPReorgainzed.forward)"""
    from ops.ssn_ops import STPPReorgainzed
    r = STPPReorgainzed(scores_v.shape[1], K + 1, K, 2 * K, True, stpp_cfg=cfg)
    return r.forward(scores_v, ticks_v, sc_v)


# ---- the golden videos ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SETS)
def test_golden_videos_in_one_call(name):
    from ops.ssn_ops import reorg_packed
    dev = _cuda()
    f = golden_set(name)
    K, cfg = f["K"], f["cfg"]
    scores = torch.from_numpy(f["scores"]).to(dev)
    tk, sc = torch.from_numpy(f["ticks"]).to(dev, torch.int32), torch.from_numpy(f["scaling"]).to(dev, torch.float32)
    act, comp, reg = reorg_packed(scores, f["tick_offsets"], tk, sc, f["offsets"], cfg, *lens(K))
    chk = IC.Checker()
    for q, g, r in zip(("act", "comp", "reg"), (act, comp, reg), (f["act64"], f["comp64"], f["reg64"])):
        chk.add("golden %s" % name, q, g.cpu(), torch.from_numpy(r), IC.REORG_BAR, rows=True)
    print("\ngolden set %s (K = %d, %s):" % (name, K, cfg), *chk.records, sep="\n  ")
    chk.assert_ok()
    stats = GOLD["reg_stats"]
    a2, c2, reg_dn = reorg_packed(scores, f["tick_offsets"], tk, sc, f["offsets"], cfg, *lens(K), reg_stats=stats)
    assert reg_dn.shape == (f["offsets"][-1], K, 2)
    assert _same_bits(a2, act) and _same_bits(c2, comp)
    assert reg_dn.cpu().numpy().tobytes() == TO.denorm32(reg.cpu().numpy(), stats).tobytes()
    assert _same_bits(reg_dn, _torch_denorm(reg, stats, K))
    # each video alone through STPPReorgainzed.forward: the same bits
    for v in range(len(f["offsets"]) - 1):
        t0, t1, r0, r1 = (int(x) for x in (f["tick_offsets"][v], f["tick_offsets"][v + 1], f["offsets"][v], f["offsets"][v + 1]))
        for g, s in zip((act, comp, reg), _single(scores[t0:t1], tk[r0:r1], sc[r0:r1], K, cfg)):
            assert _same_bits(g[r0:r1], s), (name, v)


# ---- a ragged 500-video call -------------------------------------------------------------------------------------------------
def _ragged(dev, V, K, cfg, seed, T_max=3000, N_max=1000, zero_T=(), zero_N=()):
    g = torch.Generator().manual_seed(seed)
    T = torch.randint(1, T_max + 1, (V,), generator=g)
    N = torch.randint(1, N_max + 1, (V,), generator=g)
    for v in zero_T:
        T[v] = 0
    for v in zero_N:
        N[v] = 0
    toff = [0] + torch.cumsum(T, 0).tolist()
    off = [0] + torch.cumsum(N, 0).tolist()
    # ticks per video from [-2, T + 2], sorted: raw slices, empty activity spans and stages past either end
    u = torch.rand(off[-1], 4, generator=g)
    Tr = torch.repeat_interleave(T, N).unsqueeze(1).double()
    ticks = torch.sort(torch.floor(u.double() * (Tr + 5)) - 2, 1)[0].to(torch.int32)
    sc = torch.rand(off[-1], 2, generator=g)
    gd = torch.Generator(device=dev).manual_seed(seed)
    scores = torch.randn(toff[-1], _D(K, cfg), generator=gd, device=dev)
    return scores, toff, ticks.to(dev), sc.to(dev), off


def test_ragged_500_videos_bitwise_against_single_calls():
    dev = _cuda()
    K = 100
    scores, toff, ticks, sc, off = _ragged(dev, 500, K, STD_CFG, 7)
    print("\nragged call: %d ticks, %d proposals, D = %d, workspace %.1f GB" % (toff[-1], off[-1], scores.shape[1],
                                                                             (toff[-1] + 500) * scores.shape[1] * 8 / 1e9))
    b = Batch(scores, toff, ticks, sc, off, K, STD_CFG)
    assert b() == 0
    torch.cuda.synchronize()
    got = b.rows()
    for v in range(500):
        t0, t1, r0, r1 = toff[v], toff[v + 1], off[v], off[v + 1]
        ref = _single(scores[t0:t1], ticks[r0:r1], sc[r0:r1], K, STD_CFG)
        for q, g_, r in zip(("act", "comp", "reg"), got, ref):
            assert _same_bits(g_[r0:r1], r), (v, q)
    del b


def test_empty_videos_and_untouched_rows():
    """videos with N_v = 0 write nothing and videos with T_v = 0 pool empty slices (NaN), as the oracle does; rows past
    the last one are not touched"""
    dev = _cuda()
    K = 4
    scores, toff, ticks, sc, off = _ragged(dev, 9, K, STD_CFG, 11, T_max=40, N_max=30, zero_T=(0, 4), zero_N=(2, 4, 8))
    b = Batch(scores, toff, ticks, sc, off, K, STD_CFG, fill=0x5A, spare=7)
    assert b() == 0
    torch.cuda.synchronize()
    ref = TO.reorg_packed64(scores.cpu(), toff, ticks.cpu(), sc.cpu(), off, *lens(K), STD_CFG)
    chk = IC.Checker()
    for q, g, r in zip(("act", "comp", "reg"), b.rows(), ref):
        chk.add("empty videos", q, g.cpu(), r, IC.REORG_BAR, rows=True)
    chk.assert_ok()
    assert bool(torch.isnan(b.rows()[0][off[0]:off[1]]).all())          # T_0 = 0: every activity slice is empty
    for o in b.outs:
        assert bool((_bits(o[off[-1]:]) == 0x5A5A5A5A).all())


def test_repeat_and_garbage_buffers_bitwise():
    dev = _cuda()
    K = 20
    stats = np.array([[0.031, -0.017], [0.113, 0.271]])
    scores, toff, ticks, sc, off = _ragged(dev, 40, K, STD_CFG, 3, T_max=500, N_max=300, zero_N=(5,))
    a = Batch(scores, toff, ticks, sc, off, K, STD_CFG, stats=stats, fill=0)
    b = Batch(scores, toff, ticks, sc, off, K, STD_CFG, stats=stats, fill=0xFF)
    assert a() == 0 and b() == 0
    first = [o.clone() for o in a.rows()]
    assert a() == 0
    torch.cuda.synchronize()
    for x, y, z in zip(first, a.rows(), b.rows()):
        assert _same_bits(x, y) and _same_bits(x, z)
    # the de-normalisation against the reference's torch lines on the raw call
    raw = Batch(scores, toff, ticks, sc, off, K, STD_CFG)
    assert raw() == 0
    assert _same_bits(a.rows()[2].view(-1, K, 2), _torch_denorm(raw.rows()[2], stats, K))


def test_cuda_graph_replay_on_new_scores():
    dev = _cuda()
    K = 20
    stats = np.array([[0.0123, -0.0457], [0.1789, 0.2345]])
    scores, toff, ticks, sc, off = _ragged(dev, 30, K, STD_CFG, 5, T_max=400, N_max=200)
    buf = scores.clone()
    b = Batch(buf, toff, ticks, sc, off, K, STD_CFG, stats=stats)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert b() == 0                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    before = [o.clone() for o in b.rows()]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert b() == 0
    fresh = torch.randn(scores.shape, generator=torch.Generator(device=dev).manual_seed(99), device=dev)
    buf.copy_(fresh)
    graph.replay()
    torch.cuda.synchronize()
    eager = Batch(fresh, toff, ticks, sc, off, K, STD_CFG, stats=stats)
    assert eager() == 0
    torch.cuda.synchronize()
    for x, y in zip(b.rows(), eager.rows()):
        assert _same_bits(x, y)
    assert not any(_same_bits(x, y) for x, y in zip(b.rows(), before))


def test_refusals_launch_nothing():
    import ctypes as C
    from ssn_b200._lib import lib, int_array
    dev = _cuda()
    K = 4
    scores, toff, ticks, sc, off = _ragged(dev, 5, K, STD_CFG, 13, T_max=30, N_max=20)
    b = Batch(scores, toff, ticks, sc, off, K, STD_CFG, stats=np.ones((2, 2)))
    torch.cuda.synchronize()
    n0 = lib.ssnb_global_launch_count()
    bad_toff = list(toff)
    bad_toff[2], bad_toff[3] = bad_toff[3], bad_toff[2]
    bad_off = list(off)
    bad_off[1] = off[2] + 1
    cases = [
        (dict(toff=(C.c_int64 * 6)(*bad_toff)), SSNB_EINVAL),
        (dict(off=(C.c_int64 * 6)(*bad_off)), SSNB_EINVAL),
        (dict(D=scores.shape[1] + 1), SSNB_EINVAL),
        (dict(act=K), SSNB_EINVAL),
        (dict(reg=2 * K + 1, comp=K - 1, D=(K + 1) + 5 * (3 * K)), SSNB_EINVAL),     # odd reg_len with reg_stats
        (dict(levels=int_array([1, 0, 3, 1])), SSNB_EINVAL),
        (dict(ws_bytes=b.ws_bytes - 8), SSNB_EINVAL),
        (dict(out_reg=None), SSNB_EINVAL),
        (dict(off_dev=None), SSNB_EINVAL),
        (dict(V=-1), SSNB_EINVAL),
        (dict(D=65535 * 128 + 1), SSNB_ENOSUPPORT),
    ]
    for over, rc in cases:
        assert b(**over) == rc, over
        assert lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0
    assert bool((_bits(b.outs[0]) == -1).all()) and bool((b.ws == 0xFF).all())
    # the wrapper refuses before the library is reached
    from ops.ssn_ops import reorg_packed
    with pytest.raises(ValueError):
        reorg_packed(scores, toff, ticks, sc, off[:-1] + [off[-1] + 1], STD_CFG, *lens(K))
    assert lib.ssnb_global_launch_count() == n0


# ---- end to end: two streams of a THUMOS14-like set, from the proposal list to the AP table ----------------------------------
def _thumos_like(seed, V=10, K=20):
    g = np.random.RandomState(seed)
    frame_cnt = g.randint(600, 4000, V).astype(np.int32)
    frame_cnt[3] = 7                                        # one tick
    counts = g.randint(100, 400, V)
    counts[5] = 0                                           # the fallback proposal only
    frames, gt = [], []
    for v in range(V):
        fc = int(frame_cnt[v])
        st = g.randint(0, max(fc - 2, 1), counts[v])
        ln = np.minimum(g.randint(2, max(fc // 3, 3), counts[v]), fc - st)
        frames.append(np.stack([st, st + np.maximum(ln, 1)], 1))
        for _ in range(g.randint(1, 6)):
            a = int(g.randint(0, fc - 2))
            b = min(fc, a + int(g.randint(2, max(fc // 4, 3))))
            gt.append(("video_%02d" % v, int(g.randint(1, K)), a / fc, b / fc))
    return np.concatenate(frames).astype(np.int64), counts, frame_cnt, gt


def test_two_streams_end_to_end_ap_bitwise():
    """test_proposals -> reorg_packed per stream -> fp32 weighted merge in torch -> detections_packed -> detection_ap, against
    evaluate_detections fed the dicts ssn_test.py saves (STPPReorgainzed.forward per video + the reference's de-normalisation)"""
    from ops.detection import DATASETS, detection_ap, detections_packed, evaluate_detections, pack_ground_truth
    from ops.proposal_lists import test_proposals
    from ops.ssn_ops import reorg_packed
    dev = _cuda()
    K, cfg = 20, STD_CFG
    frames, counts, frame_cnt, gt = _thumos_like(21, K=K)
    s = test_proposals(torch.from_numpy(frames).to(dev), counts, frame_cnt, new_length=1, test_interval=6)
    num_ticks = s["num_ticks"].cpu().tolist()
    toff = np.concatenate([[0], np.cumsum(num_ticks)]).tolist()
    off = s["offsets"]
    V = len(counts)
    vids = ["video_%02d" % v for v in range(V)]
    D = _D(K, cfg)
    stats = {"RGB": np.array([[0.0123, -0.0457], [0.1789, 0.2345]]), "Flow": np.array([[-0.0071, 0.0312], [0.1517, 0.2093]])}
    packed, dicts = {}, []
    for i, mod in enumerate(("RGB", "Flow")):
        scores = torch.randn(toff[-1], D, generator=torch.Generator(device=dev).manual_seed(100 + i), device=dev)
        packed[mod] = reorg_packed(scores, toff, s["ticks32"], s["scaling32"], off, cfg, *lens(K), reg_stats=stats[mod])
        d = {}
        for v, vid in enumerate(vids):
            lo, hi = off[v], off[v + 1]
            act, comp, reg = _single(scores[toff[v]:toff[v + 1]], s["proposal_ticks"][lo:hi], s["scaling"][lo:hi], K, cfg)
            reg_scores = _torch_denorm(reg, stats[mod], K)         # ssn_test.py:89-92
            d[vid] = (s["rel_prop"][lo:hi].cpu().numpy(), act.cpu().numpy(), comp.cpu().numpy(), reg_scores.cpu().numpy())
        dicts.append(d)
    # merged() of evaluate_detections on the packed tensors: x_0 * w_0 + x_1 * w_1 in fp32
    w = [0.5, 0.5]
    act, comp, reg = (packed["RGB"][i] * w[0] + packed["Flow"][i] * w[1] for i in range(3))
    ds = DATASETS["thumos14"]
    dets = detections_packed(s["rel_prop"].float(), act, comp, reg, off, ds["nms_threshold"], mode="top_k", top_k=ds["top_k"],
                             softmax_before_filter=ds["softmax_before_filter"])
    ap = detection_ap(dets, pack_ground_truth(gt, vids, dev), ds["iou_range"])["ap"].cpu().numpy()
    want = evaluate_detections(dicts, gt, "thumos14")["ap"]
    print("\nend to end: %d videos, %d proposals, mAP@0.5 %.4f" % (V, off[-1], float(np.nanmean(want[:, 4]))))
    assert ap.tobytes() == want.tobytes()
    assert np.isfinite(want).any() and (want > 0).any()
