"""Forward engines run at any frame count n up to the planned F, on the GPU: feat rows bitwise those of an engine planned
for n in every precision, RGB and Flow, InceptionV3 and BNInception; untouched output rows and poisoned workspaces;
alternating frame counts; CUDA-graph replay; the launch log's tile counts; and a ragged SSN.test_scores loop on one reserved
engine whose device memory does not grow.  Run on an H100: pytest -m gpu -s tests/test_gpu_ragged_frames.py."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import inception_v3_oracle as IV
from oracle import synth
from oracle import tile_plan as T
from ssn_b200 import _lib
from ssn_b200._lib import EXACT_FP32, FAST_FP16, EXACT_TC, lib

PRECISIONS = {"exact": EXACT_FP32, "exact_tc": EXACT_TC, "fast": FAST_FP16}
SIZE = {"InceptionV3": IV.INPUT_SIZE, "BNInception": 224}
FEAT = {"InceptionV3": IV.FEAT_DIM, "BNInception": 1024}
# frame counts around pick_box's frame boxes: bf = 2, 8, 32 and 128, and BNInception's 7 x 1 x 18 boxes of the 7x7 layers
N_SET = (1, 10, 37, 127, 128, 129, 255, 256, 257)
GRAD_SCALE = 1024.0
GIB = 1 << 30


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _free():
    gc.collect()
    torch.cuda.empty_cache()


_WEIGHTS = {}


def _weights(arch, cin):
    if (arch, cin) not in _WEIGHTS:
        _WEIGHTS[arch, cin] = IV.synth_weights(cin, seed=0) if arch == "InceptionV3" else synth.synth_backbone(cin, seed=0, calib_frames=2)
    return _WEIGHTS[arch, cin]


def _backbone(arch, cin, prec, dev):
    import model_zoo
    bm = getattr(model_zoo, arch)(in_channels=cin)
    sd = bm.state_dict()
    with torch.no_grad():
        for k, v in _weights(arch, cin).items():
            sd[k].copy_(v)
    bm = bm.to(dev).eval()
    bm.set_precision(PRECISIONS[prec], GRAD_SCALE)
    return bm


def _engine(bm, n, dev):
    """the forward-only engine a call of n frames runs on"""
    import model_zoo
    return bm.engine_for(n, dev) if isinstance(bm, model_zoo.InceptionV3) else bm.engine_for(n, False, dev)


def _frames_into(x, cin, seed):
    """uint8 - mean frames (oracle/synth.py's distribution), drawn on the device into x in place"""
    g = torch.Generator(device=x.device).manual_seed(1000 + seed)
    x.random_(0, 256, generator=g)
    return x.sub_(128.0 if cin != 3 else 117.0)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _fwd_frames(eng, x, n, feat):
    """the library's n-frame forward into a caller-sized feat (rows >= n must stay as they were)"""
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if hasattr(eng, "bn1_train"):
        rc = lib.ssnb_backbone_fwd_frames(eng.h, C.c_void_p(x.data_ptr()), n, C.c_void_p(feat.data_ptr()), s)
        _lib.check(rc, eng.h, "backbone_fwd_frames")
    else:
        _lib.check(lib.ssnb_iv3_forward_frames(eng.h, C.c_void_p(x.data_ptr()), n, C.c_void_p(feat.data_ptr()), s), None, "iv3_forward_frames")


def _need(bytes_, label):
    _free()
    free, _total = torch.cuda.mem_get_info()
    if bytes_ > free:
        pytest.skip("%s needs %.1f GiB, %.1f GiB are free" % (label, bytes_ / GIB, free / GIB))


@pytest.mark.parametrize("F", [400, 129])
@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("modality,cin", [("RGB", 3), ("Flow", 10)])
@pytest.mark.parametrize("arch", ["InceptionV3", "BNInception"])
def test_rows_bitwise_at_every_frame_count(arch, modality, cin, prec, F):
    """One engine planned for F runs n in {F, F - 1} and N_SET (n <= F): its feat rows are bitwise those of a fresh engine
    planned for n, feat rows >= n keep their sentinel, a workspace filled with 0xFF (NaN in fp16 and fp32) after a run at F
    changes no bit, F -> 37 -> F calls are stable, and a CUDA graph captured at n replays an eager call bitwise on new frames."""
    dev = _dev()
    D, S = FEAT[arch], SIZE[arch]
    ns = sorted({n for n in (F, F - 1) + N_SET if n <= F})
    bm = _backbone(arch, cin, prec, dev)
    _need(_engine_bytes(arch, cin, prec, F) + 3 * F * cin * S * S * 4 + GIB, "%s %s F=%d" % (arch, prec, F))
    x = _frames_into(torch.empty(F, cin, S, S, device=dev), cin, 1)
    bm.reserve_frames(F)
    eng = _engine(bm, 37, dev)
    assert eng.frames == F and len(bm._engines) == 1
    sentinel = torch.tensor(-1234567.0, device=dev)
    got = {}
    for n in ns:
        feat = torch.full((F, D), -1234567.0, device=dev)
        _fwd_frames(eng, x[:n], n, feat)
        assert torch.equal(_bits(feat[n:]), _bits(sentinel.expand(F - n, D))), "n=%d wrote feat rows >= n" % n
        got[n] = feat[:n].clone()
        assert torch.equal(_bits(eng.forward(x[:n])), _bits(got[n])), "Python forward at n=%d" % n
    # F -> 37 -> F on the one engine
    a = eng.forward(x).clone()
    b = eng.forward(x[:37]).clone()
    c = eng.forward(x).clone()
    assert torch.equal(_bits(a), _bits(c)) and torch.equal(_bits(b), _bits(got[37])) and torch.equal(_bits(a), _bits(got[F]))
    # 0xFF over the whole workspace after the run at F (the packed weights re-packed), then n < F: rows < n are unchanged
    eng._ws.fill_(0xFF)
    eng.packed_version = None
    assert _engine(bm, 1, dev) is eng
    for n in (1, 37, F - 1):
        feat = torch.full((F, D), -1234567.0, device=dev)
        _fwd_frames(eng, x[:n], n, feat)
        assert torch.equal(_bits(feat[:n]), _bits(got[n])), "poisoned workspace, n=%d" % n
        assert torch.equal(_bits(feat[n:]), _bits(sentinel.expand(F - n, D)))
    # a CUDA graph captured at n = 37 and replayed on other frames equals an eager call
    static_x = x[:37].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.forward(static_x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static_out = eng.forward(static_x)
    static_x.copy_(x[F - 37:].flip(0))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(static_out), _bits(eng.forward(static_x)))
    del g, static_out, eng
    # the reference: a fresh engine planned for each n, one at a time (InceptionV3 EXACT_TC plans 42.6 GB at 400 frames)
    bm.reserve_frames(None)
    bm._engines.clear()
    _free()
    bad = []
    for n in ns:
        ref = _engine(bm, n, dev).forward(x[:n])
        assert _engine(bm, n, dev).frames == n
        if not torch.equal(_bits(ref), _bits(got[n])):
            rows = [i for i in range(n) if not torch.equal(_bits(ref[i]), _bits(got[n][i]))]
            bad.append("n=%d: %d rows differ (first %d, max |diff| %.2e)" % (n, len(rows), rows[0], float((ref[rows[0]] - got[n][rows[0]]).abs().max())))
        del ref
        bm._engines.clear()
        _free()
    print("\n%s %s %s F=%d: n = %s bitwise against engines planned for n%s" % (arch, modality, prec, F, ns, "; ".join([""] + bad)))
    assert not bad, "\n".join(bad)


def _engine_bytes(arch, cin, prec, F):
    if arch == "InceptionV3":
        from ssn_b200.inception_v3 import InceptionV3Engine
        return int(InceptionV3Engine(cin, F, PRECISIONS[prec]).workspace_bytes)
    from ssn_b200.engine import BackboneEngine
    return int(BackboneEngine(cin, F, PRECISIONS[prec], False, GRAD_SCALE, None).workspace_bytes)


@pytest.mark.parametrize("prec", ["exact_tc", "fast"])
@pytest.mark.parametrize("arch", ["InceptionV3", "BNInception"])
def test_launch_log_tiles_follow_n(arch, prec):
    """At n = 37 and 129 on a 400-frame engine every umma_conv_kernel launch has n's tile count, ceil(n / bf) x tiles_h x
    tiles_w x N tiles with the box the plan chose (oracle/tile_plan.py), and the launches of an engine planned for n"""
    dev = _dev()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = SIZE[arch]
    bm = _backbone(arch, 3, prec, dev)
    _need(_engine_bytes(arch, 3, prec, 400) + 129 * 3 * S * S * 4 + GIB, "%s %s F=400" % (arch, prec))
    bm.reserve_frames(400)
    x = _frames_into(torch.empty(129, 3, S, S, device=dev), 3, 2)
    schedule = (lambda f: T.iv3_schedule(f, prec, sms)) if arch == "InceptionV3" else (lambda f: T.schedule(3, f, prec, sms, training=False))
    full = sum(l["plan"]["total"] for l in schedule(400))
    for n in (37, 129):
        eng = _engine(bm, n, dev)
        eng.forward(x[:n])
        torch.cuda.synchronize()
        lib.ssnb_timing_begin(C.c_void_p(torch.cuda.current_stream().cuda_stream))
        eng.forward(x[:n])
        got = T.parse_launch_log(lib.ssnb_timing_launches().decode())
        plan = schedule(n)
        for l in plan:
            p = l["plan"]
            assert p["total"] == -(-n // p["box"][2]) * p["tiles_h"] * p["tiles_w"] * p["n_tiles"]
        want = [T.log_key(l) for l in plan]
        bad = [(i, g_, w) for i, (g_, w) in enumerate(zip(got, want)) if g_ != w]
        assert len(got) == len(want) and not bad, (n, len(got), len(want), bad[:5])
        print("\n%s %s n=%d on a 400-frame engine: %d launches, %d tiles in all (%d at 400 frames)"
              % (arch, prec, n, len(got), sum(g_[3] for g_ in got), full))
        assert sum(g_[3] for g_ in got) < full


CHUNK_TICKS, CROPS, VIDEOS = 40, 10, 30


def _ssn(arch, prec, dev, K=4):
    import ssn_models
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model=arch, dropout=0, test_mode=True)
    sd = m.state_dict()
    with torch.no_grad():
        for k, v in _weights(arch, 3).items():
            sd["base_model." + k].copy_(v)
        for k, v in synth.synth_heads(K, m.stpp.feat_multiplier, feat_dim=FEAT[arch], seed=0, std=0.02, bias_std=0.1).items():
            sd[k].copy_(v)
    m.prepare_test_fc()
    m.set_precision(PRECISIONS[prec], GRAD_SCALE)
    return m.to(dev).eval()


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("arch", ["InceptionV3", "BNInception"])
def test_ragged_test_scores_loop_on_one_engine(arch, prec):
    """ssn_test.py's loop over 30 videos of 41-400 ticks in 40-tick chunks of 10 crops after reserve_frames(400): one engine
    serves every chunk, torch.cuda.memory_allocated does not move after the first call, and every tail chunk's scores are
    bitwise those of an engine planned for its frame count (full chunks: a fresh 400-frame engine, first three videos)"""
    dev = _dev()
    S, F = SIZE[arch], CHUNK_TICKS * CROPS
    _need(_engine_bytes(arch, 3, prec, F) + 2 * F * 3 * S * S * 4 + GIB, "%s %s F=%d" % (arch, prec, F))
    m = _ssn(arch, prec, dev)
    ticks = np.random.default_rng(5).integers(41, 401, VIDEOS)
    chunks = [(v, c, min(CHUNK_TICKS, int(t) - c)) for v, t in enumerate(ticks) for c in range(0, int(t), CHUNK_TICKS)]
    xbuf = torch.empty(F, 3, S, S, device=dev)
    m.base_model.reserve_frames(F)
    got, mem0 = {}, None
    for v, c, nt in chunks:
        x = _frames_into(xbuf[:nt * CROPS], 3, 7919 * v + c)
        got[v, c] = m.test_scores(x, num_crop=CROPS).cpu()
        assert len(m.base_model._engines) == 1
        if mem0 is None:
            mem0 = torch.cuda.memory_allocated()
        assert torch.cuda.memory_allocated() == mem0, (v, c, nt, torch.cuda.memory_allocated() - mem0)
    (eng,) = m.base_model._engines.values()
    assert eng.frames == F
    tails = sorted({nt for _, _, nt in chunks if nt < CHUNK_TICKS})
    print("\n%s %s: %d chunks of %d videos, %d distinct tail sizes on one %.1f GB engine; memory_allocated %.2f GB throughout"
          % (arch, prec, len(chunks), VIDEOS, len(tails), eng.workspace_bytes / 1e9, mem0 / 1e9))
    del eng
    m.base_model.reserve_frames(None)
    m.base_model._engines.clear()
    _free()
    bad = []
    for nt in tails + [CHUNK_TICKS]:
        for v, c, k in chunks:
            if k != nt or (nt == CHUNK_TICKS and v >= 3):
                continue
            x = _frames_into(xbuf[:nt * CROPS], 3, 7919 * v + c)
            ref = m.test_scores(x, num_crop=CROPS).cpu()
            if not torch.equal(_bits(ref), _bits(got[v, c])):
                bad.append("video %d chunk %d (%d ticks): max |diff| %.2e" % (v, c, nt, float((ref - got[v, c]).abs().max())))
        assert next(iter(m.base_model._engines.values())).frames == nt * CROPS
        m.base_model._engines.clear()
        _free()
    assert not bad, "\n".join(bad[:10])
