"""InceptionV3 at test time on the GPU: every launch against float64 on the operands it consumed, the whole backbone and
the SSN / BinaryClassifier surface against the reference's golden, repeatability, CUDA-graph replay, the refusals, and the
299 / 341 frame transforms against PIL."""
import ctypes as C
import gc
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

from oracle import inception_v3_oracle as IV
from oracle import synth, binary_oracle as B
from oracle import tile_plan as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = (("rgb", "RGB", 3, 4, 11), ("flow", "Flow", 10, 3, 12))     # as oracle/gen_golden_inception_v3.py
from ssn_b200._lib import EXACT_FP32, FAST_FP16, EXACT_TC
PRECISIONS = {"exact": EXACT_FP32, "exact_tc": EXACT_TC, "fast": FAST_FP16}
# per launch, the forward bars of the BNInception schedule check: convolution rel-L2, avg pool to the rounding of its stored
# result (fp32 / fp16), EXACT_TC operand planes against the fp32 value; max pools bitwise
CONV_BAR = {"exact": 5e-6, "exact_tc": 1.5e-5, "fast": 3e-3}
AVGPOOL_BAR = {"exact": 1e-6, "exact_tc": 1e-6, "fast": 1e-3}
PLANES_BAR = 2e-6
# whole backbone / module surface against the reference golden: EXACT 1e-4, EXACT_TC 5e-4; FAST (fp16 operands) is reported
# and only sanity-checked, as for BNInception
WHOLE_BAR = {"exact": 1e-4, "exact_tc": 5e-4, "fast": 5e-2}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_weights = {}


def _ssn(tag, modality, cin, K, dev, prec="exact"):
    import ssn_models
    if cin not in _weights:
        _weights[cin] = IV.synth_weights(cin, seed=0)
    m = ssn_models.SSN(K, 2, 5, 2, modality, base_model="InceptionV3", dropout=0, test_mode=True)
    sd = m.state_dict()
    with torch.no_grad():
        for k, v in _weights[cin].items():
            sd["base_model." + k].copy_(v)
        for k, v in synth.synth_heads(K, m.stpp.feat_multiplier, feat_dim=IV.FEAT_DIM, seed=0, std=0.02, bias_std=0.1).items():
            sd[k].copy_(v)
    m.prepare_test_fc()
    m.set_precision(PRECISIONS[prec])
    return m.to(dev).eval()


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ---- memory guard (the pattern of tests/test_gpu_tile_regimes.py) ------------------------------------------------------
GIB = 1 << 30
CHUNK = 16                                        # frames per float64 slice of the per-launch check


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def workspace_bytes(prec, frames, cin):
    """ssnb_iv3_workspace_bytes of the engine's plan (no device memory is touched)"""
    from ssn_b200.inception_v3 import InceptionV3Engine
    return int(InceptionV3Engine(cin, frames, PRECISIONS[prec]).workspace_bytes)


def check_peak_bytes(frames, cin):
    """what a per-launch check holds besides the workspace, at most: the input and feat, the op's input, output
    and (EXACT_TC) output planes read back in fp32 -- at most three copies of the largest value (conv_2: 64 x 147 x 147) --
    and the float64 slices of CHUNK frames with ATen's convolution workspace (in the fixed 2 GiB)"""
    largest = 64 * 147 * 147 * 4
    return frames * (3 * largest + cin * IV.INPUT_SIZE ** 2 * 4 + IV.FEAT_DIM * 4) + 2 * GIB


def _need_memory(label, ws, check):
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if ws + check > free:
        pytest.skip("%s needs %.1f GiB (workspace %.1f GiB + check %.1f GiB), %.1f GiB of %.1f GiB are free"
                    % (label, (ws + check) / GIB, ws / GIB, check / GIB, free / GIB, total / GIB))


def _launches_predicted(log, F, prec, sms):
    """the umma_conv_kernel launches of one forward equal tile_plan.iv3_schedule's, in order; returns the plan"""
    got = T.parse_launch_log(log)
    if prec == "exact":
        assert got == [], got[:5]
        return []
    plan = T.iv3_schedule(F, prec, sms)
    want = [T.log_key(l) for l in plan]
    bad = [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert len(got) == len(want) and not bad, \
        "%d launches logged, %d predicted; first differences (index, logged, predicted): %s" % (len(got), len(want), bad[:5])
    return plan


class _RelL2:
    """rel-L2 of a tensor accumulated over frame slices: ||got - ref|| / ||ref||"""

    def __init__(self):
        self.d = self.r = 0.0

    def add(self, got, ref):
        self.d += float(((got.double() - ref) ** 2).sum())
        self.r += float((ref ** 2).sum())

    def value(self):
        return (self.d / max(self.r, 1e-300)) ** 0.5


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("cin,F", [(3, 10), (10, 10), (3, 37), (10, 37), (3, 1), (10, 1), (3, 400), (10, 400), (3, 89), (3, 129)])
def test_every_launch_vs_float64(cin, F, prec):
    """After one forward every value still holds what its producer wrote (the engine reuses no buffer), so each op is checked
    on the exact operands its kernel consumed, over every frame in float64 slices of CHUNK frames.  The tensor-core modes'
    launch log (tiles, tile width per convolution) is held to tile_plan.iv3_schedule on this device's SM count.  F = 89 and
    129 reach the tile regimes the others miss (tile_plan.IV3_FRAME_SET); the plans do not depend on the modality."""
    from ssn_b200._lib import lib
    dev = _dev()
    label = "InceptionV3 %s F=%d cin=%d" % (prec, F, cin)
    ws = workspace_bytes(prec, F, cin)
    allowed = check_peak_bytes(F, cin)
    _need_memory(label, ws, allowed)
    sms = _sms()
    modality = "RGB" if cin == 3 else "Flow"
    m = _ssn("x", modality, cin, 3, dev, prec)
    bm = m.base_model
    x = synth.synth_frames(F, cin, IV.INPUT_SIZE, seed=5).to(dev)
    eng = bm.engine_for(F, dev)
    assert eng.workspace_bytes == ws
    torch.cuda.synchronize()
    lib.ssnb_timing_begin(C.c_void_p(torch.cuda.current_stream().cuda_stream))
    feat = eng.forward(x)
    log = lib.ssnb_timing_launches().decode()
    torch.cuda.synchronize()
    plan = _launches_predicted(log, F, prec, sms)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    convs = {n[:-len("_Conv2D")]: (getattr(bm, n), getattr(bm, n[:-len("_Conv2D")] + "_batchnorm")) for n in bm._conv_names}
    kinds = set()
    worst = (0.0, 0.0, "")
    worst_planes = 0.0
    for (kind, inp, out, _c, k, stride, pad) in eng.ops():
        xin_all = eng.read(inp)
        y_all = feat if kind == "gpool" else eng.read(out)
        planes_all = eng.read(out, planes=True) if prec == "exact_tc" and kind != "gpool" else None
        err, perr, equal = _RelL2(), _RelL2(), True
        if kind == "conv":
            conv, bn = convs[out]
            s = bn.weight.double() / torch.sqrt(bn.running_var.double() + 1e-5)
            w = conv.weight.double() * s.view(-1, 1, 1, 1)
            b = (conv.bias.double() - bn.running_mean.double()) * s + bn.bias.double()
            kinds.add((tuple(conv.kernel_size), conv.stride[0], conv.padding != (conv.kernel_size[0] // 2, conv.kernel_size[1] // 2)))
        for f0 in range(0, F, CHUNK):
            sl = slice(f0, min(F, f0 + CHUNK))
            xin, y = xin_all[sl].double(), y_all[sl]
            if kind == "gpool":
                ref = xin.mean((2, 3))
            elif kind == "conv":
                ref = torch.relu(Fn.conv2d(xin, w, b, conv.stride, conv.padding))
            elif kind == "maxpool":
                ref = Fn.max_pool2d(xin, k, stride, pad, ceil_mode=True)
                equal = equal and torch.equal(y.double(), ref)
            else:
                ref = Fn.avg_pool2d(xin, k, stride, pad, ceil_mode=True)
            err.add(y, ref)
            if planes_all is not None:                # the operand planes the next convolution reads
                perr.add(planes_all[sl], y.double())
            del xin, ref
        bar = AVGPOOL_BAR["exact"] if kind == "gpool" else CONV_BAR[prec] if kind == "conv" else 0.0 if kind == "maxpool" \
            else AVGPOOL_BAR[prec]          # gpool: an fp32 sum of the stored values, in every precision; max pools bitwise
        e = err.value()
        if bar > 0:
            worst = max(worst, (e / bar, e, out))
            assert e <= bar, (prec, kind, out, F, cin, e)
        else:
            assert equal, (prec, kind, out, F, cin, e)
        if planes_all is not None:
            worst_planes = max(worst_planes, perr.value())
            assert perr.value() <= PLANES_BAR, ("planes", kind, out, F, cin, perr.value())
        del xin_all, y_all, planes_all
    peak = torch.cuda.max_memory_allocated() - base + (x.numel() + feat.numel()) * 4
    # the stem, valid stride-1 / stride-2, 5x5 and every asymmetric shape were among the checked launches
    for need in (((3, 3), 2, True), ((3, 3), 1, True), ((5, 5), 1, False), ((1, 7), 1, False), ((7, 1), 1, False),
                 ((1, 3), 1, False), ((3, 1), 1, False)):
        assert need in kinds, need
    print("\n%s on %d SMs: %s; worst launch %s %.2e (%.2f of its bar)%s; memory: workspace %.1f GiB, check %.2f GiB "
          "measured / %.2f GiB allowed" % (label, sms, "%d umma launches as planned" % len(plan) if plan else "no umma launch",
                                           worst[2], worst[1], worst[0],
                                           ", planes %.1e" % worst_planes if prec == "exact_tc" else "", ws / GIB, peak / GIB,
                                           allowed / GIB))
    assert peak <= allowed, "the memory guard's estimate of the check is too small: %.2f GiB measured" % (peak / GIB)
    del m, bm, eng, feat
    gc.collect()
    torch.cuda.empty_cache()                      # EXACT_TC at F = 400 plans 42.6 GB; the next case plans its own


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("tag,modality,cin,K,seed", CASES)
def test_module_surface_vs_reference_golden(tag, modality, cin, K, seed, prec):
    import binary_model
    dev = _dev()
    a = np.load(os.path.join(GOLD, "inception_v3.npz"))
    m = _ssn(tag, modality, cin, K, dev, prec)
    bar = WHOLE_BAR[prec]
    x = synth.synth_frames(10, cin, IV.INPUT_SIZE, seed=seed).to(dev)
    with torch.no_grad():
        out, base_out = m(x, None, None, None, None)
    assert _rel(base_out, torch.from_numpy(a[tag + "_base_out"]).to(dev)) <= bar
    assert _rel(out, torch.from_numpy(a[tag + "_test_fc"]).to(dev)) <= bar
    # test_scores: 10 crops of one tick, crop mean folded into the test FC
    sc = m.test_scores(x, num_crop=10)
    want = torch.from_numpy(a[tag + "_test_fc"]).double().mean(0, keepdim=True).to(dev)
    assert sc.shape == want.shape and _rel(sc, want) <= bar
    bc = binary_model.BinaryClassifier(2, 5, modality, base_model="InceptionV3", dropout=0, test_mode=True)
    bsd = bc.state_dict()
    with torch.no_grad():
        for k, v in _weights[cin].items():
            bsd["base_model." + k].copy_(v)
        for k, v in B.synth_classifier(2, feat_dim=IV.FEAT_DIM, seed=0).items():
            bsd[k].copy_(v)
    bc.prepare_test_fc()
    bc.set_precision(PRECISIONS[prec])
    bc = bc.to(dev).eval()
    with torch.no_grad():
        scores, _ = bc(x, None)
    assert _rel(scores, torch.from_numpy(a[tag + "_binary_scores"]).to(dev)) <= bar
    print("InceptionV3 %s %s vs reference: base_out %.2e, test_fc %.2e, binary %.2e"
          % (tag, prec, _rel(base_out, torch.from_numpy(a[tag + "_base_out"]).to(dev)), _rel(out, torch.from_numpy(a[tag + "_test_fc"]).to(dev)),
             _rel(scores, torch.from_numpy(a[tag + "_binary_scores"]).to(dev))))


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
def test_repeat_poisoned_workspace_and_graph_replay(prec):
    dev = _dev()
    m = _ssn("rgb", "RGB", 3, 4, dev, prec)
    bm = m.base_model
    x = synth.synth_frames(37, 3, IV.INPUT_SIZE, seed=9).to(dev)
    with torch.no_grad():
        f1 = bm(x).clone()
        f2 = bm(x).clone()
        assert torch.equal(f1, f2)
        eng = bm.engine_for(37, dev)
        start = eng.ws_ptr - eng._ws.data_ptr()
        eng._ws[start:].fill_(0xFF)              # activations, arg-max and the packed weights: everything is rewritten
        eng.packed_version = None
        f3 = bm(x).clone()
        assert torch.equal(f1, f3)
        static_x = x.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            bm(static_x)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            static_out = bm(static_x)
        static_x.copy_(synth.synth_frames(37, 3, IV.INPUT_SIZE, seed=10).to(dev))
        g.replay()
        torch.cuda.synchronize()
        eager = bm(static_x)
        assert torch.equal(static_out, eager)


def test_gradients_and_training_refused_without_launch():
    from ssn_b200._lib import lib
    dev = _dev()
    m = _ssn("rgb", "RGB", 3, 4, dev)
    x = synth.synth_frames(2, 3, IV.INPUT_SIZE, seed=1).to(dev)
    n0 = lib.ssnb_global_launch_count()
    with pytest.raises(NotImplementedError, match="follow-up"):
        m.base_model(x)                           # grad mode on, parameters require grad
    with pytest.raises(NotImplementedError, match="follow-up"):
        m.fused_step(x, None, None, None, None)
    m.train()
    m.base_model.conv_batchnorm.train()           # a training-mode BatchNorm2d (bn_mode 'partial')
    with torch.no_grad(), pytest.raises(NotImplementedError, match="follow-up"):
        m.base_model(x)
    assert lib.ssnb_global_launch_count() == n0


def test_frame_transforms_299_341_bitwise_vs_pil():
    from oracle.gen_golden_frames import frames_for
    from ops.frame_transforms import oversample_frames, center_crop_frames
    import ssn_models
    _dev()
    with open(os.path.join(GOLD, "inception_v3.json")) as f:
        cases = json.load(f)["frames"]
    for name, case in sorted(cases.items()):
        frames = frames_for(case["seed"], *case["shape"])
        c = frames.shape[3]
        x = torch.from_numpy(frames)
        if case["kind"] == "oversample":
            out = oversample_frames(x, case["mean"], [1], c, crop_size=299, scale_size=341)
        else:
            out = center_crop_frames(x, case["mean"], [1], c, crop_size=299, scale_size=341)
        got = out.cpu().numpy()
        assert int(np.prod(got.shape)) == int(np.prod(case["out_shape"])), name
        assert hashlib.sha256(got.reshape(-1).tobytes()).hexdigest() == case["sha256"], name
    # the model's frame_transforms() carry 299 / 341
    m = ssn_models.SSN(3, 2, 5, 2, "RGB", base_model="InceptionV3", dropout=0, test_mode=True)
    t = m.frame_transforms()
    assert t.oversample.keywords["crop_size"] == 299 and t.oversample.keywords["scale_size"] == 341
    assert t.center_crop.keywords["crop_size"] == 299 and t.center_crop.keywords["scale_size"] == 341


# ---- frame independence --------------------------------------------------------------------------------------------------
INDEP_FRAMES = (400, 129, 37, 1)


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
def test_frame_rows_independent_of_frame_count_and_position(prec):
    """The same frames through engines planned for F = 400, 129, 37 and 1, each at other positions (and so in other pixel
    tiles and frame boxes): their feat rows are bitwise equal.  Not a documented guarantee, but what row-independent MMAs
    and per-frame pools give; where an H100 showed otherwise, the rows would be held to the per-launch bars instead."""
    dev = _dev()
    m = _ssn("rgb", "RGB", 3, 4, dev, prec)
    bm = m.base_model
    x = synth.synth_frames(400, 3, IV.INPUT_SIZE, seed=21).to(dev)
    # rows of the F = 400 run each smaller engine takes, in its own order: the last 129 reversed (frame 399 at position 0,
    # frame 271 alone in the second 128-frame box), every 11th frame from 3 on, then frame 128
    picks = {400: list(range(400)), 129: list(range(399, 270, -1)), 37: list(range(3, 400, 11)), 1: [128]}
    feats = {}
    for F in INDEP_FRAMES:
        ws = workspace_bytes(prec, F, 3)
        _need_memory("InceptionV3 %s F=%d" % (prec, F), ws, F * 3 * IV.INPUT_SIZE ** 2 * 4 + GIB)
        with torch.no_grad():
            feats[F] = bm.engine_for(F, dev).forward(x[picks[F]]).clone()
        bm._engines.clear()                          # one engine at a time: EXACT_TC at F = 400 plans 42.6 GB
        gc.collect()
        torch.cuda.empty_cache()
    bad = []
    for F in INDEP_FRAMES[1:]:
        ref = feats[400][picks[F]]
        if not torch.equal(feats[F], ref):
            rows = [i for i in range(F) if not torch.equal(feats[F][i], ref[i])]
            bad.append("F=%d: %d of %d rows differ (first: position %d = frame %d, max |diff| %.2e, rel-L2 %.2e)"
                       % (F, len(rows), F, rows[0], picks[F][rows[0]], float((feats[F][rows[0]] - ref[rows[0]]).abs().max()),
                          _rel(feats[F][rows[0]], ref[rows[0]])))
    print("\nInceptionV3 %s: feat rows of F = 129 / 37 / 1 against F = 400: %s" % (prec, "; ".join(bad) if bad else "bitwise"))
    assert not bad, "\n".join(bad)


# ---- the benchmarked call end to end -------------------------------------------------------------------------------------
TICKS, CROPS = 40, 10
_FEAT64 = {}


def _feat64(cin, x):
    """float64 oracle forward (oracle/inception_v3_oracle.forward) of the 400 frames, 40 at a time"""
    if cin not in _FEAT64:
        p = {k: v.to(x.device) for k, v in _weights[cin].items()}
        with torch.no_grad():
            _FEAT64[cin] = torch.cat([IV.forward(p, x[i:i + 40], cin, torch.float64) for i in range(0, x.shape[0], 40)])
        torch.cuda.empty_cache()
    return _FEAT64[cin]


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("K", [20, 200])
@pytest.mark.parametrize("modality,cin", [("RGB", 3), ("Flow", 10)])
def test_benchmarked_call_vs_float64(modality, cin, K, prec):
    """SSN(..., 'InceptionV3').test_scores at 40 ticks x 10 crops (400 frames, what tools/bench_inception_v3.py times) and
    BinaryClassifier scoring of the same frames, against the float64 oracle forward with the folded test FC and the crop
    mean, at the whole-backbone bars; FAST is reported and held to its sanity bar"""
    import binary_model
    dev = _dev()
    F = TICKS * CROPS
    ws = workspace_bytes(prec, F, cin)
    _need_memory("InceptionV3 %s %s F=%d" % (prec, modality, F), ws, F * cin * IV.INPUT_SIZE ** 2 * 4 + 6 * GIB)
    m = _ssn(modality.lower(), modality, cin, K, dev, prec)
    x = synth.synth_frames(F, cin, IV.INPUT_SIZE, seed=31).to(dev)
    sc = m.test_scores(x, num_crop=CROPS)
    torch.cuda.synchronize()
    m.base_model._engines.clear()
    bc = binary_model.BinaryClassifier(2, 5, modality, base_model="InceptionV3", dropout=0, test_mode=True)
    bsd = bc.state_dict()
    with torch.no_grad():
        for k, v in _weights[cin].items():
            bsd["base_model." + k].copy_(v)
        for k, v in B.synth_classifier(2, feat_dim=IV.FEAT_DIM, seed=0).items():
            bsd[k].copy_(v)
    bc.prepare_test_fc()
    bc.set_precision(PRECISIONS[prec])
    bc = bc.to(dev).eval()
    with torch.no_grad():
        scores, _ = bc(x, None)
    torch.cuda.synchronize()
    bc.base_model._engines.clear()
    gc.collect()
    torch.cuda.empty_cache()
    feat = _feat64(cin, x)
    W, b = m.test_fc.weight.double(), m.test_fc.bias.double()
    want = (feat @ W.t() + b).view(CROPS, TICKS, -1).mean(0)
    bwant = feat @ bc.test_fc.weight.double().t() + bc.test_fc.bias.double()
    e, eb = _rel(sc, want), _rel(scores, bwant)
    print("\nInceptionV3 %s %s K=%d, %d ticks x %d crops: test_scores %s rel-L2 %.2e, BinaryClassifier scores %.2e (bar %.0e)"
          % (prec, modality, K, TICKS, CROPS, tuple(sc.shape), e, eb, WHOLE_BAR[prec]))
    assert sc.shape == want.shape and scores.shape == bwant.shape
    assert e <= WHOLE_BAR[prec] and eb <= WHOLE_BAR[prec], (e, eb)
