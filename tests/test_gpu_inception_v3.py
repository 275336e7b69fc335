"""InceptionV3 at test time on the GPU: every launch against float64 on the operands it consumed, the whole backbone and
the SSN / BinaryClassifier surface against the reference's golden, repeatability, CUDA-graph replay, the refusals, and the
299 / 341 frame transforms against PIL."""
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


@pytest.mark.parametrize("prec", ["exact", "exact_tc", "fast"])
@pytest.mark.parametrize("cin,F", [(3, 10), (10, 10), (3, 37), (10, 37), (3, 1), (10, 1), (3, 400), (10, 400)])
def test_every_launch_vs_float64(cin, F, prec):
    """After one forward every value still holds what its producer wrote (the engine reuses no buffer), so each op is checked
    on the exact operands its kernel consumed.  F = 400: the first and last four frames are compared."""
    dev = _dev()
    modality = "RGB" if cin == 3 else "Flow"
    m = _ssn("x", modality, cin, 3, dev, prec)
    bm = m.base_model
    x = synth.synth_frames(F, cin, IV.INPUT_SIZE, seed=5).to(dev)
    with torch.no_grad():
        feat = bm(x)
    eng = bm.engine_for(F, dev)
    sl = list(range(F)) if F <= 37 else list(range(4)) + list(range(F - 4, F))
    convs = {n[:-len("_Conv2D")]: (getattr(bm, n), getattr(bm, n[:-len("_Conv2D")] + "_batchnorm")) for n in bm._conv_names}
    kinds = set()
    worst = (0.0, 0.0, "")
    for (kind, inp, out, _c, k, stride, pad) in eng.ops():
        xin = eng.read(inp)[sl].double()
        if kind == "gpool":
            y, ref = feat[sl], xin.mean((2, 3))
            bar = AVGPOOL_BAR["exact"]           # an fp32 sum of the stored values, in every precision
        else:
            y = eng.read(out)[sl]
            if kind == "conv":
                conv, bn = convs[out]
                s = bn.weight.double() / torch.sqrt(bn.running_var.double() + 1e-5)
                w = conv.weight.double() * s.view(-1, 1, 1, 1)
                b = (conv.bias.double() - bn.running_mean.double()) * s + bn.bias.double()
                ref = torch.relu(Fn.conv2d(xin, w, b, conv.stride, conv.padding))
                bar = CONV_BAR[prec]
                kinds.add((tuple(conv.kernel_size), conv.stride[0], conv.padding != (conv.kernel_size[0] // 2, conv.kernel_size[1] // 2)))
            elif kind == "maxpool":
                ref, bar = Fn.max_pool2d(xin, k, stride, pad, ceil_mode=True), 0.0
            else:
                ref, bar = Fn.avg_pool2d(xin, k, stride, pad, ceil_mode=True), AVGPOOL_BAR[prec]
            if prec == "exact_tc":               # the operand planes the next convolution reads
                err = _rel(eng.read(out, planes=True)[sl], y)
                assert err <= PLANES_BAR, ("planes", kind, out, F, cin, err)
        err = _rel(y, ref)
        worst = max(worst, (err / bar, err, out)) if bar > 0 else worst
        assert err <= bar, (prec, kind, out, F, cin, err)
    # the stem, valid stride-1 / stride-2, 5x5 and every asymmetric shape were among the checked launches
    for need in (((3, 3), 2, True), ((3, 3), 1, True), ((5, 5), 1, False), ((1, 7), 1, False), ((7, 1), 1, False),
                 ((1, 3), 1, False), ((3, 1), 1, False)):
        assert need in kinds, need
    print("InceptionV3 %s F=%d cin=%d: worst launch %s %.2e" % (prec, F, cin, worst[2], worst[1]))
    del m, bm, eng, feat
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
