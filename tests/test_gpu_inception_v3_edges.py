"""The InceptionV3 engine at the inputs the continuous synthetic data never produce, in every precision: exact ties (+-0
among them), NaN and +-inf in every pool op of its own, non-finite pixels and a NaN weight through the whole backbone, and
an input that drives activations past the fp16 range.  The rules are DESIGN.md's (section 2, "Non-finite values"), which
tests/test_gpu_glue_edges.py checks on BNInception.  Run on an H100: pytest -m gpu -s tests/test_gpu_inception_v3_edges.py.

A  every max / average pool op alone (write -> run_op -> read) at F = 1 and 37 against float64 ATen: the 3x3/2 unpadded
   max pools on odd sizes, the padded 3x3/1 max pool at 8x8 (mixed_10), the 3x3 average pools at 35, 17 and 8;
B  one non-finite pixel per poisoned frame at a corner, an edge and the interior of the 299 input, at F = 37 (every frame in
   one frame box) and F = 129 (the poisoned frame alone in the second 128-frame box of the 1x1x128 tiles): the other frames'
   feat is bitwise that of a clean run and at every op the poisoned frame is non-finite exactly where float64 of the op's
   consumed input is;
C  a NaN weight in a 5x5 and in a 7x1 layer; a bright patch whose stem activations pass 65504.
"""
import gc
import math

import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

from oracle import inception_v3_oracle as IV
from oracle import synth
from oracle.edge_inputs import edge_input, same, same_bits, nonfinite_masks_equal

PRECISIONS = ("exact", "exact_tc", "fast")
NAN, INF = math.nan, math.inf
AVGPOOL_BAR = {"exact": 1e-6, "exact_tc": 1e-6, "fast": 1e-3}    # tests/test_gpu_inception_v3.py's per-launch bars
PLANES_BAR = 2e-6
FP16_INF_FROM = 65520.0            # the smallest magnitude fp16 rounds to inf: an fp16 value or operand plane is non-finite


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_WEIGHTS = {}


def _weights():
    if "synth" not in _WEIGHTS:
        _WEIGHTS["synth"] = IV.synth_weights(3, seed=0)
    return _WEIGHTS["synth"]


def _engine(precision, frames, params, dev):
    from ssn_b200 import _lib
    from ssn_b200.inception_v3 import InceptionV3Engine
    prec = {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]
    eng = InceptionV3Engine(3, frames, prec, dev)
    _pack(eng, params, dev)
    return eng


def _names():
    from ssn_b200.inception_v3 import conv_table
    return [c[0] for c in conv_table(3)]


def _pack(eng, p, dev):
    n = _names()
    eng.pack(*[[p[k + suf].to(dev) for k in n] for suf in ("_Conv2D.weight", "_Conv2D.bias", "_batchnorm.weight", "_batchnorm.bias",
                                                             "_batchnorm.running_mean", "_batchnorm.running_var")])


def _release(eng):
    del eng
    gc.collect()
    torch.cuda.empty_cache()


# ---- A: every pool op on its own ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("frames", [1, 37])
def test_pool_ops_on_ties_and_non_finite(precision, frames):
    """max pools bitwise against float64 ATen (the sign of every zero and the NaN positions included); average pools at the
    per-launch bar on the finite values with the NaN / +inf / -inf positions exact; EXACT_TC: the operand planes the pool
    writes for the next convolution are non-finite exactly where the value is and equal it where it is finite (max pools
    exactly, average pools at the planes bar)"""
    dev = _cuda()
    eng = _engine(precision, frames, _weights(), dev)
    pools = [(i, o) for i, o in enumerate(eng.ops()) if o[0] in ("maxpool", "avgpool")]
    shapes = sorted({(o[0], o[4], o[5], o[6], eng.value_info(o[1])[2]) for _i, o in pools})
    assert shapes == [("avgpool", 3, 1, 1, 8), ("avgpool", 3, 1, 1, 17), ("avgpool", 3, 1, 1, 35), ("maxpool", 3, 1, 1, 8),
                      ("maxpool", 3, 2, 0, 17), ("maxpool", 3, 2, 0, 35), ("maxpool", 3, 2, 0, 71), ("maxpool", 3, 2, 0, 147)], shapes
    gen = torch.Generator().manual_seed(frames)
    bad, ties = [], []
    try:
        for i, (kind, inp, out, _c, k, s, p) in pools:
            c, h, w = eng.value_info(inp)[:3]
            x = edge_input(frames, c, h, w, s, p, gen)
            eng.write(inp, x.to(dev))
            eng.run_op(i)
            y = eng.read(out).cpu().double()
            xd = x.double()
            if kind == "maxpool":
                ref = Fn.max_pool2d(xd, k, s, p, ceil_mode=True)
                ok = same_bits(y, ref)
                if not ok.all():
                    d = (~ok).nonzero()[0].tolist()
                    bad.append("%s: %d values differ (%d of them only in the sign of zero), first at %s: %r != %r" % (
                        out, int((~ok).sum()), int((same(y, ref) & ~ok).sum()), d, float(y[tuple(d)]), float(ref[tuple(d)])))
                # the share of windows whose maximum is tied between +0 and -0 (where the first-tap rule shows)
                z = xd[:, 1::16]
                cols = Fn.unfold(Fn.pad(z, (p, p, p, p), value=-INF), k, stride=s).view(frames, z.shape[1], k * k, -1)
                ties.append(float(((cols == 0).all(2) & torch.signbit(cols).any(2) & (~torch.signbit(cols)).any(2)).double().mean()))
            else:
                ref = Fn.avg_pool2d(xd, k, s, p, ceil_mode=True)
                masks = nonfinite_masks_equal(y, ref)
                fin = torch.isfinite(ref)
                err = float((y[fin] - ref[fin]).norm() / ref[fin].norm())
                if not all(masks) or not err <= AVGPOOL_BAR[precision]:
                    bad.append("%s: [NaN, +inf, -inf] masks equal %s, rel-L2 %.2e" % (out, masks, err))
            if precision == "exact_tc":
                pl = eng.read(out, planes=True).cpu().double()
                fin = torch.isfinite(y)
                if not torch.equal(torch.isfinite(pl), fin):
                    bad.append("%s planes: finite at %d places where the value is not, non-finite at %d where it is" % (
                        out, int((torch.isfinite(pl) & ~fin).sum()), int((~torch.isfinite(pl) & fin).sum())))
                elif kind == "maxpool" and not torch.equal(pl[fin], y[fin]):
                    bad.append("%s planes: %d finite values differ from the value" % (out, int((pl[fin] != y[fin]).sum())))
                elif kind == "avgpool" and float((pl[fin] - y[fin]).norm() / y[fin].norm()) > PLANES_BAR:
                    bad.append("%s planes: rel-L2 %.2e" % (out, float((pl[fin] - y[fin]).norm() / y[fin].norm())))
    finally:
        _release(eng)
    print("\nInceptionV3 %s F=%d: %d pool ops; windows tied between +0 and -0 (max pools): %s"
          % (precision, frames, len(pools), ", ".join("%.2f" % t for t in ties)))
    assert all(t > 0.1 for t in ties), ties
    assert not bad, "\n".join(bad)


# ---- B: non-finite pixels through the whole backbone ---------------------------------------------------------------------
# frame: ((channel, row, col), value) -- a corner, an edge and the interior of the 299 input
POISON_37 = {5: ((0, 0, 0), -INF), 17: ((1, 0, 150), NAN), 36: ((2, 150, 151), INF)}
POISON_129 = [{128: ((2, 298, 298), INF)}, {128: ((0, 77, 298), -INF)}, {128: ((1, 101, 203), NAN)}]


def _fold(params, name, dev):
    s = params[name + "_batchnorm.weight"].double() / torch.sqrt(params[name + "_batchnorm.running_var"].double() + 1e-5)
    w = params[name + "_Conv2D.weight"].double() * s.view(-1, 1, 1, 1)
    b = (params[name + "_Conv2D.bias"].double() - params[name + "_batchnorm.running_mean"].double()) * s + params[name + "_batchnorm.bias"].double()
    return w.to(dev), b.to(dev)


def _nonfinite_mismatches(eng, params, feat, precision, frames):
    """per op and per frame in `frames`: the non-finite mask of what the engine stored against float64 of the op applied to
    the engine's consumed input (a convolution of EXACT_TC: the input's operand planes, where |x| >= 65520 is NaN).  FAST
    stores fp16, so a result at or past 65520 may be non-finite where float64 is not; nothing non-finite may become finite."""
    from ssn_b200.inception_v3 import conv_table
    dev = feat.device
    tc = precision == "exact_tc"
    fr = torch.tensor(frames, device=dev)
    d64 = lambda t: t[fr].to(device=dev, dtype=torch.float64)
    geo = {c[0]: c for c in conv_table(3)}
    out = []
    with torch.backends.cudnn.flags(enabled=False):          # plain im2col + GEMM: a NaN reaches exactly its own windows
        for kind, inp, o, _c, k, s, p in eng.ops():
            if kind == "gpool":
                got, ref = d64(feat), d64(eng.read(inp)).mean((2, 3))
            elif kind == "conv":
                _n, _ci, _co, _kh, _kw, st, ph, pw = geo[o]
                w, b = _fold(params, o, dev)
                ref = Fn.relu(Fn.conv2d(d64(eng.read(inp, planes=tc)), w, b, st, (ph, pw)))
                got = d64(eng.read(o))
            else:
                pool = Fn.max_pool2d if kind == "maxpool" else Fn.avg_pool2d
                ref = pool(d64(eng.read(inp)), k, s, p, ceil_mode=True)
                got = d64(eng.read(o))
            want, has = ~torch.isfinite(ref), ~torch.isfinite(got)
            extra = has & ~want
            if precision == "fast":
                extra &= ref.abs() < FP16_INF_FROM
            lost = want & ~has
            if extra.any() or lost.any():
                first = (extra | lost).nonzero()[0].tolist()
                out.append("%s: %d places non-finite only in the engine, %d finite only in the engine (engine %d, float64 %d), "
                           "first at %s" % (o, int(extra.sum()), int(lost.sum()), int(has.sum()), int(want.sum()), first))
    return out


def _poisoned(x, poison):
    x = x.clone()
    for f, ((c, r, s), v) in poison.items():
        x[f, c, r, s] = v
    return x


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("frames,poisons", [(37, [POISON_37]), (129, POISON_129)], ids=["F37", "F129"])
def test_non_finite_pixels_stay_in_their_frame(precision, frames, poisons):
    dev = _cuda()
    params = _weights()
    eng = _engine(precision, frames, params, dev)
    try:
        x = synth.synth_frames(frames, 3, IV.INPUT_SIZE, seed=17).to(dev)
        clean = eng.forward(x).clone()
        bad = []
        for poison in poisons:
            feat = eng.forward(_poisoned(x, poison))
            torch.cuda.synchronize()
            others = [f for f in range(frames) if f not in poison]
            if not torch.equal(feat[others], clean[others]):
                bad.append("%s: other frames' feat changed" % poison)
            for f in poison:
                if torch.isfinite(feat[f]).all():
                    bad.append("%s: frame %d's feat is finite" % (poison, f))
            bad += ["%s: %s" % (poison, b) for b in _nonfinite_mismatches(eng, params, feat, precision, sorted(poison))]
        print("\nInceptionV3 %s F=%d: %d poisoned runs, %s" % (precision, frames, len(poisons), "as float64" if not bad else "%d findings" % len(bad)))
        assert not bad, "\n".join(bad)
    finally:
        _release(eng)


# ---- C: a NaN weight, activations past the fp16 range -------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
def test_nan_weight_poisons_every_frame(precision):
    """one NaN weight of a 5x5 layer (mixed_tower_conv_1) or of a 7x1 layer (mixed_4_tower_conv_1): feat is NaN in every
    frame and every channel"""
    dev = _cuda()
    frames = 37
    eng = _engine(precision, frames, _weights(), dev)
    try:
        x = synth.synth_frames(frames, 3, IV.INPUT_SIZE, seed=17).to(dev)
        assert torch.isfinite(eng.forward(x)).all()
        for layer in ("mixed_tower_conv_1", "mixed_4_tower_conv_1"):
            params = {k: v.clone() for k, v in _weights().items()}
            params[layer + "_Conv2D.weight"][0, 0, 0, 0] = NAN
            _pack(eng, params, dev)
            feat = eng.forward(x)
            torch.cuda.synchronize()
            assert feat.isnan().all(), (layer, int(feat.isnan().sum()), feat.numel())
    finally:
        _release(eng)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_activations_past_fp16_range(precision):
    """a 16 x 16 patch of 4e6 in one frame drives the stem's activations past 65504 (the synthetic frames' stem activations
    are about 0.03 x the pixel value, so no patch inside fp16's range does): EXACT computes the frame (finite feat); the
    fp16 operands of FAST and the operand planes of EXACT_TC cannot and say so (non-finite feat); every other frame's feat
    is bitwise unchanged"""
    dev = _cuda()
    frames = 37
    eng = _engine(precision, frames, _weights(), dev)
    try:
        x = synth.synth_frames(frames, 3, IV.INPUT_SIZE, seed=17).to(dev)
        clean = eng.forward(x).clone()
        xo = x.clone()
        xo[9, :, 100:116, 140:156] = 4e6
        feat = eng.forward(xo)
        torch.cuda.synchronize()
        others = [f for f in range(frames) if f != 9]
        assert torch.equal(feat[others], clean[others])
        if precision == "exact":
            stem = float(eng.read("conv")[9].abs().max())
            print("\nInceptionV3 exact: largest stem activation of the bright frame %.3g" % stem)
            assert stem > FP16_INF_FROM
            assert torch.isfinite(feat[9]).all()
        else:
            assert not torch.isfinite(feat[9]).all()
    finally:
        _release(eng)
