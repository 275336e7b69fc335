"""The pooling and mask glue, and the whole backbone, at the inputs the continuous synthetic data never produce: exact ties in
max-pool windows (+-0 among them), constant and dead channels, NaN and +-inf activations, a diverged (NaN) weight and an input
beyond the fp16 range.  Run on an H100: pytest -m gpu -s tests/test_gpu_glue_edges.py.

A  every pool op alone (write -> run_op -> read) against float64 ATen, forward and backward, at F = 1 and 37;
B  the production schedule (oracle/schedule_check.py, unchanged bars) on a network with tied and constant channels, which is
   the only way to reach the 2x2 pool-gather pass folded into conv1 / conv2_3x3;
C  non-finite values through the whole schedule at F = 37: they stay in their frame, reach exactly the places float64 puts
   them (conv1 of the tensor-core modes: one known extra row / column, see DESIGN.md) and are never turned into finite numbers.
"""
import math
import os
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import schedule_check as S
from oracle import ssn_oracle as O
from oracle import synth
from oracle.edge_inputs import edge_input as _edge_input, same_bits

GRAD_SCALE = 4096.0
PRECISIONS = ("exact", "exact_tc", "fast")
NAN, INF = math.nan, math.inf


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_WEIGHTS = {}


def _weights(kind="synth"):
    if kind not in _WEIGHTS:
        p = synth.synth_backbone(3, seed=0, calib_frames=2)
        _WEIGHTS[kind] = _tied(p) if kind == "tied" else p
    return _WEIGHTS[kind]


def _names():
    return [n for (n, *_r) in O.conv_layers(3)]


def _engine(precision, frames, params, dev, unfused=False):
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    prec = {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]
    old = os.environ.get("SSNB_DISABLE_FUSION")
    os.environ["SSNB_DISABLE_FUSION"] = "1" if unfused else "0"
    try:
        eng = BackboneEngine(3, frames, prec, True, GRAD_SCALE, dev)
    finally:
        if old is None:
            os.environ.pop("SSNB_DISABLE_FUSION", None)
        else:
            os.environ["SSNB_DISABLE_FUSION"] = old
    _pack(eng, params, dev)
    return eng


def _pack(eng, p, dev):
    n = _names()
    eng.pack(*[[p[k + suf].to(dev) for k in n] for suf in (".weight", ".bias", "_bn.weight", "_bn.bias", "_bn.running_mean",
                                                             "_bn.running_var")])


def _grads(dev):
    p = _weights()
    return ([torch.zeros(p[n + ".weight"].shape, device=dev) for n in _names()],
            [torch.zeros(p[n + ".bias"].shape, device=dev) for n in _names()])


# ---- A: every pool op on its own ------------------------------------------------------------------------------------------
def _pool_ops(eng):
    """[(op index, kind, input, output, attrs, accumulates)]; accumulates: a later op reads the same input, so its gradient
    is already in d(input) when this op's backward runs"""
    ops = eng.ops()
    G = S.Graph(3)
    assert [(o["kind"], o["inp"], o["out"]) for o in G.ops] == ops
    out = []
    for i, (kind, inp, o) in enumerate(ops):
        if kind in ("maxpool", "avgpool"):
            out.append((i, kind, inp, o, G.ops[i]["a"], any(e[1] == inp for e in ops[i + 1:])))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("frames", [1, 37])
def test_pool_ops_on_ties_and_non_finite(precision, frames):
    dev = _cuda()
    t0 = time.time()
    eng = _engine(precision, frames, _weights(), dev)
    pools = _pool_ops(eng)
    kinds = [(k, a["stride"]) for _i, k, _x, _y, a, _acc in pools]
    assert kinds.count(("maxpool", 2)) == 4 and kinds.count(("maxpool", 1)) == 1 and kinds.count(("avgpool", 1)) == 7, kinds
    gen = torch.Generator().manual_seed(frames)
    bad = []
    try:
        for i, kind, inp, out, a, acc in pools:
            k, s, p = a["k"], a["stride"], a["pad"]
            c, h, w = eng.value_shape(inp)
            x = _edge_input(frames, c, h, w, s, p, gen)
            eng.write(inp, x.to(dev))
            eng.run_op(i)
            y = eng.read(out).cpu().double()
            pool = F.max_pool2d if kind == "maxpool" else F.avg_pool2d
            xr = x.double().requires_grad_(True)
            ref = pool(xr, k, s, p, ceil_mode=True)
            if kind == "maxpool":
                if not same_bits(y, ref.detach()).all():       # the sign of a tied zero included
                    bad.append("%s fwd: %d values differ" % (out, int((~same_bits(y, ref.detach())).sum())))
            else:
                r = ref.detach()
                masks = [(t(y) == t(r)).all() for t in (torch.isnan, torch.isposinf, torch.isneginf)]
                fin = torch.isfinite(r)
                err = float((y[fin] - r[fin]).norm() / r[fin].norm())
                if not all(masks) or not err <= S.ROUND[precision]:
                    bad.append("%s fwd: non-finite masks %s, rel-L2 %.2e" % (out, masks, err))
            # backward: dyadic output gradient (x 9 through the average: the 1/9 is then exact), d(input) prefilled with X
            q = 9.0 if kind == "avgpool" else 1.0
            gy = torch.randint(-8, 9, ref.shape, generator=gen).double() * 0.125 * q
            X = torch.randint(-16, 17, x.shape, generator=gen).double() * 0.25
            ref.backward(gy)
            want = xr.grad + X if acc else xr.grad
            eng.write(out, gy.to(dev), grad=True)
            eng.write(inp, X.to(dev), grad=True)
            eng.run_op(i, backward=True)
            got = eng.read(inp, grad=True).cpu().double()
            if not torch.equal(got, want):
                d = (got != want).nonzero()
                bad.append("%s bwd (%s): %d values differ, first at %s: %s != %s" % (
                    inp, "X + vjp" if acc else "vjp", len(d), d[0].tolist(), float(got[tuple(d[0])]), float(want[tuple(d[0])])))
    finally:
        del eng
        torch.cuda.empty_cache()
    print("\n%s F=%d: %d pool ops, %.1f s" % (precision, frames, len(pools), time.time() - t0))
    assert not bad, "\n".join(bad)


# ---- B: tied and constant channels through the production schedule ------------------------------------------------------
ZERO_CONV = "inception_4a_pool_proj"       # a 1x1 conv in no fused block: all-zero weights (EXACT_TC: zero weight-plane absmax)


def _tied(p):
    """every 8th output channel of every conv has zero weights and running_mean = bias, so its folded output is relu(beta):
    beta > 0 on half of them (constant channels: every max-pool window tied, average-pool borders 4c/9 and 6c/9), beta < 0
    on the other half (dead channels); ZERO_CONV has no non-zero weight at all"""
    q = {k: v.clone() for k, v in p.items()}
    for n in _names():
        w, b = q[n + ".weight"], q[n + ".bias"]
        sel = torch.arange(w.shape[0]) % 8 == 0
        w[sel] = 0.0
        q[n + "_bn.running_mean"][sel] = b[sel]
        beta = q[n + "_bn.bias"]
        beta[torch.arange(w.shape[0]) % 16 == 0] = 0.75
        beta[torch.arange(w.shape[0]) % 16 == 8] = -0.5
    q[ZERO_CONV + ".weight"].zero_()
    q[ZERO_CONV + "_bn.running_mean"].copy_(q[ZERO_CONV + ".bias"])
    return q


def _tied_fraction(v, k, s):
    """share of (frame, channel, window) whose maximum is taken by more than one tap (ceil mode, pad 0 or 1 as the op)"""
    v = v[:2].double()
    p = 1 if s == 1 else 0
    oh = S._pool_out(v.shape[2], k, s, p)
    hp = (oh - 1) * s + k
    cols = F.unfold(F.pad(v, (p, hp - v.shape[3] - p, p, hp - v.shape[2] - p), value=-INF), k, stride=s)
    cols = cols.view(v.shape[0], v.shape[1], k * k, -1)
    return float(((cols == cols.amax(2, keepdim=True)).sum(2) > 1).double().mean())


TIED_CASES = [("exact_tc", 288, False), ("exact_tc", 37, False), ("exact_tc", 1, False), ("fast", 288, False), ("fast", 37, False),
              ("fast", 1, False), ("exact", 37, False), ("exact_tc", 37, True)]


@pytest.mark.parametrize("precision,frames,unfused", TIED_CASES,
                         ids=["%s-F%d%s" % (p, f, "-unfused" if u else "") for p, f, u in TIED_CASES])
def test_schedule_with_tied_and_constant_channels(precision, frames, unfused):
    dev = _cuda()
    t0 = time.time()
    bb = _weights("tied")
    eng = _engine(precision, frames, bb, dev, unfused)
    try:
        x = synth.synth_frames(frames, 3, seed=17).to(dev)
        dfeat = (torch.randn(frames, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
        feat = eng.forward(x)
        dw, db = _grads(dev)
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        assert not eng.grad_overflow()
        ties = {o: _tied_fraction(eng.read(i), 3, a["stride"]) for _n, kind, i, o, a, _acc in _pool_ops(eng) if kind == "maxpool"}
        recs = S.check_schedule(eng, bb, x, feat, dfeat, dw, db, precision, 3)
        print("\n%s F=%d%s: %d records, %.1f s; tied max-pool windows: %s" % (
            precision, frames, " unfused" if unfused else "", len(recs), time.time() - t0,
            ", ".join("%s %.3f" % kv for kv in ties.items())))
        print("  5 worst records:", *S.worst(recs), sep="\n    ")
        assert all(f >= 0.1 for f in ties.values()), ties
        bad = S.failures(recs)
        assert not bad, "\n".join(map(repr, bad))
    finally:
        del eng
        torch.cuda.empty_cache()


# ---- C: non-finite values through the whole schedule ---------------------------------------------------------------------
FRAMES = 37
POISON = {5: ((1, 100, 116), NAN), 6: ((2, 50, 61), INF), 36: ((0, 223, 223), NAN)}      # frame: ((channel, row, col), value)


def _poisoned(x):
    x = x.clone()
    for f, ((c, r, s), v) in POISON.items():
        x[f, c, r, s] = v
    return x


def _nonfinite_mismatches(eng, params, x, feat, precision, frames):
    """per op and per frame in `frames`: the non-finite mask of what the engine stored against float64 of the op applied to
    the engine's consumed input.  conv1 of FAST / EXACT_TC runs as a 4x4 convolution over the space-to-depth input whose
    taps r, s = -1 carry zero weights: NaN * 0 puts its footprint one input row above and one column left of the 7x7 one."""
    dev = feat.device
    tc, fast = precision == "exact_tc", precision == "fast"
    fr = torch.tensor(frames, device=dev)
    d64 = lambda t: t[fr].to(device=dev, dtype=torch.float64)
    out = []
    with torch.backends.cudnn.flags(enabled=False):          # plain im2col + GEMM: a NaN reaches exactly its own windows
        for o in S.Graph(3).ops:
            a = o["a"]
            if o["kind"] == "gpool":
                got, ref = d64(feat), d64(eng.read(o["inp"])).mean((2, 3))
            elif o["kind"] == "conv":
                w, b, _s = S.fold(params, o["id"], dev)
                if o["inp"] == "data":          # what conv1 reads: fp16 x in FAST, hi + lo of x in EXACT_TC (NaN from 65520 up)
                    xin = d64(x.half().float() if fast else torch.where(x.abs() >= 65520.0, NAN, x) if tc else x)
                else:
                    xin = d64(eng.read(o["inp"], planes=tc))
                ref = F.relu(F.conv2d(xin, w, b, a["stride"], a["pad"]))
                got = d64(eng.read(o["out"]))
            else:
                pool = F.max_pool2d if o["kind"] == "maxpool" else F.avg_pool2d
                ref = pool(d64(eng.read(o["inp"])), a["k"], a["stride"], a["pad"], ceil_mode=True)
                got = d64(eng.read(o["out"]))
            want = ~torch.isfinite(ref)
            if o["inp"] == "data" and (tc or fast):
                # output (oy, ox) reads input rows 2oy-4 .. 2oy+3 (and the same columns) instead of 2oy-3 .. 2oy+3; the
                # extra row and column meet a non-finite pixel with a zero weight: NaN in every channel
                bad_px = (~torch.isfinite(xin)).any(1, keepdim=True).double()
                ones = lambda n: torch.ones(1, 1, n, n, dtype=torch.float64, device=dev)
                k8 = F.conv2d(bad_px, ones(8), stride=2, padding=4)[..., :want.shape[2], :want.shape[3]] > 0
                k7 = F.conv2d(bad_px, ones(7), stride=2, padding=3) > 0
                want = want | (k8 & ~k7)
            if not torch.equal(~torch.isfinite(got), want):
                diff = (~torch.isfinite(got)) != want
                out.append("%s: %d places differ (engine non-finite %d, reference %d), first %s" % (
                    o["id"], int(diff.sum()), int((~torch.isfinite(got)).sum()), int(want.sum()), diff.nonzero()[0].tolist()))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
def test_non_finite_pixels_stay_in_their_frame(precision):
    dev = _cuda()
    params = _weights()
    eng = _engine(precision, FRAMES, params, dev)
    try:
        x = synth.synth_frames(FRAMES, 3, seed=17).to(dev)
        clean = eng.forward(x).clone()
        xp = _poisoned(x)
        feat = eng.forward(xp)
        torch.cuda.synchronize()
        others = [f for f in range(FRAMES) if f not in POISON]
        assert torch.equal(feat[others], clean[others])
        assert all(not torch.isfinite(feat[f]).all() for f in POISON), [int((~torch.isfinite(feat[f])).sum()) for f in POISON]
        bad = _nonfinite_mismatches(eng, params, xp, feat, precision, sorted(POISON))
        assert not bad, "\n".join(bad)
        # a pixel beyond the fp16 range: EXACT computes it; the fp16 operands of FAST / EXACT_TC cannot, and say so
        xo = x.clone()
        xo[9, 1, 120, 80] = 1e5
        feat = eng.forward(xo)
        torch.cuda.synchronize()
        assert torch.equal(feat[[f for f in range(FRAMES) if f != 9]], clean[[f for f in range(FRAMES) if f != 9]])
        if precision == "exact":
            assert torch.isfinite(feat[9]).all()
            recs = S.check_schedule(eng, params, xo, feat, precision=precision)
            assert not S.failures(recs), "\n".join(map(repr, S.failures(recs)))
        else:
            assert not torch.isfinite(feat[9]).all()
    finally:
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_nan_output_gradient_stays_in_its_frame(precision):
    """a NaN row of dfeat leaves every value gradient of the other frames finite (dgrad tiles, zero-upsampled gradients and
    TMA boxes span frames)"""
    dev = _cuda()
    params = _weights()
    eng = _engine(precision, FRAMES, params, dev)
    try:
        x = synth.synth_frames(FRAMES, 3, seed=17).to(dev)
        eng.forward(x)
        dfeat = (torch.randn(FRAMES, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
        dfeat[20] = NAN
        dw, db = _grads(dev)
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        G = S.Graph(3)
        producer = {o["out"]: o for o in G.ops}
        others = [f for f in range(FRAMES) if f != 20]
        bad = []
        for v in G.shape:
            if v == "data":
                continue
            conv_out = v in producer and producer[v]["kind"] == "conv"        # (block outputs have no producer op)
            g = eng.read(v, grad=True, planes=conv_out and precision == "exact_tc")      # what the next kernel consumed
            if not torch.isfinite(g[others]).all():
                bad.append("%s: %d non-finite values in other frames" % (v, int((~torch.isfinite(g[others])).sum())))
            if not conv_out and v in G.consumers and torch.isfinite(g[20]).all():
                bad.append("%s: frame 20 is finite" % v)
        assert not bad, "\n".join(bad)
    finally:
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_nan_weight_poisons_every_frame(precision):
    """one NaN weight of inception_4a_3x3: feat is NaN in every frame (the step's loss with it); a backward with NaN dfeat
    raises the overflow flag where there is one; a backward with finite dfeat gives non-finite dW exactly where float64
    autograd of the same network does (the masks zero dz below every NaN y, 0 * NaN activation is still NaN)"""
    dev = _cuda()
    params = {k: v.clone() for k, v in _weights().items()}
    params["inception_4a_3x3.weight"][0, 0, 0, 0] = NAN
    eng = _engine(precision, FRAMES, params, dev)
    try:
        x = synth.synth_frames(FRAMES, 3, seed=17).to(dev)
        feat = eng.forward(x)
        torch.cuda.synchronize()
        assert feat.isnan().all(), int(feat.isnan().sum())
        dw, db = _grads(dev)
        eng.backward(torch.full((FRAMES, 1024), NAN, device=dev), dw, db)
        torch.cuda.synchronize()
        if precision != "exact":
            assert eng.grad_overflow()
        eng.forward(x)
        dfeat = (torch.randn(FRAMES, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
        dw, db = _grads(dev)
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        flag = eng.grad_overflow()
        p64 = {k: v.to(device=dev, dtype=torch.float64).requires_grad_(k.endswith(".weight") and "_bn" not in k)
               for k, v in params.items()}
        with torch.backends.cudnn.flags(enabled=False):
            ref = O.backbone_forward(p64, x.double(), 3)
            ref.backward(dfeat.double())
        bad = []
        for n, g in zip(_names(), dw):
            want = ~torch.isfinite(p64[n + ".weight"].grad)
            if not torch.equal(~torch.isfinite(g), want):
                bad.append("%s: engine %d non-finite, reference %d" % (n, int((~torch.isfinite(g)).sum()), int(want.sum())))
        print("\n%s: finite dfeat through a NaN weight: %d of 69 dW with non-finite entries, grad_overflow %s"
              % (precision, sum(not torch.isfinite(g).all() for g in dw), flag))
        assert not bad, "\n".join(bad)
    finally:
        del eng
        torch.cuda.empty_cache()
