"""The per-launch float64 check of the backward (oracle/schedule_check.py, bars unchanged) at the gradient magnitudes an SSN
training step produces, on the engines and weights of tests/test_gpu_schedule.py.

The other schedule tests feed dfeat = 0.01 * randn.  The step's real dfeat is 2 to 4 orders of magnitude smaller: heads
initialised N(0, 0.001) as ssn_models does, dropout 0.8 and SSN's loss.  EXACT_TC reads every gradient as the fp16 planes
hi + lo of dz * grad_scale * 2^k, and FAST stores it in fp16 times the same factor, so a gradient too small for fp16 loses
bits or flushes to zero.  The backward picks 2^k on the device from max |dfeat| (oracle/split_operands.grad_exponent).
  - the real step's dfeat (float64 from the engine's own feat, bench-shaped proposals) at grad_scale 4096 and 1;
  - dfeat * 2^j for j from -24 up to where the largest gradient plane * grad_scale nears 2^15;
  - power-of-two scaling of dfeat is exact: dW and db scale by exactly 2^j, layer by layer.
Run on an H100: pytest -m gpu -s tests/test_gpu_grad_range.py."""
import math
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import schedule_check as S
from oracle import split_operands as SO
from oracle import step_check as SC
from oracle import ssn_oracle as O
from oracle import synth

GRAD_SCALE = 4096.0
J_MIN = -24


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_WEIGHTS = {}


def _weights():
    if not _WEIGHTS:
        _WEIGHTS[3] = synth.synth_backbone(3, seed=0, calib_frames=2)
    return _WEIGHTS[3]


def _names():
    return [n for (n, *_r) in O.conv_layers(3)]


def _engine(precision, frames, dev, grad_scale=GRAD_SCALE, bn1_train=False):
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    prec = {"fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]
    old = os.environ.get("SSNB_DISABLE_FUSION")
    os.environ["SSNB_DISABLE_FUSION"] = "0"
    try:
        eng = BackboneEngine(3, frames, prec, True, grad_scale, dev, bn1_train=bn1_train)
    finally:
        if old is None:
            os.environ.pop("SSNB_DISABLE_FUSION")
        else:
            os.environ["SSNB_DISABLE_FUSION"] = old
    bb = _weights()
    eng.pack(*[[bb[n + k].to(dev) for n in _names()] for k in (".weight", ".bias", "_bn.weight", "_bn.bias", "_bn.running_mean",
                                                                "_bn.running_var")])
    return eng


def _grads(dev):
    bb = _weights()
    return ([torch.zeros(bb[n + ".weight"].shape, device=dev) for n in _names()],
            [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in _names()])


def _step_dfeat(feat):
    """the step's dfeat (oracle step_check.ssn_step_dfeat) for the engine's F frames.  Below 288 frames: the first F rows that
    are not all zero -- a frame of a proposal the loss does not reach gets no gradient, and in bn_mode='partial' its conv1 dz
    is then the BatchNorm's batch term alone, a cancellation that fp32 resolves to ~6e-6 of itself (measured on the H100),
    a property of the vjp's arithmetic that the per-frame bar is not meant for"""
    n = SC.STEP_VIDEOS * SC.STEP_PROPS * SC.STEP_SEG
    if feat.shape[0] == n:
        return SC.ssn_step_dfeat(feat)
    full = SC.ssn_step_dfeat(feat.repeat((n + feat.shape[0] - 1) // feat.shape[0], 1)[:n])
    return full[full.abs().amax(1) > 0][:feat.shape[0]].contiguous()


def _grad_plane_max(eng, G, precision):
    """max |dz| over what the tensor cores read of the gradients (un-scaled): every convolution output and the max-pool
    branches of the stride-2 blocks; EXACT_TC: the hi + lo planes, FAST: the fp16 storage"""
    names = [o["out"] for o in G.ops if o["kind"] == "conv"]
    names += [v for v in G.branch if any(o["out"] == v and o["kind"] == "maxpool" for o in G.ops)]
    return max(float(eng.read(v, grad=True, planes=precision == "exact_tc").abs().max()) for v in names)


def _growth(eng, G, dfeat, precision):
    """largest ratio over the convolution outputs of max |dz| to the entry value max |dfeat| / 49"""
    entry = float(dfeat.abs().max()) / 49.0
    names = [o["out"] for o in G.ops if o["kind"] == "conv"]
    best = (0.0, None)
    for v in names:
        m = float(eng.read(v, grad=True, planes=precision == "exact_tc").abs().max())
        best = max(best, (m / entry, v))
    return best


def _worst(recs, quantity):
    rs = [r for r in recs if r.quantity == quantity]
    return max(rs, key=lambda r: r.err) if rs else None


def _report(label, recs, extra=""):
    print("\n%s: %d records; worst %s%s" % (label, len(recs), ", ".join(
        "%s %.2e (%s)" % (q, r.err, r.op) for q, r in ((q, _worst(recs, q)) for q in ("dZ", "G", "dW", "db")) if r), extra))
    bad = S.failures(recs)
    if bad:
        print("  %d records beyond their bars, worst:" % len(bad), *sorted(bad, key=lambda r: -r.score)[:5], sep="\n    ")
    return bad


# ---- the real step's gradient ----------------------------------------------------------------------------------------------
# (precision, frames, grad_scale, bn1_train): bench.py's EXACT_TC and FAST at its grad_scale, EXACT_TC at set_precision's
# default grad_scale 1.0, a ragged frame count, and bn_mode='partial'
REAL_CASES = [("exact_tc", 288, 4096.0, False), ("exact_tc", 288, 1.0, False), ("fast", 288, 4096.0, False),
              ("exact_tc", 37, 4096.0, False), ("exact_tc", 37, 4096.0, True)]


@pytest.mark.parametrize("precision,frames,grad_scale,bn1_train", REAL_CASES,
                         ids=["%s-F%d-gs%g%s" % (p, f, g, "-bn1" if b else "") for p, f, g, b in REAL_CASES])
def test_real_step_gradient(precision, frames, grad_scale, bn1_train):
    dev = _cuda()
    t0 = time.time()
    eng = _engine(precision, frames, dev, grad_scale, bn1_train)
    try:
        bn1 = None
        if bn1_train:
            bb = _weights()
            bn = torch.nn.BatchNorm2d(64).to(dev)
            with torch.no_grad():
                for k in ("weight", "bias", "running_mean", "running_var"):
                    getattr(bn, k).copy_(bb["conv1_7x7_s2_bn." + k])
            dgamma, dbeta = torch.zeros(64, device=dev), torch.zeros(64, device=dev)
            eng.set_bn1(bn, dgamma, dbeta)
            rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        x = synth.synth_frames(frames, 3, seed=17).to(dev)
        feat = eng.forward(x)
        dfeat = _step_dfeat(feat)
        dw, db = _grads(dev)
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        overflow = eng.grad_overflow()
        t1 = time.time()
        if bn1_train:
            bn1 = dict(gamma=bn.weight.detach(), beta=bn.bias.detach(), momentum=bn.momentum, eps=bn.eps, running_mean0=rm0,
                       running_var0=rv0, running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone(), dgamma=dgamma,
                       dbeta=dbeta)
        recs = S.check_schedule(eng, _weights(), x, feat, dfeat, dw, db, precision, 3, bn1=bn1)
        growth, where = _growth(eng, S.Graph(3, bn1_train=bn1_train), dfeat, precision)
        nz = dfeat[dfeat != 0].abs()
        bad = _report("real step %s F=%d grad_scale %g%s" % (precision, frames, grad_scale, " bn1" if bn1_train else ""), recs,
                      "; |dfeat| max %.2e median %.2e; largest plane / entry growth %.1fx (%s); engine %.1f s, check %.1f s"
                      % (float(nz.max()), float(nz.median()), growth, where, t1 - t0, time.time() - t1))
        assert not overflow
        assert not bad, "\n".join(map(repr, bad))
    finally:
        del eng
        torch.cuda.empty_cache()


# ---- power-of-two sweep ----------------------------------------------------------------------------------------------------
def _sweep_setup(precision, dev):
    eng = _engine(precision, 37, dev)
    x = synth.synth_frames(37, 3, seed=17).to(dev)
    dfeat = (torch.randn(37, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
    feat = eng.forward(x)
    dw, db = _grads(dev)
    eng.backward(dfeat, dw, db)
    torch.cuda.synchronize()
    m = _grad_plane_max(eng, S.Graph(3), precision)
    # largest j with (largest gradient plane) * grad_scale * 2^j below 2^15
    j_max = math.ceil(15 - math.log2(m * GRAD_SCALE)) - 1
    return eng, x, feat, dfeat, [t.clone() for t in dw], [t.clone() for t in db], j_max


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_power_of_two_sweep(precision):
    """every record within its bar at every magnitude of dfeat"""
    dev = _cuda()
    t0 = time.time()
    eng, x, feat, dfeat, _dw0, _db0, j_max = _sweep_setup(precision, dev)
    try:
        rows, failed = [], []
        for j in range(J_MIN, j_max + 1):
            d = dfeat * 2.0 ** j
            dw, db = _grads(dev)
            eng.backward(d, dw, db)
            recs = S.check_schedule(eng, _weights(), x, feat, d, dw, db, precision, 3)
            w = _worst(recs, "dZ")
            bad = S.failures(recs)
            rows.append("j=%+3d (gradient exponent k=%d) worst dZ %.2e (%s)%s" % (
                j, SO.grad_exponent(float(d.abs().max()), GRAD_SCALE), w.err, w.op,
                ", %d records beyond their bars (worst %s %s %.2e)" % (len(bad), bad[0].op, bad[0].quantity, bad[0].err) if bad else ""))
            if bad:
                failed.append((j, sorted(bad, key=lambda r: -r.score)[0]))
        print("\n%s F=37 dfeat x 2^j, j = %d..%d (%.1f s):" % (precision, J_MIN, j_max, time.time() - t0), *rows, sep="\n  ")
        assert not failed, "\n".join("j=%d: %r" % f for f in failed)
    finally:
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_power_of_two_scaling_is_exact(precision):
    """dW(2^j dfeat) == 2^j dW(dfeat) and the same for db, bitwise, every layer, every j of the sweep"""
    dev = _cuda()
    eng, _x, _feat, dfeat, dw0, db0, j_max = _sweep_setup(precision, dev)
    names = _names()
    try:
        differ = {}
        for j in range(J_MIN, j_max + 1):
            dw, db = _grads(dev)
            eng.backward(dfeat * 2.0 ** j, dw, db)
            for q, got, ref in (("dW", dw, dw0), ("db", db, db0)):
                for n, a, b in zip(names, got, ref):
                    if not torch.equal(a, b * 2.0 ** j):
                        differ.setdefault(j, []).append("%s %s" % (n, q))
        print("\n%s F=37 dfeat x 2^j, j = %d..%d: %s" % (precision, J_MIN, j_max, "exact" if not differ else "; ".join(
            "j=%d: %d tensors differ (%s)" % (j, len(v), ", ".join(v[:3])) for j, v in sorted(differ.items()))))
        assert not differ
    finally:
        del eng
        torch.cuda.empty_cache()
