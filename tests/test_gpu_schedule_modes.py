"""The per-launch float64 check (oracle/schedule_check.py) on the two engine configurations besides the frozen-BatchNorm
training engine of tests/test_gpu_schedule.py, and the loss-scale guard:
  - forward-only engines (training=0: no gradient buffers, no upsample region, no split-K partials), as SSN.test_scores,
    BinaryClassifier scoring and bench.py --mode infer run them, at the frame count the benchmark uses (40 ticks x 10 crops)
    and at ragged ones; and their forward is bitwise the forward of a training engine;
  - bn_mode='partial' engines (bn1_train): conv1 raw, the training-mode BatchNorm of csrc/bn_train.cu (batch statistics,
    running statistics, dgamma / dbeta, dz and its operand planes), pool1 not folded into conv1;
  - ssnb_grad_overflow: set when a NaN / inf arrives in dfeat or a gradient operand plane leaves the fp16 range, and cleared
    on request; dfeat far outside fp16's range (x 2^+-40) is brought back by the backward's gradient exponent and gives
    exactly scaled gradients.  The values involved are ordinary IEEE infinities / NaNs in the buffers.
Run on an H100: pytest -m gpu -s tests/test_gpu_schedule_modes.py."""
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import schedule_check as S
from oracle import ssn_oracle as O
from oracle import synth

GRAD_SCALE = 4096.0
HALF_MAX = 65504.0


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_WEIGHTS = {}


def _weights(in_channels):
    if in_channels not in _WEIGHTS:
        _WEIGHTS[in_channels] = synth.synth_backbone(in_channels, seed=0, calib_frames=2)
    return _WEIGHTS[in_channels]


def _engine(precision, frames, in_channels, training, dev, unfused=False, bn1_train=False):
    """a packed BackboneEngine on the synthetic weights (SSNB_DISABLE_FUSION is read while the engine binds its plans)"""
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    prec = {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]
    old = os.environ.get("SSNB_DISABLE_FUSION")
    os.environ["SSNB_DISABLE_FUSION"] = "1" if unfused else "0"
    try:
        eng = BackboneEngine(in_channels, frames, prec, training, GRAD_SCALE, dev, bn1_train=bn1_train)
    finally:
        if old is None:
            os.environ.pop("SSNB_DISABLE_FUSION")
        else:
            os.environ["SSNB_DISABLE_FUSION"] = old
    bb = _weights(in_channels)
    names = [n for (n, *_r) in O.conv_layers(in_channels)]
    eng.pack(*[[bb[n + k].to(dev) for n in names] for k in (".weight", ".bias", "_bn.weight", "_bn.bias", "_bn.running_mean",
                                                             "_bn.running_var")])
    return eng


def _bn1_module(in_channels, dev):
    """the first BatchNorm2d of a bn_mode='partial' model, on the synthetic weights, and zeroed dgamma / dbeta"""
    bb = _weights(in_channels)
    bn = torch.nn.BatchNorm2d(64).to(dev)
    with torch.no_grad():
        for k in ("weight", "bias", "running_mean", "running_var"):
            getattr(bn, k).copy_(bb["conv1_7x7_s2_bn." + k])
    return bn, torch.zeros(64, device=dev), torch.zeros(64, device=dev)


def _inputs(frames, in_channels, dev):
    x = synth.synth_frames(frames, in_channels, seed=17).to(dev)
    dfeat = (torch.randn(frames, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
    return x, dfeat


def _grads(in_channels, dev):
    bb = _weights(in_channels)
    names = [n for (n, *_r) in O.conv_layers(in_channels)]
    return [torch.zeros(bb[n + ".weight"].shape, device=dev) for n in names], [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in names]


def _report(label, recs, t_engine, t_check, show=()):
    """print the worst records (and the records of the ops in `show`), then fail on any record beyond its bar"""
    worst = {}
    for r in recs:                 # worst value per quantity, for the records in DESIGN.md
        if r.quantity not in worst or r.err > worst[r.quantity].err:
            worst[r.quantity] = r
    print("\n%s: %d records, engine %.1f s, float64 check %.1f s; worst per quantity: %s"
          % (label, len(recs), t_engine, t_check, ", ".join("%s %.2e (%s)" % (q, r.err, r.op) for q, r in worst.items())))
    print("  5 worst records (closest to their bars):", *S.worst(recs), sep="\n    ")
    if show:
        print("  records of %s:" % ", ".join(show), *[r for r in recs if r.op in show], sep="\n    ")
    bad = S.failures(recs)
    assert not bad, "\n".join(map(repr, bad))


# ---- forward-only engines ------------------------------------------------------------------------------------------------
# (precision, frames, in_channels): bench.py --mode infer's 40 ticks x 10 crops, RGB and Flow; a partial chunk of 13 ticks;
# one frame; the SIMT fp32 path
INFER_CASES = [("exact_tc", 400, 3), ("exact_tc", 400, 10), ("fast", 400, 3), ("exact_tc", 130, 3), ("fast", 1, 3),
               ("exact", 37, 3)]


@pytest.mark.parametrize("precision,frames,in_channels", INFER_CASES, ids=["%s-F%d-c%d" % c for c in INFER_CASES])
def test_inference_per_launch(precision, frames, in_channels):
    dev = _cuda()
    t0 = time.time()
    eng = _engine(precision, frames, in_channels, False, dev)
    try:
        x, _ = _inputs(frames, in_channels, dev)
        feat = eng.forward(x)
        torch.cuda.synchronize()
        t1 = time.time()
        recs = S.check_schedule(eng, _weights(in_channels), x, feat, precision=precision, in_channels=in_channels)
        assert {r.quantity for r in recs} <= {"fwd", "planes"}
        _report("inference %s F=%d in_channels=%d" % (precision, frames, in_channels), recs, t1 - t0, time.time() - t1)
    finally:
        del eng
        torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_inference_forward_equals_training_forward(precision):
    """a training=0 engine binds the same forward plans as a training=1 engine: feat and every stored value (EXACT_TC: and its
    operand planes) are bitwise equal, although the two workspaces are laid out differently"""
    dev = _cuda()
    x, _ = _inputs(37, 3, dev)
    engs = [_engine(precision, 37, 3, training, dev) for training in (False, True)]
    try:
        feats = [e.forward(x) for e in engs]
        assert torch.equal(feats[0], feats[1])
        differ = []
        for name in S.Graph(3).shape:
            if name == "data":
                continue
            for planes in ((False, True) if precision == "exact_tc" else (False,)):
                a, b = (e.read(name, planes=planes) for e in engs)
                if not torch.equal(a, b):
                    differ.append((name, planes, float((a - b).abs().max())))
        assert not differ, differ
    finally:
        del engs
        torch.cuda.empty_cache()


# ---- bn_mode='partial' ---------------------------------------------------------------------------------------------------
# (precision, frames, in_channels, SSNB_DISABLE_FUSION): F = 288 puts the BatchNorm reductions at their 592-CTA cap
BN1_CASES = [("exact_tc", 288, 3, False), ("exact_tc", 37, 3, False), ("exact_tc", 1, 3, False), ("exact_tc", 37, 10, False),
             ("exact_tc", 37, 3, True), ("exact", 37, 3, False)]


def _bn1_state(bn, rm0, rv0, dgamma, dbeta):
    return dict(gamma=bn.weight.detach(), beta=bn.bias.detach(), momentum=bn.momentum, eps=bn.eps, running_mean0=rm0,
                running_var0=rv0, running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone(), dgamma=dgamma,
                dbeta=dbeta)


@pytest.mark.parametrize("precision,frames,in_channels,unfused", BN1_CASES,
                         ids=["%s-F%d-c%d%s" % (p, f, c, "-unfused" if u else "") for p, f, c, u in BN1_CASES])
def test_bn1_per_launch(precision, frames, in_channels, unfused):
    dev = _cuda()
    t0 = time.time()
    bb = _weights(in_channels)
    eng = _engine(precision, frames, in_channels, True, dev, unfused=unfused, bn1_train=True)
    try:
        bn, dgamma, dbeta = _bn1_module(in_channels, dev)
        eng.set_bn1(bn, dgamma, dbeta)
        x, dfeat = _inputs(frames, in_channels, dev)
        dw, db = _grads(in_channels, dev)
        rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        feat = eng.forward(x)
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        assert not eng.grad_overflow()
        t1 = time.time()
        st = _bn1_state(bn, rm0, rv0, dgamma, dbeta)
        recs = S.check_schedule(eng, bb, x, feat, dfeat, dw, db, precision, in_channels, bn1=st)
        # the BatchNorm's fwd (+ planes), running_mean / running_var, G via pool1, dgamma / dbeta
        assert sum(r.op == S.BN1_OUT for r in recs) == (7 if precision == "exact_tc" else 6)
        _report("bn1 %s F=%d in_channels=%d%s" % (precision, frames, in_channels, " SSNB_DISABLE_FUSION=1" if unfused else ""),
                recs, t1 - t0, time.time() - t1, show=(S.BN1_CONV, S.BN1_OUT))
        if precision == "exact_tc" and frames == 37 and in_channels == 3 and not unfused:
            # an accumulating backward adds exactly the same gradients again, dgamma / dbeta included
            saved = [t.clone() for t in dw + db + [dgamma, dbeta]]
            eng.backward(dfeat, dw, db, accumulate=True)
            torch.cuda.synchronize()
            names = [n for (n, *_r) in O.conv_layers(in_channels)]
            names = [n + ".weight" for n in names] + [n + ".bias" for n in names] + ["bn1.weight", "bn1.bias"]
            assert all(torch.equal(a, 2 * b) for a, b in zip(dw + db + [dgamma, dbeta], saved)), \
                [n for n, a, b in zip(names, dw + db + [dgamma, dbeta], saved) if not torch.equal(a, 2 * b)]
            # a second forward: the same feat bitwise; the running statistics take a second momentum step
            assert torch.equal(eng.forward(x), feat)
            z = eng.read(S.BN1_RAW).double()
            n = z.numel() // 64
            mu, var = z.mean((0, 2, 3)), z.var((0, 2, 3), unbiased=True)
            m = bn.momentum
            rm, rv = rm0.double(), rv0.double()
            for _ in range(2):
                rm, rv = (1 - m) * rm + m * mu, (1 - m) * rv + m * var
            e_rm = float((bn.running_mean.double() - rm).norm() / rm.norm())
            e_rv = float((bn.running_var.double() - rv).norm() / rv.norm())
            print("  two forwards: running_mean %.2e, running_var %.2e (rows per channel %d)" % (e_rm, e_rv, n))
            assert e_rm <= S.RUNSTAT_BAR and e_rv <= S.RUNSTAT_BAR
    finally:
        del eng
        torch.cuda.empty_cache()


# ---- the loss-scale guard ------------------------------------------------------------------------------------------------
def _scaled_backward_flags(eng, dfeat, dw, db, extra=()):
    """dfeat x 2^-40 and x 2^40: the backward brings the entry gradient back into range (its gradient exponent), so the flag
    stays clear and every dW / db (and `extra`, e.g. dgamma / dbeta) is exactly 2^+-40 times the ordinary one"""
    eng.backward(dfeat, dw, db)
    ref = [t.clone() for t in list(dw) + list(db) + list(extra)]
    flags, exact = {}, {}
    for j in (-40, 40):
        eng.backward(dfeat * 2.0 ** j, dw, db)
        flags["dfeat x 2^%d" % j] = eng.grad_overflow()
        exact["dfeat x 2^%d" % j] = all(torch.equal(a, b * 2.0 ** j) for a, b in zip(list(dw) + list(db) + list(extra), ref))
    return flags, exact


GUARD_CONV = "inception_5b_3x3_bn"


def _conv_guard_flags(eng, precision, k):
    """one convolution's backward on its own (run_op, which bypasses the entry) on a dy scaled so that the largest gradient
    the tensor cores read (EXACT_TC: the planes of dz * grad_scale * 2^k, FAST: the fp16 storage) is 0.5x / 2x the fp16 range;
    k: the gradient exponent of the last backward, whose units ssnb_value_write stores the gradient in"""
    m = float(eng.read(GUARD_CONV, grad=True, planes=precision == "exact_tc").abs().max())
    dy = eng.read(GUARD_CONV, grad=True)
    op = [o for _kd, _i, o in eng.ops()].index(GUARD_CONV)
    flags = {}
    for f in (0.5, 2.0):
        eng.write(GUARD_CONV, dy * (f * HALF_MAX / (m * GRAD_SCALE * 2.0 ** k)), grad=True)
        eng.run_op(op, backward=True)
        flags["%s backward %.1fx" % (GUARD_CONV, f)] = eng.grad_overflow()
    return flags


@pytest.mark.parametrize("bn1_train", [False, True], ids=["frozen", "bn1"])
def test_grad_guard_exact_tc(bn1_train):
    """dfeat scaled by 2^+-40 raises no flag and scales every gradient exactly (the gradient exponent normalises the entry);
    a NaN in dfeat raises the flag, and reading it with clear=True clears it.  The split passes still guard the planes: a
    convolution's backward on its own (run_op, which bypasses the entry) on a dy scaled so that its largest plane is 0.5x / 2x
    the fp16 range leaves the flag clear / raises it; bn1: the same for bn_bwd_apply_kernel and conv1's dz"""
    from oracle import split_operands as SO
    dev = _cuda()
    eng = _engine("exact_tc", 8, 3, True, dev, bn1_train=bn1_train)
    try:
        extra = ()
        if bn1_train:
            bn, dgamma, dbeta = _bn1_module(3, dev)
            eng.set_bn1(bn, dgamma, dbeta)
            extra = (dgamma, dbeta)
        x, dfeat = _inputs(8, 3, dev)
        dw, db = _grads(3, dev)
        feat = eng.forward(x)
        eng.backward(dfeat, dw, db)
        flags = {"ordinary": eng.grad_overflow()}
        # the planes hold dz * grad_scale * 2^k with k chosen from this dfeat; a write stores dy times the same 2^k
        k = SO.grad_exponent(float(dfeat.abs().max()), GRAD_SCALE)
        flags.update(_conv_guard_flags(eng, "exact_tc", k))
        if bn1_train:
            dy = eng.read(S.BN1_OUT, grad=True)
            mb = float(eng.read(S.BN1_RAW, grad=True, planes=True).abs().max())
            bn_op = [kd for kd, _i, _o in eng.ops()].index("bn")
            for f in (0.5, 2.0):
                eng.write(S.BN1_OUT, dy * (f * HALF_MAX / (mb * GRAD_SCALE * 2.0 ** k)), grad=True)
                eng.run_op(bn_op, backward=True)
                flags["bn_bwd_apply %.1fx" % f] = eng.grad_overflow()
        f2, exact = _scaled_backward_flags(eng, dfeat, dw, db, extra)
        flags.update(f2)
        nan = dfeat.clone()
        nan[0, int(feat[0].argmax())] = float("nan")      # a channel that is active in frame 0
        eng.backward(nan, dw, db)
        flags["NaN in dfeat"] = eng.grad_overflow(clear=False)
        flags["NaN in dfeat, after clear"] = eng.grad_overflow(clear=True) and eng.grad_overflow()
        print("\nEXACT_TC F=8%s: flags %s; exactly scaled gradients %s" % (" bn1" if bn1_train else "", flags, exact))
        want = {"ordinary": False, "dfeat x 2^-40": False, "dfeat x 2^40": False, "NaN in dfeat": True, "NaN in dfeat, after clear": False,
                GUARD_CONV + " backward 0.5x": False, GUARD_CONV + " backward 2.0x": True}
        if bn1_train:
            want.update({"bn_bwd_apply 0.5x": False, "bn_bwd_apply 2.0x": True})
        assert flags == want
        assert all(exact.values()), exact
    finally:
        del eng
        torch.cuda.empty_cache()


def test_grad_guard_fast():
    """FAST stores gradients in fp16 times grad_scale * 2^k: dfeat scaled by 2^+-40 raises no flag and scales every gradient
    exactly; a NaN in dfeat raises the flag; an ordinary dfeat after it does not.  A convolution's backward on its own (run_op)
    on a dy whose fp16 storage would be 0.5x / 2x the fp16 range: clear / raised (the weight-gradient sums of an inf)"""
    from oracle import split_operands as SO
    dev = _cuda()
    eng = _engine("fast", 8, 3, True, dev)
    try:
        x, dfeat = _inputs(8, 3, dev)
        dw, db = _grads(3, dev)
        eng.forward(x)
        eng.backward(dfeat, dw, db)
        flags = {"ordinary": eng.grad_overflow()}
        flags.update(_conv_guard_flags(eng, "fast", SO.grad_exponent(float(dfeat.abs().max()), GRAD_SCALE)))
        f2, exact = _scaled_backward_flags(eng, dfeat, dw, db)
        flags.update(f2)
        nan = dfeat.clone()
        nan[0, 0] = float("nan")
        eng.backward(nan, dw, db)
        flags["NaN in dfeat"] = eng.grad_overflow()
        eng.backward(dfeat, dw, db)
        flags["ordinary again"] = eng.grad_overflow()
        print("\nFAST F=8: flags %s; exactly scaled gradients %s" % (flags, exact))
        assert flags == {"ordinary": False, "dfeat x 2^-40": False, "dfeat x 2^40": False, "NaN in dfeat": True, "ordinary again": False,
                         GUARD_CONV + " backward 0.5x": False, GUARD_CONV + " backward 2.0x": True}
        assert all(exact.values()), exact
    finally:
        del eng
        torch.cuda.empty_cache()
