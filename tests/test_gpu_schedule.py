"""Every launch of the real backbone schedule (ssnb_backbone_fwd + ssnb_backbone_bwd: fused sibling 1x1 launches, last-writer
masking, bias gradients on the weight-gradient MMAs, max-pool backward folded into conv1 / conv2_3x3, batched weight-gradient
finalize, conv1 straight from the NCHW input) held to a per-launch float64 bar (oracle/schedule_check.py), at the frame
count bench.py times and at frame counts that leave partial tiles in every TMA box and split-K range.  Run on an H100:
pytest -m gpu -s tests/test_gpu_schedule.py."""
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import schedule_check as S
from oracle import ssn_oracle as O
from oracle import synth

GRAD_SCALE = 4096.0

# (precision, frames, in_channels, SSNB_DISABLE_FUSION)
CASES = [("exact_tc", 288, 3, False), ("exact_tc", 37, 3, False), ("exact_tc", 1, 3, False),
         ("fast", 288, 3, False), ("fast", 37, 3, False), ("fast", 1, 3, False),
         ("exact_tc", 37, 10, False), ("fast", 37, 10, False),
         ("exact_tc", 37, 3, True), ("fast", 37, 3, True),
         ("exact", 37, 3, False)]


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


_WEIGHTS = {}


def _weights(in_channels):
    if in_channels not in _WEIGHTS:
        _WEIGHTS[in_channels] = synth.synth_backbone(in_channels, seed=0, calib_frames=2)
    return _WEIGHTS[in_channels]


def _engine(precision, frames, in_channels, env, dev):
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    prec = {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return BackboneEngine(in_channels, frames, prec, True, GRAD_SCALE, dev)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("precision,frames,in_channels,unfused", CASES,
                         ids=["%s-F%d-c%d%s" % (p, f, c, "-unfused" if u else "") for p, f, c, u in CASES])
def test_schedule_per_launch(precision, frames, in_channels, unfused):
    dev = _cuda()
    t0 = time.time()
    bb = _weights(in_channels)
    names = [n for (n, *_r) in O.conv_layers(in_channels)]
    eng = _engine(precision, frames, in_channels, {"SSNB_DISABLE_FUSION": "1" if unfused else "0"}, dev)
    try:
        eng.pack([bb[n + ".weight"].to(dev) for n in names], [bb[n + ".bias"].to(dev) for n in names],
                 [bb[n + "_bn.weight"].to(dev) for n in names], [bb[n + "_bn.bias"].to(dev) for n in names],
                 [bb[n + "_bn.running_mean"].to(dev) for n in names], [bb[n + "_bn.running_var"].to(dev) for n in names])
        x = synth.synth_frames(frames, in_channels, seed=17).to(dev)
        dfeat = (torch.randn(frames, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
        feat = eng.forward(x)
        dw = [torch.zeros(bb[n + ".weight"].shape, device=dev) for n in names]
        db = [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in names]
        eng.backward(dfeat, dw, db)
        torch.cuda.synchronize()
        assert not eng.grad_overflow()
        t1 = time.time()
        recs = S.check_schedule(eng, bb, x, feat, dfeat, dw, db, precision, in_channels)
        t2 = time.time()
        worst = {}
        for r in recs:                 # worst value per quantity, for the records in DESIGN.md
            if r.quantity not in worst or r.err > worst[r.quantity].err:
                worst[r.quantity] = r
        print("\n%s F=%d in_channels=%d%s: %d records, engine %.1f s, float64 check %.1f s; worst per quantity: %s"
              % (precision, frames, in_channels, " SSNB_DISABLE_FUSION=1" if unfused else "", len(recs), t1 - t0, t2 - t1,
                 ", ".join("%s %.2e (%s)" % (q, r.err, r.op) for q, r in worst.items())))
        print("  5 worst records (closest to their bars):", *S.worst(recs), sep="\n    ")
        bad = S.failures(recs)
        assert not bad, "\n".join(map(repr, bad))
        if precision == "exact_tc" and frames == 37 and in_channels == 3 and not unfused:
            # split-K partials are reduced in a fixed order: the schedule is bitwise reproducible, and accumulation adds
            # exactly the same gradients again
            assert torch.equal(eng.forward(x), feat)
            dw1, db1 = [t.clone() for t in dw], [t.clone() for t in db]
            eng.backward(dfeat, dw, db, accumulate=True)
            torch.cuda.synchronize()
            assert all(torch.equal(a, 2 * b) for a, b in zip(dw, dw1)), [n for n, a, b in zip(names, dw, dw1) if not torch.equal(a, 2 * b)]
            assert all(torch.equal(a, 2 * b) for a, b in zip(db, db1)), [n for n, a, b in zip(names, db, db1) if not torch.equal(a, 2 * b)]
    finally:
        del eng
        torch.cuda.empty_cache()
