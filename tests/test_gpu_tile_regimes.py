"""The backbone swept over frame counts that reach every tile-schedule regime of the wgmma kernels (oracle/tile_plan.py,
tests/test_tile_regimes.py), and the two benchmarked training shapes outside the frame counts tests/test_gpu_schedule.py
runs: configs[3] (ActivityNet heads, 8 videos = 576 frames per GPU) and configs[2] (Flow, 288 frames of 10 channels).

Each case first holds the launch log of one forward + backward (ssnb_timing_launches: every umma_conv_kernel's tile count
and tile width, every umma_wgrad_kernel's CTAs per split and split count) to the plan restatement on this device's SM
count, launch by launch, then checks every launch against float64 with the per-launch bars of oracle/schedule_check.py,
unchanged.  Cases whose workspace and float64 check do not fit in the free device memory are skipped with both numbers.
Run on an H100: pytest -m gpu -s tests/test_gpu_tile_regimes.py."""
import ctypes as C
import gc
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import schedule_check as S
from oracle import ssn_oracle as O
from oracle import step_check as SC
from oracle import synth
from oracle import tile_plan as T

GRAD_SCALE = 4096.0
GIB = 1 << 30


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_WEIGHTS = {}


def _weights(in_channels):
    if in_channels not in _WEIGHTS:
        _WEIGHTS[in_channels] = synth.synth_backbone(in_channels, seed=0, calib_frames=2)
    return _WEIGHTS[in_channels]


def _prec(precision):
    from ssn_b200 import _lib
    return {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[precision]


# ---- memory guard --------------------------------------------------------------------------------------------------------
def workspace_bytes(precision, frames, in_channels, training=True, bn1_train=False):
    """ssnb_workspace_bytes of the engine's plan (no device memory is touched)"""
    from ssn_b200 import _lib
    cfg = _lib.Config(in_channels, frames, _prec(precision), 1 if training else 0, GRAD_SCALE, 1 if bn1_train else 0)
    h = C.c_void_p()
    _lib.check(_lib.lib.ssnb_create(C.byref(cfg), C.byref(h)), None, "ssnb_create")
    try:
        return int(_lib.lib.ssnb_workspace_bytes(h))
    finally:
        _lib.lib.ssnb_destroy(h)


def check_peak_bytes(frames, in_channels):
    """what the case holds besides the workspace, at most: the input, dfeat, feat, the gradients and the float64 check, whose
    reader keeps up to five fp32 tensors of the largest value (conv1's 64 x 112 x 112 output) and works in 16-frame float64
    chunks.  tests below print the measured peak beside it."""
    largest = 64 * 112 * 112 * 4
    return frames * (6 * largest + in_channels * 224 * 224 * 4 + 3 * 1024 * 4) + 2 * GIB


def _need_memory(label, ws, frames, in_channels):
    gc.collect()
    torch.cuda.empty_cache()
    need = ws + check_peak_bytes(frames, in_channels)
    free, total = torch.cuda.mem_get_info()
    if need > free:
        pytest.skip("%s needs %.1f GiB (workspace %.1f GiB + check %.1f GiB), %.1f GiB of %.1f GiB are free"
                    % (label, need / GIB, ws / GIB, (need - ws) / GIB, free / GIB, total / GIB))
    return need


# ---- one case ------------------------------------------------------------------------------------------------------------
def _engine(precision, frames, in_channels, dev, bn1_train=False):
    from ssn_b200.engine import BackboneEngine
    old = os.environ.pop("SSNB_DISABLE_FUSION", None)      # the default schedule (fusion on)
    try:
        eng = BackboneEngine(in_channels, frames, _prec(precision), True, GRAD_SCALE, dev, bn1_train=bn1_train)
    finally:
        if old is not None:
            os.environ["SSNB_DISABLE_FUSION"] = old
    bb = _weights(in_channels)
    names = [n for (n, *_r) in O.conv_layers(in_channels)]
    eng.pack(*[[bb[n + k].to(dev) for n in names] for k in (".weight", ".bias", "_bn.weight", "_bn.bias", "_bn.running_mean",
                                                             "_bn.running_var")])
    return eng


def assert_launches_predicted(log, in_channels, frames, precision, sms):
    """the umma launches of one forward + backward equal the restated plan's, in order; returns the plan"""
    got = T.parse_launch_log(log)
    if precision == "exact":
        assert got == [], got[:5]
        return []
    plan = T.schedule(in_channels, frames, precision, sms)
    want = [T.log_key(l) for l in plan]
    bad = [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert len(got) == len(want) and not bad, \
        "%d launches logged, %d predicted; first differences (index, logged, predicted): %s" % (len(got), len(want), bad[:5])
    return plan


def _regime_summary(plan):
    n = {}
    for l in plan:
        for r in T.regimes(l):
            n[r] = n.get(r, 0) + 1
    return ", ".join("%s %d" % kv for kv in sorted(n.items()))


def _run_engine(precision, frames, in_channels, bn1_train, dev):
    """one forward + backward with the launch log open, and the per-launch check of it; the engine is gone on return, so a
    failing assertion of the caller holds no workspace"""
    from ssn_b200 import _lib
    bb = _weights(in_channels)
    names = [n for (n, *_r) in O.conv_layers(in_channels)]
    eng = _engine(precision, frames, in_channels, dev, bn1_train)
    try:
        bn1 = None
        if bn1_train:
            bn = torch.nn.BatchNorm2d(64).to(dev)
            with torch.no_grad():
                for k in ("weight", "bias", "running_mean", "running_var"):
                    getattr(bn, k).copy_(bb["conv1_7x7_s2_bn." + k])
            dgamma, dbeta = torch.zeros(64, device=dev), torch.zeros(64, device=dev)
            eng.set_bn1(bn, dgamma, dbeta)
            rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        x = synth.synth_frames(frames, in_channels, seed=17).to(dev)
        dfeat = (torch.randn(frames, 1024, generator=torch.Generator().manual_seed(18)) * 0.01).to(dev)
        dw = [torch.zeros(bb[n + ".weight"].shape, device=dev) for n in names]
        db = [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in names]
        torch.cuda.synchronize()
        _lib.lib.ssnb_timing_begin(C.c_void_p(torch.cuda.current_stream().cuda_stream))
        feat = eng.forward(x)
        eng.backward(dfeat, dw, db)
        log = _lib.lib.ssnb_timing_launches().decode()
        torch.cuda.synchronize()
        overflow = eng.grad_overflow()
        if bn1_train:
            bn1 = dict(gamma=bn.weight.detach(), beta=bn.bias.detach(), momentum=bn.momentum, eps=bn.eps, running_mean0=rm0,
                       running_var0=rv0, running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone(), dgamma=dgamma,
                       dbeta=dbeta)
        t1 = time.time()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        recs = S.check_schedule(eng, bb, x, feat, dfeat, dw, db, precision, in_channels, bn1=bn1)
        peak = torch.cuda.max_memory_allocated() - base + (x.numel() + dfeat.numel() + feat.numel()) * 4
        return dict(ws=eng.workspace_bytes, log=log, overflow=overflow, recs=recs, peak=peak, t_check=time.time() - t1)
    finally:
        del eng
        gc.collect()
        torch.cuda.empty_cache()


def run_case(label, precision, frames, in_channels=3, bn1_train=False):
    """predict + per-launch float64 check of one training engine; returns the records"""
    dev = _cuda()
    t0 = time.time()
    ws = workspace_bytes(precision, frames, in_channels, True, bn1_train)
    need = _need_memory(label, ws, frames, in_channels)
    sms = _sms()
    r = _run_engine(precision, frames, in_channels, bn1_train, dev)
    assert r["ws"] == ws and not r["overflow"]
    plan = assert_launches_predicted(r["log"], in_channels, frames, precision, sms)
    recs = r["recs"]
    print("\n%s: %s F=%d in_channels=%d%s on %d SMs: %d umma launches as predicted (%s); %d records, worst %s; %.1f s (check "
          "%.1f s); memory: workspace %.1f GiB, check %.2f GiB measured / %.2f GiB allowed"
          % (label, precision, frames, in_channels, " bn1_train" if bn1_train else "", sms, len(plan), _regime_summary(plan),
             len(recs), S.worst(recs, 1)[0], time.time() - t0, r["t_check"], ws / GIB, r["peak"] / GIB, (need - ws) / GIB))
    bad = S.failures(recs)
    assert not bad, "\n".join(map(repr, bad))
    assert r["peak"] <= need - ws, "the memory guard's estimate of the check is too small: %.2f GiB measured" % (r["peak"] / GIB)
    return recs


# ---- the frame-count sweep -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frames", T.FRAME_SET)
@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_frame_sweep(precision, frames):
    """the frame counts of tile_plan.FRAME_SET, which together reach every (launch, regime) pair the range [1, 640] reaches
    on a 132-SM card; on another SM count the coverage of the set there is printed"""
    _cuda()
    sms = _sms()
    if sms != T.SMS_H100_SXM and frames == T.FRAME_SET[0] and precision == "exact_tc":
        per = {f: T.reached(3, f, sms) for f in T.FRAME_SET}
        cov = set().union(*per.values())
        allp = set().union(*(T.reached(3, f, sms) for f in range(1, T.FRAME_RANGE + 1)))
        print("\n%d SMs: the frame set reaches %d of %d (precision, launch, regime) pairs" % (sms, len(cov), len(allp)))
    run_case("sweep", precision, frames)


def test_frame_sweep_exact_fp32():
    """EXACT_FP32 (SIMT kernels only: no wgmma launch in the log) at one frame count of the set"""
    run_case("sweep", "exact", 41)


# ---- the benchmarked training shapes -------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_flow_288(precision):
    """configs[2]: Flow, 288 frames of 10 channels (conv1 over a 40-channel space-to-depth input)"""
    run_case("configs[2] Flow", precision, 288, 10)


@pytest.mark.parametrize("precision,bn1_train", [("fast", False), ("exact_tc", False), ("exact_tc", True)],
                         ids=["fast", "exact_tc", "exact_tc-bn1"])
def test_frames_576(precision, bn1_train):
    """configs[3]: 8 videos x 8 proposals x 9 segments = 576 frames per GPU"""
    run_case("configs[3] backbone", precision, 576, 3, bn1_train)


def test_fused_step_configs3():
    """configs[3]'s heads and loss: 8 videos, K = 200, through step_check (a seeded heads case, then one SSN.fused_step in
    EXACT_TC at 576 frames): the step's pool + STPP, heads + loss, STPP backward at step_check's bars, and its backbone
    forward + backward launch by launch at schedule_check's bars, on the dfeat the step handed the backbone"""
    import types
    import ssn_models
    from ssn_b200 import _lib
    from ssn_b200.engine import _stream, heads_loss_fused
    dev = _cuda()
    t0 = time.time()
    videos, K, frames = 8, 200, 576
    chk = SC.Checker()
    # the heads + loss kernel on a seeded case of this shape
    case = SC.heads_case(videos, K, 5, seed=41)
    fcs = [types.SimpleNamespace(weight=case["heads"][n + ".weight"].to(dev), bias=case["heads"][n + ".bias"].to(dev))
           for n in ("activity_fc", "completeness_fc", "regressor_fc")]
    t = {k: case[k].to(dev) for k in ("course", "stpp", "prop_type", "target", "reg_target")}
    out = heads_loss_fused(t["course"], t["stpp"], *fcs, t["prop_type"], t["target"], t["reg_target"], K, 5)
    SC.check_heads(chk, "heads (seeded case)", out, SC.heads_loss64(t["course"], t["stpp"], {k: v.to(dev) for k, v in case["heads"].items()},
                                                                   t["prop_type"], t["target"], t["reg_target"], case["cfg"]))
    # one fused step
    ws = workspace_bytes("exact_tc", frames, 3)
    need = _need_memory("fused_step at configs[3]", ws, frames, 3)
    bb = _weights(3)
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    sd = m.state_dict()
    for k, v in bb.items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1).items():
        sd[k].copy_(v)
    m = m.to(dev).train()
    m.set_precision(_lib.EXACT_TC, GRAD_SCALE)
    batch = [x.to(dev) for x in synth.synth_batch(videos, K, 3, seed=7)]
    x, sc, tg, rt, pt = batch
    try:
        m.fused_step(*batch)
        torch.cuda.synchronize()
        lf = m.last_fused
        eng = next(iter(m.base_model._engines.values()))
        assert eng.frames == frames and not eng.grad_overflow()
        table = SC.part_table((1, (1, 2), 1), [2, 7, 9])
        sc2 = sc.contiguous().float().view(-1, 2)
        n = frames // 9
        SC.check_pool_stpp(chk, "gpool_stpp", eng.read("inception_5b_output"), None, sc2, table, 9, (2, 7), lf["feat"], lf["course"],
                           lf["stpp"], bar=SC.POOL_BARS["exact_tc"])
        heads = {k: v.detach() for k, v in m.state_dict().items() if k in SC.HEAD_KEYS}
        ref = SC.heads_loss64(lf["course"], lf["stpp"], heads, pt, tg, rt, SC.heads_cfg(n, 8, K, 5))
        gap = SC.ohem_gap(ref["raw_comp"], pt, tg, SC.heads_cfg(n, 8, K, 5))
        assert gap >= SC.OHEM_GAP, "an OHEM choice of this batch is within %.1e of a tie" % gap
        SC.check_heads(chk, "heads (fused_step)", lf, ref)
        # the STPP backward again (deterministic): the dfeat the backbone's backward consumed
        dft = torch.empty(frames, 1024, device=dev)
        lo, hi, nm, col = table
        _lib.check(_lib.lib.ssnb_stpp_bwd(lf["d_course"].data_ptr(), lf["d_stpp"].data_ptr(), sc2.data_ptr(), n, 9, 1024, len(lo),
                                          _lib.int_array(lo), _lib.int_array(hi), _lib.int_array(nm), _lib.int_array(col), 2, 7,
                                          dft.data_ptr(), _stream()), None, "stpp_bwd")
        chk.add("stpp_bwd", "dft", dft, SC.stpp_vjp64(lf["d_course"], lf["d_stpp"], sc2, table, 9, (2, 7)), SC.STPP_BWD_BAR, rows=True)
        t1 = time.time()
        cs = m.base_model._convs()
        recs = S.check_schedule(eng, bb, x.reshape(-1, 3, 224, 224), lf["feat"], dft, [c.weight.grad for c in cs],
                                [c.bias.grad for c in cs], "exact_tc", 3)
        t2 = time.time()
        print("\nfused_step configs[3] (8 videos, K=200, F=576, exact_tc): step_check records:", *chk.records, sep="\n  ")
        print("  backbone: %d records, worst %s; OHEM gap %.1e; step + step_check %.1f s, per-launch check %.1f s; memory need "
              "%.1f GiB (workspace %.1f GiB)" % (len(recs), S.worst(recs, 1)[0], gap, t1 - t0, t2 - t1, need / GIB, ws / GIB))
        chk.assert_ok()
        bad = S.failures(recs)
        assert not bad, "\n".join(map(repr, bad))
    finally:
        del m
        torch.cuda.empty_cache()
