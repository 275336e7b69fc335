"""The SSN training step around the backbone, against float64 (oracle/step_check.py): the fused global pool + dropout + STPP
of both tensor-core precisions, the STPP backward through each of its kernels, the heads + multi-task loss kernel at the
shapes where its passes and chunks have tails, its repeatability, data parallelism split over shards on one GPU, a
training trajectory run eagerly and replayed from a CUDA graph as bench.py runs it, and SSN with the reference's dropout.
Run on an H100: pytest -m gpu -s tests/test_gpu_step_tail.py."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ssn_oracle as O
from oracle import step_check as S
from oracle import synth

GRAD_SCALE = 4096.0
SSN_TABLE = S.part_table((1, (1, 2), 1), [2, 7, 9])                   # 5 parts over 2 + 5 + 2 segments
DEEP_TABLE = S.part_table(((1, 2), (1, 2, 4), 2), [4, 12, 16])        # 12 parts over 4 + 8 + 4 segments
WIDE_TABLE = S.part_table((1, (1, 2), 1), [5, 15, 20])                # 20 segments: beyond the vectorised kernels
# whole-network bars of the trajectory check (e), EXACT_TC against a float64 backbone at the same parameters: feat (worst
# row) and the four losses.  Measured on an H100 80GB HBM3 (400 W): 3.3e-4 and 9.4e-6 (loss_comp); the bars are about 4x.
TRAJ_FEAT_BAR, TRAJ_LOSS_BAR = 1.3e-3, 4e-5
TRAJ_MARGIN = 20.0
TRAJ_LR = 5e-5           # moves the oracle's feat by about 90x, and its total loss by about 190x, their bars per step


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _prec(name):
    from ssn_b200 import _lib
    return {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[name]


_BB = {}


def _bb():
    if "rgb" not in _BB:
        _BB["rgb"] = synth.synth_backbone(3, seed=0, calib_frames=2)
    return _BB["rgb"]


def _engine(precision, frames, dev):
    from ssn_b200.engine import BackboneEngine
    bb = _bb()
    names = [n for (n, *_r) in O.conv_layers(3)]
    eng = BackboneEngine(3, frames, _prec(precision), True, GRAD_SCALE, dev)
    eng.pack(*[[bb[n + k].to(dev) for n in names] for k in (".weight", ".bias", "_bn.weight", "_bn.bias", "_bn.running_mean",
                                                             "_bn.running_var")])
    return eng


def _ints(v):
    from ssn_b200 import _lib
    return _lib.int_array(v)


def _gpool(eng, mask, scaling, n_seg, table, course):
    from ssn_b200._lib import lib, check
    from ssn_b200.engine import _stream
    F_ = eng.frames
    n = F_ // n_seg
    dev = eng.device
    feat, crs = torch.empty(F_, 1024, device=dev), torch.empty(n, 1024, device=dev)
    stpp = torch.empty(n, len(table[0]) * 1024, device=dev)
    check(lib.ssnb_gpool_stpp_fwd(eng.h, None if mask is None else mask.data_ptr(), scaling.data_ptr(), n_seg, len(table[0]),
                                  *[_ints(t) for t in table], course[0], course[1], feat.data_ptr(), crs.data_ptr(),
                                  stpp.data_ptr(), _stream()), eng.h, "gpool_stpp_fwd")
    return feat, crs, stpp


def _stpp_bwd(d_course, d_stpp, scaling, n_seg, table, course, d_ft):
    from ssn_b200._lib import lib, check
    from ssn_b200.engine import _stream
    n, D = d_course.shape
    check(lib.ssnb_stpp_bwd(d_course.data_ptr(), d_stpp.data_ptr(), scaling.data_ptr(), n, n_seg, D, len(table[0]),
                            *[_ints(t) for t in table], course[0], course[1], d_ft.data_ptr(), _stream()), None, "stpp_bwd")


def _report(title, chk):
    print("\n%s:" % title, *chk.records, sep="\n  ")


# ---- (a) fused pool + STPP, STPP backward ----------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_pool_stpp_vs_float64(precision):
    """gpool_stpp_v2_kernel (fp32 / fp16 5b output) with SSN's table at F = 288, and the first-generation gpool_stpp_kernel
    with a 16-segment table at F = 48, each with and without a dropout mask, against float64 of the engine's own 5b output"""
    dev = _cuda()
    chk = S.Checker()
    g = torch.Generator().manual_seed(21)
    for frames, n_seg, table, course, kernel in ((288, 9, SSN_TABLE, (2, 7), "v2"), (48, 16, DEEP_TABLE, (4, 12), "first_gen")):
        eng = _engine(precision, frames, dev)
        x = synth.synth_frames(frames, 3, seed=23).to(dev)
        eng.forward(x)
        y5b = eng.read("inception_5b_output")
        assert y5b.shape == (frames, 1024, 7, 7)
        n = frames // n_seg
        scaling = torch.rand(n, 2, generator=g).to(dev)
        for masked in (False, True):
            mask = (torch.bernoulli(torch.full((frames, 1024), 0.2), generator=g) / 0.2).to(dev) if masked else None
            feat, crs, stpp = _gpool(eng, mask, scaling, n_seg, table, course)
            S.check_pool_stpp(chk, "%s F=%d%s" % (kernel, frames, " masked" if masked else ""), y5b, mask, scaling, table,
                              n_seg, course, feat, crs, stpp, bar=S.POOL_BARS[precision])
        del eng
    _report("gpool_stpp %s vs float64" % precision, chk)
    chk.assert_ok()


def test_stpp_backward_dispatch_vs_float64():
    """ssnb_stpp_bwd through stpp_bwd_v4_kernel<9, 8>, <16, 16> and the scalar kernel (a d_ft view 4 bytes off a 16-byte
    boundary, and 20 segments)"""
    dev = _cuda()
    chk = S.Checker()
    g = torch.Generator().manual_seed(22)
    n, D = 40, 1024
    for name, n_seg, table, course, misaligned in (("v4<9,8>", 9, SSN_TABLE, (2, 7), False),
                                                   ("v4<16,16>", 16, DEEP_TABLE, (4, 12), False),
                                                   ("scalar misaligned d_ft", 9, SSN_TABLE, (2, 7), True),
                                                   ("scalar n_seg=20", 20, WIDE_TABLE, (5, 15), False)):
        dc = torch.randn(n, D, generator=g).to(dev)
        ds = torch.randn(n, len(table[0]) * D, generator=g).to(dev)
        sc = torch.rand(n, 2, generator=g).to(dev)
        buf = torch.full((n * n_seg * D + 1,), float("nan"), device=dev)
        d_ft = (buf[1:] if misaligned else buf[:-1]).view(n * n_seg, D)
        assert (d_ft.data_ptr() % 16 != 0) == misaligned
        _stpp_bwd(dc, ds, sc, n_seg, table, course, d_ft)
        chk.add("stpp_bwd " + name, "dft", d_ft, S.stpp_vjp64(dc, ds, sc, table, n_seg, course), S.STPP_BWD_BAR, rows=True)
    _report("stpp_bwd vs float64", chk)
    chk.assert_ok()


# ---- (b) heads + loss kernel ----------------------------------------------------------------------------------------------
def _fcs(heads, dev):
    ns = types.SimpleNamespace
    return [ns(weight=heads[nm + ".weight"].to(dev), bias=heads[nm + ".bias"].to(dev))
            for nm in ("activity_fc", "completeness_fc", "regressor_fc")]


def _heads_kernel(case, dev, rows=None, global_videos=None, loss_scale=None):
    from ssn_b200.engine import heads_loss_fused
    c = case["cfg"]
    r = slice(None) if rows is None else rows
    t = {k: case[k][r].to(dev) for k in ("course", "stpp", "prop_type", "target", "reg_target")}
    out = heads_loss_fused(t["course"], t["stpp"], *_fcs(case["heads"], dev), t["prop_type"], t["target"], t["reg_target"],
                           c["num_class"], c["feat_mult"], c["fg_per_video"], c["comp_group"], c["props_per_video"],
                           global_videos=global_videos, loss_scale=c["loss_scale"] if loss_scale is None else loss_scale)
    torch.cuda.synchronize()
    return out


def _heads_ref(case, dev, rows=None, **cfg_kw):
    c = case["cfg"]
    r = slice(None) if rows is None else rows
    t = {k: case[k][r].to(dev) for k in ("course", "stpp", "prop_type", "target", "reg_target")}
    cfg = S.heads_cfg(t["course"].shape[0], c["props_per_video"], c["num_class"], c["feat_mult"], c["fg_per_video"],
                      c["comp_group"], **cfg_kw) if cfg_kw else c
    return S.heads_loss64(t["course"], t["stpp"], {k: v.to(dev) for k, v in case["heads"].items()}, t["prop_type"], t["target"],
                          t["reg_target"], cfg)


HEADS_CASES = {                          # videos, K, M and the layout of a video
    "bench": dict(videos=4, num_class=20, feat_mult=5),
    "baseline_K200": dict(videos=8, num_class=200, feat_mult=5),
    "rows40": dict(videos=5, num_class=20, feat_mult=5),                  # n = 40: a 32-row pass and a tail of 8
    "K22": dict(videos=4, num_class=22, feat_mult=5),                     # 3K = 66: a 64-column chunk and a tail of 2
    "fg2": dict(videos=4, num_class=20, feat_mult=5, fg_per_video=2),
    "neg64": dict(videos=2, num_class=20, feat_mult=5, comp_group=65, props_per_video=66),     # 64 negatives per group
    "deep_M12": dict(videos=4, num_class=20, feat_mult=12),               # 8 + 96 = 104 feature slices (CTAs)
}


@pytest.mark.parametrize("name", sorted(HEADS_CASES))
def test_heads_loss_kernel_vs_float64(name):
    dev = _cuda()
    case = S.heads_case(seed=31, **HEADS_CASES[name])
    out = _heads_kernel(case, dev)
    chk = S.Checker()
    S.check_heads(chk, "heads", out, _heads_ref(case, dev))
    _report("heads_loss_kernel %s (n=%d, K=%d, M=%d) vs float64" % (name, case["cfg"]["n"], case["cfg"]["num_class"],
                                                                    case["cfg"]["feat_mult"]), chk)
    chk.assert_ok()
    # a power-of-two loss_scale scales every gradient exactly and leaves logits and losses alone
    for s in (0.5, 8.0):
        o2 = _heads_kernel(case, dev, loss_scale=s)
        for k in ("raw_act", "raw_comp", "raw_reg", "losses"):
            assert torch.equal(o2[k], out[k]), (s, k)
        for k in S.PARAM_KEYS + ("d_course", "d_stpp"):
            assert torch.equal(o2[k], out[k] * s), (s, k)


# ---- (c) repeatability ----------------------------------------------------------------------------------------------------
def test_heads_loss_kernel_repeatable():
    """64 videos, K = 20: three calls give the same bits in every output, the losses included"""
    dev = _cuda()
    case = S.heads_case(64, 20, 5, seed=32)
    outs = [_heads_kernel(case, dev) for _ in range(3)]
    for o in outs[1:]:
        diff = [k for k in outs[0] if not torch.equal(o[k], outs[0][k])]
        assert not diff, (diff, outs[0]["losses"].tolist(), o["losses"].tolist())


# ---- (d) data parallelism on one GPU -------------------------------------------------------------------------------------
def test_heads_data_parallel_shards():
    """64 global videos in two shards of 32 with global_videos = 64, loss_scale = 1/2 (what each of two ranks runs): per-row
    outputs equal the full call's rows bit for bit, summed dW / db and mean losses match the full call, and the shards and
    the full call match heads_loss64 of the global batch"""
    dev = _cuda()
    case = S.heads_case(64, 20, 5, seed=33)
    full = _heads_kernel(case, dev)
    ref = _heads_ref(case, dev)
    halves = (slice(0, 256), slice(256, 512))
    shards = [_heads_kernel(case, dev, rows=r, global_videos=64, loss_scale=0.5) for r in halves]
    chk = S.Checker()
    S.check_heads(chk, "full", full, ref)
    for i, (r, sh) in enumerate(zip(halves, shards)):
        S.check_heads(chk, "shard %d" % i, sh, _heads_ref(case, dev, rows=r, global_videos=64, loss_scale=0.5))
        for k in S.ROW_KEYS:
            chk.add("shard %d vs global" % i, k, sh[k], ref[k][r], S.LOGIT_BAR, rows=True)
            assert torch.equal(sh[k], full[k][r]), (i, k)
    for k in S.PARAM_KEYS:
        summed = shards[0][k] + shards[1][k]
        chk.add("shards summed vs global", k, summed, ref[k], S.LOGIT_BAR)
        chk.add("shards summed vs full call", k, summed, full[k], S.LOGIT_BAR)
    mean = (shards[0]["losses"] + shards[1]["losses"]) / 2
    for i, q in enumerate(S.LOSS_NAMES):
        chk.add("shard mean vs global", q, mean[i:i + 1], ref["losses"][i:i + 1], S.LOSS_BAR, rows=True)
        chk.add("shard mean vs full call", q, mean[i:i + 1], full["losses"][i:i + 1], S.LOSS_BAR, rows=True)
    _report("heads, 64 videos as 2 x 32", chk)
    chk.assert_ok()


def _ssn(K, precision, heads_seed=0, dropout=0, grad_scale=1024.0, std=0.02, bias_std=0.1):
    import ssn_models
    dev = _cuda()
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=dropout, stpp_cfg=(1, (1, 2), 1))
    sd = m.state_dict()
    for k, v in _bb().items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=heads_seed, std=std, bias_std=bias_std).items():
        sd[k].copy_(v)
    m = m.to(dev).train()
    m.set_precision(_prec(precision), grad_scale)
    return m


def _rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def test_fused_step_data_parallel_shards():
    """SSN.fused_step in EXACT_TC on 4 videos, and on 2 + 2 videos in two model instances with global_videos = 4,
    loss_scale = 1/2: mean losses and summed gradients at test_dp_nccl.py's bars; the per-frame forward bit for bit"""
    dev = _cuda()
    K = 4
    batch = [t.to(dev) for t in synth.synth_batch(4, K, 3, seed=3)]
    full = _ssn(K, "exact_tc")
    l_full = full.fused_step(*batch).clone()
    parts = []
    for i in range(2):
        m = _ssn(K, "exact_tc")
        vs = slice(2 * i, 2 * i + 2)
        parts.append((m, m.fused_step(*[t[vs] for t in batch], global_videos=4, loss_scale=0.5).clone()))
    torch.cuda.synchronize()
    rows = {"feat": 144, "course": 16, "stpp": 16}
    for i, (m, _l) in enumerate(parts):
        for k, r in rows.items():
            assert torch.equal(m.last_fused[k], full.last_fused[k][i * r:(i + 1) * r]), (i, k)
    l_mean = (parts[0][1] + parts[1][1]) / 2
    num = den = worst = 0.0
    worst_name = ""
    p0, p1 = dict(parts[0][0].named_parameters()), dict(parts[1][0].named_parameters())
    for n_, q in full.named_parameters():
        if q.grad is None:
            continue
        gs = p0[n_].grad + p1[n_].grad
        e = _rel(gs, q.grad)
        num += float((gs.double() - q.grad.double()).pow(2).sum()); den += float(q.grad.double().pow(2).sum())
        if e > worst:
            worst, worst_name = e, n_
    r = {"losses": _rel(l_mean, l_full), "aggregate_grad": (num / den) ** 0.5, "worst_grad": worst}
    print("\nfused_step 4 videos as 2 + 2: %s (worst %s)" % ({k: "%.2e" % v for k, v in r.items()}, worst_name))
    assert r["losses"] < 1e-5 and r["aggregate_grad"] < 1e-4 and r["worst_grad"] < 2e-3, r


# ---- (e) training trajectory, eager and graph-replayed ---------------------------------------------------------------------
def _train(K, lr):
    """SSN at EXACT_TC with FusedSGD over flat buffers and a GradSync, as bench.py builds them (world 1: the sync is off)"""
    from ssn_b200.dp import GradSync
    from ssn_b200.optim import FusedSGD
    torch.manual_seed(0)
    model = _ssn(K, "exact_tc", std=0.01, bias_std=0.05)
    order = [p for p in model.parameters() if p.requires_grad]
    opt = FusedSGD(model.get_optim_policies(), lr=lr, momentum=0.9, weight_decay=5e-4, order=order,
                   on_step=[model.base_model.invalidate_packed])
    sync = GradSync(opt.flat_grad, order, model)
    assert not sync.enabled

    def step(batch):
        opt.flat_grad.zero_()
        losses = model.fused_step(*batch, global_videos=2, loss_scale=1.0, grad_sync=sync)
        sync.finish()
        opt.step()
        return losses
    return model, opt, step


def _params_at(model, opt, flat):
    """name -> tensor of the parameters held in `flat` (a copy of opt.flat_param); everything else from the model"""
    names = {id(p): n for n, p in model.named_parameters()}
    out = {k: v for k, v in model.state_dict().items()}
    for p, off, k in opt.views:
        out[names[id(p)]] = flat[off:off + k].view(p.shape)
    return out


def _oracle_step(params, batch, K, chunk=48):
    """float64 on the GPU: the backbone over the batch's frames, STPP, heads + loss at `params` -> (feat, losses)"""
    x, sc, tg, rt, pt = batch
    bb = {k[len("base_model."):]: v.double() for k, v in params.items() if k.startswith("base_model.") and not k.startswith("base_model.fc")}
    frames = x.reshape(-1, 3, 224, 224)
    with torch.no_grad():
        feat = torch.cat([O.backbone_forward(bb, frames[i:i + chunk].double(), 3) for i in range(0, frames.shape[0], chunk)])
    course, stpp = S.stpp64(feat, sc, SSN_TABLE, 9, (2, 7))
    n = course.shape[0]
    heads = {k: params[k] for k in S.HEAD_KEYS}
    ref = S.heads_loss64(course, stpp, heads, pt, tg, rt, S.heads_cfg(n, 8, K, 5))
    return feat, ref["losses"]


def _row_err(got, ref):
    got, ref = got.double(), ref.double()
    return float(((got - ref).abs().amax(1) / ref.abs().amax(1)).max())


def test_training_trajectory_eager_graph_and_oracle():
    """2 videos, EXACT_TC, FusedSGD(on_step=[invalidate_packed]) + GradSync, 3 warm-up steps then 4 steps alternating two
    batches.  The CUDA-graph twin (warm-up on a side stream, capture, replay on static inputs, bench.py's graphed()) matches
    the eager twin bit for bit after every step.  The eager twin's feat and losses are checked, step by step, against float64
    at the parameters read before that step, and the oracle's feat and losses move between consecutive parameter sets by at
    least TRAJ_MARGIN x their bars (so a step that ran with the previous step's packed weights would fail).  Every parameter
    update matches sgd64 of the step's own gradient and momentum."""
    dev = _cuda()
    K = 20
    batches = [tuple(t.to(dev) for t in synth.synth_batch(2, K, 3, seed=100 + i)) for i in range(2)]
    seq = [batches[i % 2] for i in range(4)]
    # eager twin
    m1, opt1, step1 = _train(K, TRAJ_LR)
    for _ in range(3):
        step1(batches[0])
    eager = []
    for b in seq:
        p0, mom0 = opt1.flat_param.clone(), opt1.flat_mom.clone()
        losses = step1(b).clone()
        torch.cuda.synchronize()
        eager.append(dict(p0=p0, mom0=mom0, losses=losses, feat=m1.last_fused["feat"].clone(), grad=opt1.flat_grad.clone(),
                          param=opt1.flat_param.clone(), mom=opt1.flat_mom.clone()))
    # graph twin
    m2, opt2, step2 = _train(K, TRAJ_LR)
    static = tuple(torch.empty_like(t) for t in batches[0])
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            for d_, s_ in zip(static, batches[0]):
                d_.copy_(s_)
            step2(static)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_losses = step2(static)
    for k, b in enumerate(seq):
        for d_, s_ in zip(static, b):
            d_.copy_(s_)
        graph.replay()
        torch.cuda.synchronize()
        e = eager[k]
        for name, got, want in (("losses", static_losses, e["losses"]), ("flat_param", opt2.flat_param, e["param"]),
                                ("flat_grad", opt2.flat_grad, e["grad"]), ("flat_mom", opt2.flat_mom, e["mom"])):
            assert torch.equal(got, want), (k, name)
    del graph
    # teacher-forced float64 oracle and the SGD update, on the eager twin's record
    chk = S.Checker()
    prev = None
    for k, (b, e) in enumerate(zip(seq, eager)):
        params = _params_at(m1, opt1, e["p0"])
        feat64, loss64 = _oracle_step(params, b, K)
        chk.add("step %d" % k, "feat", e["feat"], feat64, TRAJ_FEAT_BAR, rows=True)
        for i, q in enumerate(S.LOSS_NAMES):
            chk.add("step %d" % k, q, e["losses"][i:i + 1], loss64[i:i + 1], TRAJ_LOSS_BAR, rows=True)
        if prev is not None:
            # the same batch at the previous step's parameters
            feat_prev, loss_prev = _oracle_step(_params_at(m1, opt1, prev), b, K)
            mf = _row_err(feat_prev, feat64) / TRAJ_FEAT_BAR
            ml = float(((loss_prev - loss64).abs() / loss64.abs())[3]) / TRAJ_LOSS_BAR
            print("step %d: oracle moved by %.1f x the feat bar, %.1f x the total-loss bar" % (k, mf, ml))
            assert mf >= TRAJ_MARGIN and ml >= TRAJ_MARGIN, (k, mf, ml)
        prev = e["p0"]
        rp, rm = S.sgd64(e["p0"], e["grad"], e["mom0"], opt1._seg_end, opt1._seg_lr, opt1._seg_wd, opt1.momentum)
        S.check_sgd(chk, "sgd step %d" % k, opt1._seg_end, e["param"], e["mom"], rp, rm)
    _report("trajectory, 2 videos EXACT_TC, lr %g" % TRAJ_LR, chk)
    chk.assert_ok()


# ---- (f) SSN with the reference's dropout ---------------------------------------------------------------------------------
def test_fused_step_dropout_bench_shape():
    """fused_step at the bench shape (4 videos, K = 20, EXACT_TC) with dropout 0.8 (ssn_opts.py:11): the step keeps its mask,
    and course / stpp / losses / head gradients match float64 run with that mask, at test_fused_step_bench_shape's bars"""
    dev = _cuda()
    K = 20
    m = _ssn(K, "exact_tc", dropout=0.8, grad_scale=4096.0, std=0.01, bias_std=0.05)
    batch = [t.to(dev) for t in synth.synth_batch(4, K, 3, seed=100)]
    torch.manual_seed(12)
    losses = m.fused_step(*batch)
    torch.cuda.synchronize()
    lf = m.last_fused
    mask = lf["mask"]
    assert mask is not None and mask.shape == (288, 1024) and 0.15 < float((mask != 0).float().mean()) < 0.25
    x, sc, tg, rt, pt = batch
    bb = {k: v.to(dev).double() for k, v in _bb().items()}
    with torch.no_grad():
        feat = torch.cat([O.backbone_forward(bb, x.reshape(-1, 3, 224, 224)[i:i + 48].double(), 3) for i in range(0, 288, 48)])
    feat = feat * mask.double()
    course, stpp = S.stpp64(feat, sc, SSN_TABLE, 9, (2, 7))
    heads = {k: v.detach() for k, v in m.state_dict().items() if k in S.HEAD_KEYS}
    ref = S.heads_loss64(course, stpp, heads, pt, tg, rt, S.heads_cfg(32, 8, K, 5))
    params = dict(m.named_parameters())
    head_grad = {k: params[k].grad for k in S.HEAD_KEYS}
    ref_grad = {"activity_fc.weight": ref["d_act_w"], "activity_fc.bias": ref["d_act_b"], "completeness_fc.weight": ref["d_comp_w"],
                "completeness_fc.bias": ref["d_comp_b"], "regressor_fc.weight": ref["d_reg_w"], "regressor_fc.bias": ref["d_reg_b"]}
    num = sum(float((head_grad[k].double() - ref_grad[k]).pow(2).sum()) for k in S.HEAD_KEYS)
    den = sum(float(ref_grad[k].pow(2).sum()) for k in S.HEAD_KEYS)
    e = {"feat": _rel(lf["feat"], feat), "course": _rel(lf["course"], course), "stpp": _rel(lf["stpp"], stpp),
         "loss": float((losses.double() - ref["losses"]).abs().max() / ref["losses"].abs().max()), "head_grads": (num / den) ** 0.5}
    print("\nfused_step F=288 dropout 0.8 (exact_tc) vs float64: %s" % {k: "%.3e" % v for k, v in e.items()})
    bars = {"feat": 2e-4, "course": 2e-4, "stpp": 2e-4, "loss": 1e-4, "head_grads": 5e-4}
    for k, b in bars.items():
        assert e[k] < b, (k, e[k], b)
