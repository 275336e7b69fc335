"""The training loop's update block on the device against the reference's loop and plain float64 / numpy restatements of
each kernel's rule (oracle/train_loop_oracle.py): gradient accumulation over micro-batches is an exact fp32 sum, the
reference's iter_size / clip schedule end to end (eager and CUDA-graph replayed), the reference's own update blocks and
accuracy() batches (tests/golden/train_loop.npz), and ssnb_train_meters, ssnb_grad_norm, ssnb_grad_clip and
ssnb_sgd_step_groups_clipped swept through their shapes, alignments, magnitudes and boundaries.  Run on an H100:
pytest -m gpu -s tests/test_gpu_update_block.py."""
import ctypes as C
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import binary_oracle as B
from oracle import synth
from oracle import train_loop_oracle as TL

SSN_FLAT = 10578993              # the flat gradient buffer of SSN(K=20) on BNInception: what ssnb_grad_clip scales per step
FLT_MAX = float(np.finfo(np.float32).max)
_BB = {}


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _prec(name):
    from ssn_b200 import _lib
    return {"exact_tc": _lib.EXACT_TC, "fast": _lib.FAST_FP16}[name]


def _bb():
    if "rgb" not in _BB:
        _BB["rgb"] = synth.synth_backbone(3, seed=0, calib_frames=2)
    return _BB["rgb"]


def _ssn(prec, bn_mode="frozen", dropout=0.8, K=20):
    import ssn_models
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=dropout, bn_mode=bn_mode)
    sd = m.state_dict()
    for k, v in _bb().items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1).items():
        sd[k].copy_(v)
    m = m.to(_cuda()).train()
    m.set_precision(_prec(prec), 1024.0)
    return m


def _binary(prec, dropout=0.8, K=2):
    import binary_model
    m = binary_model.BinaryClassifier(K, 5, "RGB", base_model="BNInception", dropout=dropout)
    sd = m.state_dict()
    for k, v in _bb().items():
        sd["base_model." + k].copy_(v)
    for k, v in B.synth_classifier(K, seed=0).items():
        sd[k].copy_(v)
    m = m.to(_cuda()).train()
    m.set_precision(_prec(prec), 1024.0)
    return m


def _opt(m, lr=1e-3):
    from ssn_b200.optim import FusedSGD
    order = [p for p in m.parameters() if p.requires_grad]
    return FusedSGD(m.get_optim_policies(), lr=lr, momentum=0.9, weight_decay=5e-4, order=order,
                    on_step=[m.base_model.invalidate_packed])


def _extras(tensors):
    from ssn_b200._lib import ExtraGrads
    ex = ExtraGrads()
    ex.count = len(tensors)
    for i, t in enumerate(tensors):
        ex.grad[i], ex.numel[i] = (t.data_ptr() if t.numel() else None), t.numel()
    return ex


def _ulps(got, want):
    """|got - want| in fp32 units in the last place at want (want may be float64)"""
    got, want = np.asarray(got, np.float32).astype(np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)


def _bits_equal(got, want):
    """bitwise, except that a NaN matches any NaN (the device writes the canonical NaN, numpy keeps the operand's bits)"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and got[~nan].tobytes() == want[~nan].tobytes()


def _first_mismatch(opt, m, got, want):
    names = {id(p): n for n, p in m.named_parameters()}
    for p, off, k in opt.views:
        a, b = got[off:off + k], want[off:off + k]
        if not torch.equal(a, b):
            bad = int((a != b).sum())
            return "%s: %d of %d elements, worst %.3g" % (names[id(p)], bad, k, float((a - b).abs().max()))
    return "none"


# ---- 1. accumulation is a sum --------------------------------------------------------------------------------------------
def _micro(kind, m, opt, batch, seed, sync):
    """one micro-batch's forward + backward, adding into .grad; returns its outputs (losses and what the step keeps)"""
    torch.cuda.manual_seed(seed)
    if kind == "ssn_partial":
        from ops.ssn_ops import ClassWiseRegressionLoss, CompletenessLoss
        a, at, c, ct, r, rl, rtg = m(*batch)
        act = torch.nn.CrossEntropyLoss()(a, at)
        comp = CompletenessLoss()(c, ct, 1, 7)
        reg = ClassWiseRegressionLoss()(r, rl, rtg)
        loss = act + 0.1 * comp + 0.1 * reg
        loss.backward()
        opt.rebind_grads()
        return [t.detach().clone() for t in (act, comp, reg, loss, a, c, r)]
    losses = m.fused_step(*batch, grad_sync=sync)
    if sync is not None:
        sync.finish()
    return [losses.clone()] + [v.clone() for _k, v in sorted(m.last_fused.items()) if isinstance(v, torch.Tensor)]


@pytest.mark.parametrize("kind,bucketed,prec", [(k, b, p) for k, b in (("ssn", False), ("ssn", True), ("binary", False), ("binary", True))
                                                for p in ("exact_tc", "fast")] + [("ssn_partial", False, "exact_tc")])
def test_accumulation_is_a_sum(kind, bucketed, prec):
    """micro-batch A then B without zeroing leaves fl(gA + gB) in the flat buffer and the extras, bitwise, where gA and gB
    are what each leaves alone; every output of each micro-batch is that of its separate run (dfeat, dcourse and the head
    gradients of a step do not accumulate).  Every gradient writer adds one fp32 rounding of its sum to the old value.
    bn_mode='partial' trains through the module path (BackboneFunction) in EXACT_TC only; its dγ / dβ are the extras."""
    from ssn_b200.dp import GradSync
    dev = _cuda()
    if kind == "binary":
        make = lambda: _binary(prec)                                       # noqa: E731
        batches = [tuple(t.to(dev) for t in B.synth_binary_batch(2, 4, 2, 3, seed=s)) for s in (21, 22)]
    else:
        make = lambda: _ssn(prec, bn_mode="partial" if kind == "ssn_partial" else "frozen")  # noqa: E731
        batches = [tuple(t.to(dev) for t in synth.synth_batch(2, 20, seed=s)) for s in (21, 22)]
    twins = []
    for _ in range(2):
        m = make()
        opt = _opt(m)
        sync = GradSync(opt.flat_grad, [p for p in m.parameters() if p.requires_grad], m) if bucketed else None
        twins.append((m, opt, sync, opt.ungrouped(m.parameters())))
    assert len(twins[0][3]) == (2 if kind == "ssn_partial" else 0)
    # twin 0: zero before each micro-batch
    m, opt, sync, extra = twins[0]
    sep, g, e = [], [], []
    for i, batch in enumerate(batches):
        opt.zero_grad()
        for p in extra:
            p.grad = None
        sep.append(_micro(kind, m, opt, batch, 7 + i, sync))
        g.append(opt.flat_grad.clone())
        e.append([p.grad.clone() for p in extra])
    assert all(float(t.abs().sum()) > 0 for t in g), "a micro-batch left no gradient"
    # twin 1: A then B into the same buffers
    m, opt, sync, extra = twins[1]
    opt.zero_grad()
    for i, batch in enumerate(batches):
        outs = _micro(kind, m, opt, batch, 7 + i, sync)
        assert len(outs) == len(sep[i])
        for j, (a, b) in enumerate(zip(outs, sep[i])):
            assert torch.equal(a, b), ("micro-batch output differs from its separate run", i, j)
    want = g[0] + g[1]
    assert torch.equal(opt.flat_grad, want), _first_mismatch(opt, m, opt.flat_grad, want)
    for p, a, b in zip(extra, e[0], e[1]):
        assert torch.equal(p.grad, a + b), ("extra gradient", tuple(p.shape))
    if bucketed:
        assert len(sync.launched) > 1


# ---- 2. the reference's loop, end to end ---------------------------------------------------------------------------------
def _per_tensor_err(opt, got, want):
    worst = 0.0
    for _p, off, k in opt.views:
        ref = want[off:off + k]
        scale = np.abs(ref).max()
        if scale > 0:
            worst = max(worst, float(np.abs(got[off:off + k] - ref).max() / scale))
    return worst


@pytest.mark.parametrize("iter_size", [1, 3])
@pytest.mark.parametrize("clip", ["none", "below", "above"])
def test_reference_loop_vs_float64(iter_size, clip):
    """2 * iter_size + 1 micro-batches on the reference's schedule (a step after micro-batch 0, then after every iter_size
    more), each step FusedSGD.step(1 / iter_size, max_norm) then zero_grad; the oracle runs the update block in float64 on
    the gradients each micro-batch leaves alone (a zeroing twin at the same parameters and dropout seed)"""
    from ssn_b200.meters import StepMeters
    dev = _cuda()
    m, z = _binary("exact_tc"), _binary("exact_tc")
    opt, oz = _opt(m, lr=0.05), _opt(z, lr=0.05)
    meters = StepMeters("binary", dev)
    batches = [tuple(t.to(dev) for t in B.synth_binary_batch(2, 4, 2, 3, seed=s)) for s in (31, 32)]
    sizes = np.array([k for _p, _o, k in opt.views])
    lr = np.repeat(opt._seg_lr.double().cpu().numpy(), sizes)
    wd = np.repeat(opt._seg_wd.double().cpu().numpy(), sizes)
    p64 = opt.flat_param.double().cpu().numpy()
    b64 = np.zeros_like(p64)
    acc = np.zeros_like(p64)
    mbuf = np.zeros((4, 2))
    max_norm, worst, steps = None, [0.0, 0.0, 0.0], 0
    for i, step in enumerate(TL.step_schedule(2 * iter_size + 1, iter_size)):
        x, target = batches[i % 2]
        oz.flat_param.copy_(opt.flat_param)
        z.base_model.invalidate_packed()
        oz.zero_grad()
        torch.cuda.manual_seed(100 + i)
        z.fused_step(x, target)
        gi = oz.flat_grad.double().cpu().numpy()
        acc += gi
        torch.cuda.manual_seed(100 + i)
        loss = m.fused_step(x, target, meters=meters)
        TL.meters_update(mbuf, m.last_fused["logits"].cpu().numpy(), target.reshape(-1).cpu().numpy(), None,
                         loss.cpu().numpy(), x.size(0))
        assert meters.buf.cpu().numpy().tobytes() == mbuf.tobytes(), (i, meters.buf, mbuf)
        if not step:
            continue
        norm64 = float(np.linalg.norm(acc / iter_size))
        if max_norm is None and clip != "none":
            max_norm = norm64 * (0.5 if clip == "below" else 2.0)
        c = None
        if clip == "none":
            assert opt.step(grad_mult=1.0 / iter_size) is None
        else:
            norm = float(opt.step(grad_mult=1.0 / iter_size, max_norm=max_norm))
            worst[2] = max(worst[2], abs(norm - norm64) / norm64)
            c = float(np.float32(max_norm)) / (norm64 + 1e-6)
            c = c if c < 1 else None
        g = acc / iter_size * (1.0 if c is None else c)
        b64 = 0.9 * b64 + g + wd * p64
        p64 = p64 - lr * b64
        worst[0] = max(worst[0], _per_tensor_err(opt, opt.flat_param.double().cpu().numpy(), p64))
        worst[1] = max(worst[1], _per_tensor_err(opt, opt.flat_mom.double().cpu().numpy(), b64))
        opt.zero_grad()
        acc[:] = 0
        steps += 1
    print("iter_size %d clip %s: %d steps, param %.2e momentum %.2e norm %.2e" % (iter_size, clip, steps, *worst))
    assert steps == 3
    assert worst[0] <= 1e-6 and worst[1] <= 1e-6 and worst[2] <= 1e-6, worst


def test_accumulation_period_graph_replay_equals_eager():
    """one whole period (iter_size = 3 fused_steps with meters, the clipped step, zero_grad) captured in a CUDA graph:
    its replays leave the parameters, momentum, norm, losses and meters of the same loop run eagerly, bitwise"""
    from ssn_b200.meters import StepMeters
    dev = _cuda()
    batches = [tuple(t.to(dev) for t in B.synth_binary_batch(2, 4, 2, 3, seed=s)) for s in (41, 42, 43)]
    iter_size, max_norm = 3, 1e-3

    def make():
        m = _binary("exact_tc", dropout=0)
        opt = _opt(m)
        meters = StepMeters("binary", dev)

        def micro(j):
            return m.fused_step(*batches[j], meters=meters)

        def period():
            losses = [micro(j) for j in range(iter_size)]
            norm = opt.step(grad_mult=1.0 / iter_size, max_norm=max_norm)
            opt.zero_grad()
            return losses, norm
        # the reference's first step: micro-batch 0 alone
        opt.zero_grad()
        micro(0)
        opt.step(grad_mult=1.0 / iter_size, max_norm=max_norm)
        opt.zero_grad()
        return opt, meters, period
    o1, me1, period1 = make()
    o2, me2, period2 = make()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        period2()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_losses, static_norm = period2()
    for _ in range(2):
        graph.replay()
    for _ in range(3):
        losses, norm = period1()
    torch.cuda.synchronize()
    assert float(norm) > max_norm, "the test must clip"
    assert torch.equal(norm, static_norm) and all(torch.equal(a, b) for a, b in zip(losses, static_losses))
    assert torch.equal(o1.flat_param, o2.flat_param) and torch.equal(o1.flat_mom, o2.flat_mom)
    assert torch.equal(o1.flat_grad, o2.flat_grad) and float(o1.flat_grad.abs().sum()) == 0
    assert torch.equal(me1.buf, me2.buf) and float(me1.buf[0, 1]) == (1 + 3 * iter_size) * 2


# ---- 3. the golden replay ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "train_loop.npz"))


@pytest.mark.parametrize("tag", ["ssn", "binary"])
@pytest.mark.parametrize("case", range(5))
def test_reference_update_blocks_on_device(gold, tag, case):
    """the reference's update block (p.grad /= iter_size, clip_grad_norm over the groups and an extra gradient,
    optimizer.step()) through FusedSGD + extra_grads: total_norm and the parameters within 1e-6; the gradients the step
    sees and the clipped extra bitwise clipped_grad at the device's own norm, and within 2 ulp of the reference where no
    clip applies (the device forms c from its fp32 norm, which moves it by up to 1 ulp: 3 ulp with a clip)"""
    from ssn_b200.optim import FusedSGD
    dev = _cuda()
    p = "%s_upd%d_" % (tag, case)
    iter_size, clip = gold[p + "cfg"]
    clip = None if np.isnan(clip) else float(clip)
    params = [torch.nn.Parameter(torch.from_numpy(gold[p + "param%d" % j]).to(dev)) for j in range(4)]
    policies = [{"params": params[:2], "lr_mult": 1, "decay_mult": 1}, {"params": params[2:3], "lr_mult": 2, "decay_mult": 0}]
    opt = FusedSGD(policies, lr=0.1, momentum=0.9, weight_decay=5e-4)
    assert opt.ungrouped(params) == [params[3]]
    grads = [torch.from_numpy(gold[p + "grad%d" % j]).to(dev) for j in range(3)]
    for q, gr in zip(params[:3], grads):
        q.grad.copy_(gr)
    extra = torch.from_numpy(gold[p + "grad3"]).to(dev)
    gm = 1.0 / float(iter_size)
    # without a clip the reference's norm is 0 and nothing is clipped: max_norm = inf writes back the divided gradients
    norm = float(opt.step(grad_mult=gm, max_norm=float("inf") if clip is None else clip, extra_grads=[extra]))
    flat_g = np.concatenate([gold[p + "grad%d" % j].reshape(-1) for j in range(3)])
    c = None
    if clip is not None:
        assert abs(norm - gold[p + "total_norm"]) <= 1e-6 * gold[p + "total_norm"], (norm, gold[p + "total_norm"])
        c = TL.clip_coef(norm, clip)
        assert c is not None or clip >= norm
    seen = opt.flat_grad.cpu().numpy()
    assert seen.tobytes() == TL.clipped_grad(flat_g, gm, c).tobytes()
    assert extra.cpu().numpy().tobytes() == TL.clipped_grad(gold[p + "grad3"], 1.0, c).tobytes()
    want_seen = np.concatenate([gold[p + "seen%d" % j].reshape(-1) for j in range(3)])
    bar = 2 if c is None else 3
    assert _ulps(seen, want_seen).max() <= bar and _ulps(extra.cpu().numpy(), gold[p + "extra_after"]).max() <= bar
    for j in range(3):
        want = gold[p + "param_after%d" % j]
        got = params[j].detach().cpu().numpy()
        assert np.abs(got.astype(np.float64) - want).max() <= 1e-6 * np.abs(want).max(), j
    assert params[3].detach().cpu().numpy().tobytes() == gold[p + "param3"].tobytes()      # no group: not stepped


@pytest.mark.parametrize("tag", ["ssn", "binary"])
def test_reference_accuracy_batches_through_step_meters(gold, tag):
    from ssn_b200.meters import StepMeters
    dev = _cuda()
    meters = StepMeters(tag, dev)
    n_losses = 4 if tag == "ssn" else 1
    for step in range(3):
        q = "%s_acc%d_" % (tag, step)
        scores = torch.from_numpy(gold[q + "scores"]).to(dev)
        target = torch.from_numpy(gold[q + "target"]).to(dev)
        before = meters.buf.cpu().numpy()[n_losses:].copy()
        meters._update(torch.zeros(n_losses, device=dev), scores, target, None, 1.0)
        now = meters.buf.cpu().numpy()[n_losses:]
        vals = np.array([(now[k, 0] - before[k, 0]) / (now[k, 1] - before[k, 1]) for k in range(3)], np.float32)
        assert vals.tobytes() == gold[q + "vals"].tobytes()
    assert meters.buf.cpu().numpy()[n_losses:].tobytes() == gold[tag + "_meters"].tobytes()


# ---- 4. kernel sweeps ----------------------------------------------------------------------------------------------------
def _meter_scores(rows, cols, rng):
    """rows of seven kinds in turn: continuous; quantised with the maximum tied in columns c, c + 32 and c + 64 (three
    lanes of the kernel's warp); one NaN; several NaNs; +inf and -inf; -0 against +0 as the maximum; all -inf"""
    s = rng.standard_normal((rows, cols)).astype(np.float32)
    kind = np.arange(rows) % 7
    for r in np.flatnonzero(kind == 1):
        s[r] = np.round(s[r] * 2) / 2
        c = int(rng.integers(0, min(cols, 32)))
        s[r, c::32][:3] = s[r].max() + 1
    for r in np.flatnonzero(kind == 2):
        s[r, rng.integers(0, cols)] = np.nan
    for r in np.flatnonzero(kind == 3):
        s[r, rng.choice(cols, min(cols, 3), replace=False)] = np.nan
    for r in np.flatnonzero(kind == 4):
        idx = rng.choice(cols, min(cols, 4), replace=False)
        s[r, idx] = np.where(np.arange(len(idx)) % 2 == 0, np.inf, -np.inf)
    for r in np.flatnonzero(kind == 5):
        s[r] = -np.abs(s[r]) - 1
        idx = rng.choice(cols, min(cols, 2), replace=False)
        s[r, idx] = [-0.0, 0.0][:len(idx)] if r % 2 else [0.0, -0.0][:len(idx)]
    s[kind == 6] = -np.inf
    return s


METER_SHAPES = [(r, c) for r in (2, 8, 256, 258, 4096) for c in (1, 2, 21, 31, 32, 33, 64, 201, 1000)] + \
               [(65536, 2), (65536, 201)]


@pytest.mark.parametrize("rows,cols", METER_SHAPES)
def test_train_meters_sweep(rows, cols):
    """5 accumulated ssnb_train_meters calls against meters_update, bitwise; prop_type NULL, or random types with type-1
    rows interleaved (odd activity counts included); targets hit, miss and out of range; 0 ... 8 losses"""
    from ssn_b200._lib import lib, check
    dev = _cuda()
    case = METER_SHAPES.index((rows, cols))
    rng = np.random.default_rng(1000 + case)
    n_losses = case % 9
    with_types = case % 2 == 1 or rows == 65536 and cols == 201
    buf = torch.zeros(n_losses + 3, 2, dtype=torch.float64, device=dev)
    want = np.zeros((n_losses + 3, 2))
    secs = 0.0
    for step in range(5):
        s = _meter_scores(rows, cols, rng)
        t = rng.integers(0, cols, rows)
        hit = rng.random(rows) < 0.5
        t[hit] = TL.top1(s)[hit]
        t[rng.random(rows) < 0.05] = -1
        t[rng.random(rows) < 0.05] = cols
        pt = rng.choice([0, 1, 2], rows, p=[0.35, 0.3, 0.35]) if with_types else None
        losses = rng.standard_normal(max(n_losses, 1)).astype(np.float32)
        loss_n = float(rng.choice([1, 2, 3, 64]))
        ds, dt, dl = torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev), torch.from_numpy(losses).to(dev)
        dp = None if pt is None else torch.from_numpy(pt).to(dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(lib.ssnb_train_meters(ds.data_ptr(), rows, cols, dt.data_ptr(), None if dp is None else dp.data_ptr(),
                                    dl.data_ptr(), n_losses, loss_n, buf.data_ptr(), _stream()), None, "train_meters")
        torch.cuda.synchronize()
        secs += time.perf_counter() - t0
        TL.meters_update(want, s, t, pt, losses[:n_losses], loss_n)
        assert buf.cpu().numpy().tobytes() == want.tobytes(), (step, buf.cpu().numpy(), want)
    if rows == 65536:
        print("train_meters %d x %d (prop_type %s): %.1f ms per call" % (rows, cols, with_types, secs / 5 * 1e3))


def test_train_meters_odd_activity_rows():
    """an odd count of activity rows: the last one counts in act_acc only; fg and bg cover the pairs before it"""
    from ssn_b200.meters import StepMeters
    dev = _cuda()
    m = StepMeters("ssn", dev)
    pt = torch.tensor([0, 1, 2, 1, 1, 0, 2, 1, 0], device=dev)
    tg = torch.tensor([0, 9, 0, 9, 9, 1, 1, 9, 0], device=dev)
    m.update_ssn(torch.zeros(4, device=dev), torch.zeros(9, 2, device=dev), tg, pt, 1)
    want = TL.meters_update(np.zeros((7, 2)), np.zeros((9, 2), np.float32), tg.cpu().numpy(), pt.cpu().numpy(), np.zeros(4), 1.0)
    assert m.buf.cpu().numpy().tobytes() == want.tobytes()
    assert want[5].tolist() == [100.0, 2.0] and want[6].tolist() == [100.0, 2.0]     # never above 100 %
    b = StepMeters("binary", dev)
    b.update_binary(torch.zeros(1, device=dev), torch.zeros(1, 2, device=dev), torch.zeros(1, dtype=torch.int64, device=dev), 1)
    assert b.buf.cpu().tolist()[1:] == [[100.0, 1.0], [0.0, 0.0], [0.0, 0.0]]


def _norm_call(g_ptr, n, gm, extras, partials, out):
    from ssn_b200._lib import lib, check
    ex = _extras(extras)
    check(lib.ssnb_grad_norm(g_ptr, n, gm, C.byref(ex), partials.data_ptr(), out.data_ptr(), _stream()), None, "grad_norm")


def _norm_ok(got, want):
    if want > FLT_MAX:
        return got == float("inf")
    if want == 0:
        return got == 0
    return _ulps(got, want) <= 1


@pytest.mark.parametrize("n", [0, 1, 3, 5, 512 * 256 * 4 - 1, 512 * 256 * 4 + 1, SSN_FLAT])
def test_grad_norm_sweep(n):
    """the flat pointer 0 ... 3 floats into a buffer (16-byte aligned: float4 body + scalar tail; else the scalar path),
    grad_mult 1 and 1/3, 0 ... 8 extras of sizes 0, 1, 7 and n + 13, magnitudes 1, 1e-30 and 1e19: within 1 fp32 ulp of
    the float64 norm"""
    from ssn_b200._lib import GRAD_NORM_CTAS
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(n)
    base = torch.randn(n + 4, generator=gen, device=dev)
    partials = torch.empty(GRAD_NORM_CTAS, dtype=torch.float64, device=dev)
    out = torch.empty((), device=dev)
    worst, calls = 0.0, 0
    for scale in (1.0, 1e-30, 1e19):
        buf = base * scale
        host = buf.cpu().numpy()
        for off in range(4):
            for gm in (1.0, 1.0 / 3):
                k = (calls + n) % 9
                extras = [torch.randn((0, 1, 7, n + 13)[j % 4], generator=gen, device=dev) * scale for j in range(k)]
                _norm_call(buf.data_ptr() + 4 * off, n, gm, extras, partials, out)
                got = float(out)
                want = TL.grad_norm64(host[off:off + n], gm, [e.cpu().numpy() for e in extras])
                assert _norm_ok(got, want), (scale, off, gm, k, got, want)
                if want:
                    worst = max(worst, float(_ulps(got, want)))
                calls += 1
    print("grad_norm n=%d: worst %.2f ulp over %d calls" % (n, worst, calls))


def test_grad_norm_non_finite_and_overflow():
    from ssn_b200._lib import GRAD_NORM_CTAS
    dev = _cuda()
    partials = torch.empty(GRAD_NORM_CTAS, dtype=torch.float64, device=dev)
    out = torch.empty((), device=dev)
    n = 1031                                                       # 257 float4s and a 3-element tail
    for where in ("body", "tail", "extra"):
        for bad in (float("nan"), float("inf"), -float("inf")):
            for off in (0, 1):
                g = torch.ones(n + 4, device=dev)
                e = torch.ones(7, device=dev)
                if where == "extra":
                    e[3] = bad
                else:
                    g[off + (5 if where == "body" else n - 1)] = bad
                _norm_call(g.data_ptr() + 4 * off, n, 1.0, [e], partials, out)
                got = float(out)
                assert (np.isnan(got) if np.isnan(bad) else got == float("inf")), (where, bad, off, got)
    big = torch.full((9,), 3e38, device=dev)                         # finite elements, a norm above FLT_MAX
    _norm_call(big.data_ptr(), 9, 1.0, [], partials, out)
    assert float(out) == float("inf")
    _norm_call(big.data_ptr(), 1, 1.0, [], partials, out)
    assert float(out) == np.float32(3e38)


def test_grad_norm_bitwise_repeatable():
    """calls, a second stream and graph replays at a fixed pointer give one value, aligned and not"""
    from ssn_b200._lib import GRAD_NORM_CTAS
    dev = _cuda()
    g = torch.randn(SSN_FLAT + 1, generator=torch.Generator(device=dev).manual_seed(3), device=dev) * 1e-3
    e = torch.randn(4097, device=dev)
    partials = torch.empty(GRAD_NORM_CTAS, dtype=torch.float64, device=dev)
    out = torch.empty((), device=dev)
    for off in (0, 1):
        vals = []
        for _ in range(3):
            _norm_call(g.data_ptr() + 4 * off, SSN_FLAT, 1.0 / 3, [e], partials, out)
            vals.append(out.clone())
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            _norm_call(g.data_ptr() + 4 * off, SSN_FLAT, 1.0 / 3, [e], partials, out)
            vals.append(out.clone())
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            _norm_call(g.data_ptr() + 4 * off, SSN_FLAT, 1.0 / 3, [e], partials, out)
        for _ in range(2):
            out.zero_()
            graph.replay()
            vals.append(out.clone())
        torch.cuda.synchronize()
        assert all(torch.equal(vals[0], v) for v in vals[1:]), (off, vals)


@pytest.mark.parametrize("norm,max_norm", [(2.0, 1.0), (1.5, 1.5), (3e10, 3e10), (5.0, 0.0), (float("nan"), 1.0),
                                           (float("inf"), 1.0), (0.5, 1.0), (0.0, 0.0)])
def test_grad_clip_sweep(norm, max_norm):
    """ssnb_grad_clip over SSN's flat size (about 20 passes of its 2048-CTA grid) and extras of sizes 0, 7 and n + 1000:
    every element g * fp32(c) bitwise where c = max_norm / (norm + 1e-6) < 1, else untouched (norm == max_norm: c just
    under 1, or 1 at 3e10; max_norm 0 and an inf norm: c = 0; a NaN norm: no clip)"""
    from ssn_b200._lib import lib, check
    dev = _cuda()
    n = SSN_FLAT
    gen = torch.Generator(device=dev).manual_seed(5)
    g = torch.randn(n, generator=gen, device=dev)
    g[17], g[n - 2] = float("inf"), float("nan")
    extras = [torch.randn(k, generator=gen, device=dev) for k in (0, 7, n + 1000)]
    host_g, host_e = g.cpu().numpy(), [e.cpu().numpy() for e in extras]
    dnorm = torch.tensor(norm, dtype=torch.float32, device=dev)
    ex = _extras(extras)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    check(lib.ssnb_grad_clip(dnorm.data_ptr(), max_norm, g.data_ptr(), n, C.byref(ex), _stream()), None, "grad_clip")
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    c = TL.clip_coef(np.float32(norm), max_norm)
    assert (c is None) == (norm != norm or (norm, max_norm) in ((3e10, 3e10), (0.5, 1.0)))
    want = host_g if c is None else TL.clipped_grad(host_g, 1.0, c)
    assert _bits_equal(g.cpu().numpy(), want)
    for e, h in zip(extras, host_e):
        assert _bits_equal(e.cpu().numpy(), h if c is None else TL.clipped_grad(h, 1.0, c))
    print("grad_clip n=%d (+%d extra) c=%s: %.2f ms" % (n, n + 1007, c, ms))


def _segments(rng):
    """512 segments whose ends land on, just before and just after multiples of 256, with empty and one-element ones"""
    sizes = rng.choice([0, 1, 2, 255, 256, 257, 511], 512)
    sizes[0], sizes[-1], sizes[100:104] = 0, 0, [1, 0, 0, 1]
    sizes[1:7] = [255, 0, 1, 255, 1, 1]                 # ends 255, 255, 256, 511, 512, 513
    ends = np.cumsum(sizes)
    assert {0, 1, 255} <= set((ends % 256).tolist())
    return ends


@pytest.mark.parametrize("write_back", [0, 1])
def test_sgd_step_groups_clipped_sweep(write_back):
    """ssnb_grad_norm -> ssnb_sgd_step_groups_clipped over 512 segments with random lr / wd: parameters and momentum within
    1e-6 of float64 (of the magnitude of the terms each is formed from), written-back gradients bitwise g * fl(gm * fl(c)),
    extras clipped only with write_back; an unclipped call (c >= 1, or a NaN norm) bitwise the plain kernel"""
    from ssn_b200._lib import lib, check, GRAD_NORM_CTAS
    dev = _cuda()
    rng = np.random.default_rng(7 + write_back)
    ends = _segments(rng)
    n = int(ends[-1])
    seg_lr = rng.uniform(1e-3, 1e-1, 512).astype(np.float32)
    seg_wd = np.where(rng.random(512) < 0.3, 0, rng.uniform(0, 1e-3, 512)).astype(np.float32)
    p0 = rng.standard_normal(n).astype(np.float32)
    g0 = (rng.standard_normal(n) * 0.3).astype(np.float32)
    b0 = (rng.standard_normal(n) * 0.1).astype(np.float32)
    e0 = [rng.standard_normal(k).astype(np.float32) for k in (7, 1000)]
    d_end, d_lr, d_wd = (torch.from_numpy(a).to(dev) for a in (ends.astype(np.int64), seg_lr, seg_wd))
    gm = 1.0 / 3
    partials = torch.empty(GRAD_NORM_CTAS, dtype=torch.float64, device=dev)
    out = torch.empty((), device=dev)

    def run(clipped, max_norm, norm=None):
        p, g, b = (torch.from_numpy(a.copy()).to(dev) for a in (p0, g0, b0))
        ex_t = [torch.from_numpy(a.copy()).to(dev) for a in e0]
        if not clipped:
            check(lib.ssnb_sgd_step_groups(p.data_ptr(), g.data_ptr(), b.data_ptr(), n, d_end.data_ptr(), d_lr.data_ptr(),
                                           d_wd.data_ptr(), 512, 0.9, gm, _stream()), None, "sgd_step_groups")
        else:
            if norm is None:
                _norm_call(g.data_ptr(), n, gm, ex_t, partials, out)
            else:
                out.fill_(norm)
            ex = _extras(ex_t)
            check(lib.ssnb_sgd_step_groups_clipped(p.data_ptr(), g.data_ptr(), b.data_ptr(), n, d_end.data_ptr(), d_lr.data_ptr(),
                                                   d_wd.data_ptr(), 512, 0.9, gm, out.data_ptr(), max_norm, write_back, C.byref(ex),
                                                   _stream()), None, "sgd_step_groups_clipped")
        return [t.cpu().numpy() for t in (p, g, b)] + [[e.cpu().numpy() for e in ex_t], float(out)]

    # clipped: the norm the kernel before wrote, then the step
    norm64 = TL.grad_norm64(g0, gm, e0)
    p, g, b, ex, norm = run(True, float(np.float32(norm64 / 4)))
    assert _ulps(norm, norm64) <= 1
    c = TL.clip_coef(norm, np.float32(norm64 / 4))
    assert c is not None and c < 0.3
    wp, wb, ps, bs = TL.sgd64(p0, g0, b0, ends, seg_lr, seg_wd, 0.9, gm, c)
    perr = float((np.abs(p - wp) / ps).max())
    berr = float((np.abs(b - wb) / bs).max())
    assert perr <= 1e-6 and berr <= 1e-6, (perr, berr)
    assert g.tobytes() == (TL.clipped_grad(g0, gm, c) if write_back else g0).tobytes()
    for got, e in zip(ex, e0):
        assert got.tobytes() == (TL.clipped_grad(e, 1.0, c) if write_back else e).tobytes()
    print("sgd_step_groups_clipped n=%d write_back=%d: param %.2e momentum %.2e" % (n, write_back, perr, berr))
    # unclipped: bitwise the plain kernel
    plain = run(False, None)
    for norm_v, max_norm in ((0.5, 1.0), (float("nan"), 1.0), (1e30, float("inf"))):
        p, g, b, ex, _ = run(True, max_norm, norm_v)
        assert p.tobytes() == plain[0].tobytes() and b.tobytes() == plain[2].tobytes(), norm_v
        assert g.tobytes() == (g0 * np.float32(gm) if write_back else g0).tobytes()
        assert all(a.tobytes() == e.tobytes() for a, e in zip(ex, e0))
    assert plain[1].tobytes() == g0.tobytes()
    # the 512-segment cap
    q = out.data_ptr()
    assert lib.ssnb_sgd_step_groups_clipped(q, q, q, 1, d_end.data_ptr(), q, q, 513, 0.9, gm, q, 1.0, write_back, None, None) == 1
