"""The rest of the training step on the device (ssn_train.py:213-250, binary_train.py:170-197) and validate()'s forward:
the gradient norm of clip_grad_norm against float64 torch over the real parameter sets, the clipped FusedSGD step against
clip_grad_norm_ + torch.optim.SGD, the meters against the reference's accuracy(), a graph-replayed loop with clip and meters
against the same loop run eagerly, and fused_eval against the module path.  Run on an H100: pytest -m gpu."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import binary_oracle as B
from oracle import synth
from oracle import train_loop_oracle as TL

_BB = {}


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _bb():
    if "rgb" not in _BB:
        _BB["rgb"] = synth.synth_backbone(3, seed=0, calib_frames=2)
    return _BB["rgb"]


def _ssn(K, bn_mode="frozen", dropout=0):
    import ssn_models
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=dropout, bn_mode=bn_mode)
    sd = m.state_dict()
    for k, v in _bb().items():
        sd["base_model." + k].copy_(v)
    m = m.to(_cuda()).train()
    from ssn_b200 import _lib
    m.set_precision(_lib.EXACT_TC, 1024.0)
    return m


def _binary(K=2, dropout=0):
    import binary_model
    m = binary_model.BinaryClassifier(K, 5, "RGB", base_model="BNInception", dropout=dropout)
    sd = m.state_dict()
    for k, v in _bb().items():
        sd["base_model." + k].copy_(v)
    for k, v in B.synth_classifier(K, seed=0).items():
        sd[k].copy_(v)
    m = m.to(_cuda()).train()
    from ssn_b200 import _lib
    m.set_precision(_lib.EXACT_TC, 1024.0)
    return m


def _opt(m, lr=1e-3):
    from ssn_b200.optim import FusedSGD
    order = [p for p in m.parameters() if p.requires_grad]
    return FusedSGD(m.get_optim_policies(), lr=lr, momentum=0.9, weight_decay=5e-4, order=order,
                    on_step=[m.base_model.invalidate_packed])


def _torch_norm(tensors):
    return float(torch.nn.utils.get_total_norm([t.double() for t in tensors]))


# ---- norm ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["ssn20", "ssn200", "binary", "ssn20_partial"])
def test_grad_norm_vs_float64(model):
    from ssn_b200.optim import clip_grad_norm
    m = {"ssn20": lambda: _ssn(20), "ssn200": lambda: _ssn(200), "binary": _binary,
         "ssn20_partial": lambda: _ssn(20, bn_mode="partial")}[model]()
    opt = _opt(m)
    extra_p = opt.ungrouped(m.parameters())
    assert len(extra_p) == (2 if model.endswith("partial") else 0)
    g = torch.Generator(device=opt.device).manual_seed(1)
    opt.flat_grad.copy_(torch.randn(opt.n, generator=g, device=opt.device) * 1e-3)
    extra = [torch.randn(p.shape, generator=g, device=opt.device) for p in extra_p]
    for p, e in zip(extra_p, extra):
        p.grad = e
    want = _torch_norm([p.grad for p in m.parameters() if p.grad is not None])
    norms = [clip_grad_norm(opt, float("inf"), extra).clone() for _ in range(3)]
    assert all(torch.equal(norms[0], n) for n in norms[1:]), "not bitwise repeatable"
    assert abs(float(norms[0]) - want) <= 1e-6 * want, (float(norms[0]), want)
    # the iter_size division applies to the groups only, as in the reference
    from ssn_b200.optim import _extra_grads
    opt._grad_norm(1.0 / 3, _extra_grads(extra, opt.device))
    want3 = _torch_norm([opt.flat_grad / 3] + extra)
    assert abs(float(opt.norm) - want3) <= 1e-6 * want3
    # zero, NaN and inf gradients
    opt.flat_grad.zero_()
    for e in extra:
        e.zero_()
    assert float(clip_grad_norm(opt, 1.0, extra)) == 0.0
    opt.flat_grad[opt.n // 2] = float("nan")
    assert torch.isnan(clip_grad_norm(opt, 1.0, extra))
    opt.flat_grad.zero_()
    opt.flat_grad[7] = float("inf")
    assert torch.isinf(clip_grad_norm(opt, 1.0, extra))


# ---- step ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ratio", [0.5, 1.0, 2.0])
def test_clipped_step_vs_torch(ratio):
    """FusedSGD.step(grad_mult=1/iter_size, max_norm) against p.grad /= iter_size, clip_grad_norm_ and torch.optim.SGD, two
    steps; max_norm below (0.5), at (1.0) and above (2.0) the first step's norm"""
    dev = _cuda()
    m1, m2 = _binary(), _binary()
    lr, wd, mom, iter_size = 0.01, 5e-4, 0.9, 3
    groups = [{"params": g["params"], "lr": lr * g["lr_mult"], "weight_decay": wd * g["decay_mult"]}
              for g in m1.get_optim_policies() if g["params"]]
    ref = torch.optim.SGD(groups, lr=lr, momentum=mom)
    from ssn_b200.optim import FusedSGD
    opt = FusedSGD(m2.get_optim_policies(), lr=lr, momentum=mom, weight_decay=wd)
    p1 = [p for g in groups for p in g["params"]]
    p2 = [p for g in opt.param_groups for p in g["params"]]
    g = torch.Generator().manual_seed(4)
    max_norm = None
    for step in range(2):
        for a, b in zip(p1, p2):
            gr = (torch.randn(a.shape, generator=g) * 1e-2).to(dev)
            a.grad = gr.clone()
            b.grad.copy_(gr)
        for a in p1:
            a.grad /= iter_size
        if max_norm is None:
            max_norm = ratio * _torch_norm([a.grad for a in p1])
        tn = torch.nn.utils.clip_grad_norm_(p1, max_norm)
        ref.step()
        norm = opt.step(grad_mult=1.0 / iter_size, max_norm=max_norm)
        assert abs(float(norm) - float(tn)) <= 1e-6 * float(tn)
        worst = max(float((b.detach().double() - a.detach().double()).norm() / a.detach().double().norm()) for a, b in zip(p1, p2))
        assert worst < 1e-6, (step, worst)
        gw = max(float((b.grad.double() - a.grad.double()).norm() / a.grad.double().norm()) for a, b in zip(p1, p2))
        assert gw < 1e-6, ("written-back gradient", step, gw)
    # no clipping: bitwise the plain step
    m3, m4 = _binary(), _binary()
    o3 = FusedSGD(m3.get_optim_policies(), lr=lr, momentum=mom, weight_decay=wd)
    o4 = FusedSGD(m4.get_optim_policies(), lr=lr, momentum=mom, weight_decay=wd)
    gr = torch.randn(o3.n, generator=g).to(dev)
    for _ in range(2):
        o3.flat_grad.copy_(gr)
        o4.flat_grad.copy_(gr)
        assert o3.step(grad_mult=0.25) is None
        o4.step(grad_mult=0.25, max_norm=1e30)
    assert torch.equal(o3.flat_param, o4.flat_param) and torch.equal(o3.flat_mom, o4.flat_mom)


# ---- meters --------------------------------------------------------------------------------------------------------------
def test_meters_vs_reference_accuracy():
    dev = _cuda()
    from ssn_b200.meters import StepMeters
    g = torch.Generator().manual_seed(5)
    K, videos = 20, 6
    n = videos * 8
    prop_type = torch.tensor([0, 1, 1, 1, 1, 1, 1, 2]).repeat(videos)
    want = TL.new_meters(TL.SSN_METERS)
    meters = StepMeters("ssn", dev)
    for step in range(3):
        raw_act = torch.randn(n, K + 1, generator=g)         # continuous: tie-free
        target = torch.randint(0, K + 1, (n,), generator=g)
        target[::3] = raw_act[::3].argmax(1)                   # plenty of hits
        losses = torch.rand(4, generator=g)
        meters.update_ssn(losses.to(dev), raw_act.to(dev), target.to(dev), prop_type.to(dev), videos)
        TL.update_ssn_meters(want, losses, raw_act, target, prop_type, videos)
    got = meters.buf.cpu()
    ref = torch.tensor([want[k] for k in TL.SSN_METERS], dtype=torch.float64)
    assert torch.equal(got, ref), (got, ref)
    r = meters.read()
    assert r["act_acc"] == want["act_acc"][0] / want["act_acc"][1]
    meters.reset()
    assert meters.buf.abs().sum() == 0
    # ties: every score equal -> class 0, the lowest index: 4 of 8 rows, 3 of the 4 fg rows, 1 of the 4 bg rows
    bm = StepMeters("binary", dev)
    scores = torch.zeros(8, 2, device=dev)
    target = torch.tensor([0, 1, 0, 1, 1, 0, 0, 1], device=dev)
    bm.update_binary(torch.ones(1, device=dev), scores, target, 4)
    r = bm.read()
    assert (r["act_acc"], r["fg_acc"], r["bg_acc"]) == (50.0, 75.0, 25.0), r
    assert (bm.buf[1:, 1].cpu() == torch.tensor([8.0, 4.0, 4.0], dtype=torch.float64)).all()


# ---- graph replay --------------------------------------------------------------------------------------------------------
def test_graph_replay_with_clip_and_meters_equals_eager():
    dev = _cuda()
    from ssn_b200.meters import StepMeters
    x, target = (t.to(dev) for t in B.synth_binary_batch(2, 4, 2, 3, seed=3))

    def make():
        m = _binary()
        opt = _opt(m)
        meters = StepMeters("binary", dev)

        def step():
            opt.flat_grad.zero_()
            loss = m.fused_step(x, target, meters=meters)
            norm = opt.step(grad_mult=0.5, max_norm=1e-3)
            return loss, norm
        return opt, meters, step
    opt1, me1, step1 = make()
    opt2, me2, step2 = make()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step2()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss, static_norm = step2()
    for _ in range(4):
        graph.replay()
    for _ in range(7):
        l1, n1 = step1()
    torch.cuda.synchronize()
    assert torch.equal(l1, static_loss) and torch.equal(n1, static_norm)
    assert float(n1) > 1e-3, "the test must clip"
    assert torch.equal(opt1.flat_param, opt2.flat_param) and torch.equal(opt1.flat_mom, opt2.flat_mom)
    assert torch.equal(me1.buf, me2.buf) and float(me1.buf[0, 1]) == 7 * 2


# ---- fused_eval ----------------------------------------------------------------------------------------------------------
def test_ssn_fused_eval_vs_module_path():
    dev = _cuda()
    from ops.ssn_ops import ClassWiseRegressionLoss, CompletenessLoss
    from ssn_b200.meters import StepMeters
    m = _ssn(20, bn_mode="partial", dropout=0.8)
    x, sc, tg, rt, pt = (t.to(dev) for t in synth.synth_batch(2, 20, seed=7))
    for p in m.parameters():
        if p.requires_grad:
            p.grad = torch.full_like(p, 0.5)
    bn1 = m.base_model.conv1_7x7_s2_bn
    stats = (bn1.running_mean.clone(), bn1.running_var.clone())
    other = StepMeters("ssn", dev)
    other.buf.fill_(3.0)
    m.eval()
    meters = StepMeters("ssn", dev)
    losses = m.fused_eval(x, sc, tg, rt, pt, meters=meters)
    with torch.no_grad():
        a, at, c, ct, r, rl, rtg = m(x, sc, tg, rt, pt)
        act = torch.nn.CrossEntropyLoss()(a, at)
        comp = CompletenessLoss()(c, ct, 1, 7)
        reg = ClassWiseRegressionLoss()(r, rl, rtg)
        want = torch.stack([v.reshape(()) for v in (act, comp, reg, act + 0.1 * comp + 0.1 * reg)]).cpu()
    err = ((losses.cpu().double() - want.double()).abs() / want.double().abs()).max()
    assert err < 1e-4, (losses, want)
    assert all(torch.equal(p.grad, torch.full_like(p, 0.5)) for p in m.parameters() if p.requires_grad)
    assert torch.equal(bn1.running_mean, stats[0]) and torch.equal(bn1.running_var, stats[1])
    assert (other.buf == 3.0).all() and float(meters.buf[3, 1]) == 2
    with pytest.raises(RuntimeError):
        m.train()
        m.fused_eval(x, sc, tg, rt, pt)


def test_binary_fused_eval_vs_module_path_and_fused_step():
    dev = _cuda()
    from ssn_b200.meters import StepMeters
    m = _binary(dropout=0.8)
    x, target = (t.to(dev) for t in B.synth_binary_batch(2, 4, 2, 3, seed=8))
    m.eval()
    meters = StepMeters("binary", dev)
    loss = m.fused_eval(x, target, meters=meters)
    with torch.no_grad():
        raw, tgt = m(x, target)
        want = torch.nn.CrossEntropyLoss()(raw, tgt)
    assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want))
    assert (m.last_eval["logits"] - raw).abs().max() <= 1e-5 * raw.abs().max()
    for p in m.parameters():
        assert p.grad is None
    step_loss = m.fused_step(x, target)                       # eval(): no dropout, the same forward half
    assert abs(float(step_loss) - float(loss)) <= 1e-5 * abs(float(loss))
    r = meters.read()
    assert set(r) == {"loss", "act_acc", "fg_acc", "bg_acc"} and r["loss"] == float(loss)
