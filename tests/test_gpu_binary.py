"""BinaryClassifier (TAG actionness) on the GPU: the classifier + cross-entropy kernel against float64 torch, course-only
pooling, the module path, fused_step (eager and CUDA-graph replayed), test mode, bn_mode='partial' and GradSync coverage,
against the CPU oracle (oracle/binary_oracle.py).  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import binary_oracle as B
from oracle import ssn_oracle as O
from oracle import synth

E2E_TOL = {"exact": 1e-4, "exact_tc": 5e-4}       # the whole-network bars of test_gpu_parity
_BB = {}


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _max_rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _prec(name):
    from ssn_b200 import _lib
    return {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[name]


def _backbone(C_):
    if C_ not in _BB:
        _BB[C_] = synth.synth_backbone(C_, seed=0, calib_frames=2)
    return _BB[C_]


def _model(K, modality, precision="exact_tc", dropout=0, bn_mode="frozen"):
    import binary_model
    C_ = 3 if modality == "RGB" else 10
    m = binary_model.BinaryClassifier(K, 5, modality, base_model="BNInception", dropout=dropout, bn_mode=bn_mode)
    sd = m.state_dict()
    for k, v in _backbone(C_).items():
        sd["base_model." + k].copy_(v)
    for k, v in B.synth_classifier(K, seed=0).items():
        sd[k].copy_(v)
    m = m.to(_cuda()).train()
    m.set_precision(_prec(precision), 4096.0 if precision == "fast" else 1024.0)
    return m


def _oracle(C_, K, x, target, mask=None, bn_train_first=False):
    """oracle forward + CrossEntropyLoss + backward: (scores, loss, {parameter name: gradient}, backbone params, taps)"""
    bbo = {k: v.clone() for k, v in _backbone(C_).items()}
    hdo = B.synth_classifier(K, seed=0)
    for d in (bbo, hdo):
        for k in d:
            if "_bn." not in k or (bn_train_first and k in ("conv1_7x7_s2_bn.weight", "conv1_7x7_s2_bn.bias")):
                d[k].requires_grad_(True)
    taps = {}
    raw, tgt = B.binary_train_forward(bbo, hdo, x, target, in_channels=C_, mask=mask, taps=taps, bn_train_first=bn_train_first)
    loss = B.cross_entropy(raw, tgt)
    loss.backward()
    grads = {"base_model." + k: v.grad for k, v in bbo.items() if v.grad is not None}
    grads.update({k: v.grad for k, v in hdo.items()})
    return raw.detach(), loss.item(), grads, bbo, taps


def _agg_rel(params, ref):
    num = sum(float((params[n].grad.double().cpu() - r.double()).pow(2).sum()) for n, r in ref.items())
    return (num / sum(float(r.double().pow(2).sum()) for r in ref.values())) ** 0.5


def _cos(params, ref):
    dot = na = nb = 0.0
    for n, r in ref.items():
        a, b = params[n].grad.double().cpu().flatten(), r.double().flatten()
        dot += float(a @ b); na += float(a @ a); nb += float(b @ b)
    return dot / (na * nb) ** 0.5


# ---- 1. classifier + cross-entropy kernel -------------------------------------------------------------------------------
def _ce(x, w, b, t, loss_scale=1.0):
    from ssn_b200._lib import lib, check
    n, D = x.shape
    K = w.shape[0]
    out = dict(logits=torch.empty(n, K, device=x.device), loss=torch.empty(1, device=x.device), dx=torch.empty_like(x),
               dw=torch.empty_like(w), db=torch.empty_like(b))
    ws = torch.empty(lib.ssnb_classifier_ce_workspace_bytes(n, K), dtype=torch.uint8, device=x.device)
    check(lib.ssnb_classifier_ce_fwd_bwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), t.data_ptr(), n, D, K, loss_scale,
                                         out["logits"].data_ptr(), out["loss"].data_ptr(), out["dx"].data_ptr(),
                                         out["dw"].data_ptr(), out["db"].data_ptr(), ws.data_ptr(),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "classifier_ce")
    return out


@pytest.mark.parametrize("n,K", [(48, 2), (96, 100), (1, 2)])
def test_classifier_ce_kernel_vs_float64(n, K):
    dev = _cuda()
    g = torch.Generator().manual_seed(n * 1000 + K)
    x = torch.randn(n, 1024, generator=g)
    w = torch.randn(K, 1024, generator=g) * 0.05
    b = torch.randn(K, generator=g) * 0.1
    t = torch.randint(0, K, (n,), generator=g)
    xd, wd, bd = (v.double().requires_grad_(True) for v in (x, w, b))
    logits = torch.nn.functional.linear(xd, wd, bd)
    loss = torch.nn.CrossEntropyLoss()(logits, t)
    loss.backward()
    args = [v.to(dev) for v in (x, w, b, t)]
    o = _ce(*args)
    torch.cuda.synchronize()
    errs = {"logits": _max_rel(o["logits"], logits.detach()), "loss": _max_rel(o["loss"], loss.detach().view(1)),
            "dx": _max_rel(o["dx"], xd.grad), "dw": _max_rel(o["dw"], wd.grad), "db": _max_rel(o["db"], bd.grad)}
    print("classifier_ce n=%d K=%d max rel err vs float64: %s" % (n, K, {k: "%.1e" % v for k, v in errs.items()}))
    assert all(v < 1e-6 for v in errs.values()), errs
    o2 = _ce(*args)
    for k in o:
        assert torch.equal(o[k], o2[k]), k                      # deterministic: bitwise equal
    for s in (0.25, 8.0):
        o3 = _ce(*args, loss_scale=s)
        assert torch.equal(o3["logits"], o["logits"]) and torch.equal(o3["loss"], o["loss"])
        for k in ("dx", "dw", "db"):
            assert torch.equal(o3[k], o[k] * s), (s, k)
    # a target outside [0, K): NaN loss, no gradient from that row, nothing read out of bounds
    bad = args[3].clone()
    bad[0] = K
    o4 = _ce(args[0], args[1], args[2], bad)
    assert torch.isnan(o4["loss"]).all() and torch.isfinite(o4["dw"]).all() and not o4["dx"][0].any()


# ---- 2. course-only pooling ----------------------------------------------------------------------------------------------
def test_zero_part_pooling():
    dev = _cuda()
    from ssn_b200.engine import STPPFunction, _stream
    from ssn_b200._lib import lib, check
    g = torch.Generator().manual_seed(3)
    ft = torch.randn(6 * 5, 1024, generator=g).to(dev).requires_grad_(True)
    course, comp = STPPFunction.apply(ft, None, ([], [], [], []), 5, (0, 5))
    ref = ft.detach().double().view(-1, 5, 1024).mean(1)
    assert comp.shape == (6, 0) and rel_l2(course.detach(), ref) < 1e-6
    dc = torch.randn(6, 1024, generator=g).to(dev)
    course.backward(dc)
    assert rel_l2(ft.grad, (dc.double() / 5).repeat_interleave(5, 0)) < 1e-6
    # fused global pool (+ dropout mask) + course mean, reading the engine's last activation
    m = _model(2, "RGB", "exact_tc")
    x = synth.synth_frames(10, 3, seed=4).to(dev)
    eng = m.base_model.engine_for(10, True, dev)
    pooled = eng.forward(x)
    for use_mask in (False, True):
        mask = (torch.bernoulli(torch.full((10, 1024), 0.2), generator=g) / 0.2).to(dev) if use_mask else None
        feat, crs = torch.empty(10, 1024, device=dev), torch.empty(2, 1024, device=dev)
        check(lib.ssnb_gpool_stpp_fwd(eng.h, None if mask is None else mask.data_ptr(), None, 5, 0, None, None, None, None, 0, 5,
                                      feat.data_ptr(), crs.data_ptr(), None, _stream()), eng.h, "gpool_stpp_fwd")
        want = pooled if mask is None else pooled * mask
        assert rel_l2(feat, want) < 1e-6, use_mask
        assert rel_l2(crs, feat.double().view(-1, 5, 1024).mean(1)) < 1e-6, use_mask


# ---- 3. module path -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("modality,precision", [("RGB", "exact"), ("RGB", "exact_tc"), ("Flow", "exact_tc")])
def test_module_path_vs_oracle(modality, precision):
    dev = _cuda()
    C_, K, V, P = (3, 2, 2, 4) if modality == "RGB" else (10, 100, 2, 2)
    m = _model(K, modality, precision)
    x, target = B.synth_binary_batch(V, P, K, C_, seed=1)
    raw, tgt = m(x.to(dev), target.to(dev))
    loss = torch.nn.CrossEntropyLoss()(raw, tgt)
    loss.backward()
    oraw, oloss, ref, _bbo, _t = _oracle(C_, K, x, target)
    params = dict(m.named_parameters())
    e_s, e_l = rel_l2(raw.detach(), oraw), abs(loss.item() - oloss) / abs(oloss)
    agg, cos = _agg_rel(params, ref), _cos(params, ref)
    print("binary module path %s %s: scores %.2e loss %.2e grads %.2e cosine %.6f" % (modality, precision, e_s, e_l, agg, cos))
    assert torch.equal(tgt.cpu(), target.view(-1))
    assert e_s < E2E_TOL[precision] and e_l < E2E_TOL[precision], (e_s, e_l)
    assert agg < (3e-2 if precision == "exact" else 1e-1) and cos > 0.995, (agg, cos)


# ---- 4. fused_step at the reference training shape ------------------------------------------------------------------------
class _MaskMul(torch.nn.Module):
    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def forward(self, x):
        return x * self.mask


_FUSED_REF = {}


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_fused_step_reference_shape(precision):
    """4 videos x 12 proposals x 5 segments = 240 RGB frames, K=2, dropout 0.8 (binary_train.py:25,91), against the oracle
    run with the step's own dropout mask; and against the module path of the same precision with that mask"""
    dev = _cuda()
    K = 2
    m = _model(K, "RGB", precision, dropout=0.8)
    x, target = B.synth_binary_batch(4, 12, K, 3, seed=2)
    torch.manual_seed(11)                           # same mask in both precisions: one oracle run serves both
    loss = m.fused_step(x.to(dev), target.to(dev))
    torch.cuda.synchronize()
    assert not m.base_model.grad_overflow()
    lf = m.last_fused
    mask = lf["mask"].cpu()
    assert mask is not None and 0.15 < float((mask != 0).float().mean()) < 0.25
    if "ref" not in _FUSED_REF or not torch.equal(_FUSED_REF["mask"], mask):
        _FUSED_REF.update(mask=mask, ref=_oracle(3, K, x, target, mask=mask))
    oraw, oloss, ref, _bbo, taps = _FUSED_REF["ref"]
    params = dict(m.named_parameters())
    head = {k: v for k, v in ref.items() if k.startswith("classifier_fc.")}
    bb = {k: v for k, v in ref.items() if k.startswith("base_model.")}
    e = {"feat": rel_l2(lf["feat"], taps["base_out"].detach()), "course": rel_l2(lf["course"], taps["course_ft"].detach()),
         "scores": rel_l2(lf["logits"], oraw), "loss": abs(loss.item() - oloss) / abs(oloss),
         "head_grads": _agg_rel(params, head), "backbone_grads": _agg_rel(params, bb), "backbone_grads_cos": _cos(params, bb)}
    print("binary fused_step F=240 (%s) vs oracle: %s" % (precision, {k: "%.3e" % v for k, v in e.items()}))
    bars = {"exact_tc": {"feat": 2e-4, "course": 2e-4, "scores": 2e-4, "loss": 1e-4, "head_grads": 5e-4, "backbone_grads": 5e-2},
            "fast": {"feat": 3e-2, "course": 3e-2, "scores": 3e-2, "loss": 3e-3, "head_grads": 2e-2, "backbone_grads": 0.6}}[precision]
    for k, b in bars.items():
        assert e[k] < b, (k, e[k], b)
    assert e["backbone_grads_cos"] > (0.999 if precision == "exact_tc" else 0.9), e["backbone_grads_cos"]
    # the module path with the same mask, same precision (forward only; the same engine)
    m.base_model.fc = _MaskMul(lf["mask"])
    raw, tgt = m(x.to(dev), target.to(dev))
    mloss = torch.nn.CrossEntropyLoss()(raw, tgt)
    assert rel_l2(raw.detach(), lf["logits"]) < 1e-5 and abs(mloss.item() - loss.item()) <= 1e-5 * abs(loss.item())


# ---- 5. CUDA graph ----------------------------------------------------------------------------------------------------
def test_fused_step_graph_replay_equals_eager():
    dev = _cuda()
    from ssn_b200.optim import FusedSGD
    K = 2
    x, target = (t.to(dev) for t in B.synth_binary_batch(2, 4, K, 3, seed=3))

    def make():
        m = _model(K, "RGB", "exact_tc")
        order = [p for p in m.parameters() if p.requires_grad]
        opt = FusedSGD(m.get_optim_policies(), lr=1e-3, momentum=0.9, weight_decay=5e-4, order=order,
                       on_step=[m.base_model.invalidate_packed])

        def step():
            opt.flat_grad.zero_()
            loss = m.fused_step(x, target)
            opt.step()
            return loss
        return m, opt, step
    m1, opt1, step1 = make()
    m2, opt2, step2 = make()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step2()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step2()
    graph.replay()
    for _ in range(4):
        l1 = step1()
    torch.cuda.synchronize()
    assert torch.equal(l1, static_loss)
    assert torch.equal(opt1.flat_param, opt2.flat_param) and torch.equal(opt1.flat_grad, opt2.flat_grad)


# ---- 6. test mode ---------------------------------------------------------------------------------------------------------
def test_test_mode_checkpoint_and_scores():
    """binary_test.py:100-140: a training checkpoint (DataParallel `module.` keys) loads after the prefix is stripped, then
    prepare_test_fc, then net(frames, None) over 4 ticks x 10 crops"""
    dev = _cuda()
    import binary_model
    K = 2
    trained = _model(K, "RGB", "exact")
    ckpt = {"module." + k: v.detach().cpu() for k, v in trained.state_dict().items()}
    net = binary_model.BinaryClassifier(K, 5, "RGB", test_mode=True, new_length=1, base_model="BNInception")
    net.load_state_dict({'.'.join(k.split('.')[1:]): v for k, v in ckpt.items()})
    net.prepare_test_fc()
    net.eval()
    net.cuda()
    frames = synth.synth_frames(40, 3, seed=5)
    with torch.no_grad():
        rst, base = net(frames.view(-1, 3, 224, 224).to(dev), None)
    assert rst.shape == (40, K) and base.shape == (40, 1024)
    oscores, obase = B.binary_test_forward(_backbone(3), B.synth_classifier(K, seed=0), frames, 3)
    print("binary test mode: scores %.2e base_out %.2e" % (rel_l2(rst, oscores), rel_l2(base, obase)))
    assert rel_l2(rst, oscores) < 1e-4 and rel_l2(base, obase) < 1e-4


# ---- 7. bn_mode='partial' ---------------------------------------------------------------------------------------------
def test_bn_mode_partial_module_path():
    dev = _cuda()
    K = 2
    m = _model(K, "RGB", "exact_tc", bn_mode="partial")
    bn1 = m.base_model.conv1_7x7_s2_bn
    assert bn1.training and bn1.weight.requires_grad and not m.base_model.conv2_3x3_bn.training
    x, target = B.synth_binary_batch(2, 2, K, 3, seed=6)
    raw, tgt = m(x.to(dev), target.to(dev))
    torch.nn.CrossEntropyLoss()(raw, tgt).backward()
    with pytest.raises(NotImplementedError):
        m.fused_step(x.to(dev), target.to(dev))
    oraw, _ol, ref, bbo, taps = _oracle(3, K, x, target, bn_train_first=True)
    params = dict(m.named_parameters())
    e = {"fwd": rel_l2(raw.detach(), oraw), "running_mean": rel_l2(bn1.running_mean, bbo["conv1_7x7_s2_bn.running_mean"]),
         "running_var": rel_l2(bn1.running_var, bbo["conv1_7x7_s2_bn.running_var"]),
         "dgamma": rel_l2(bn1.weight.grad, ref["base_model.conv1_7x7_s2_bn.weight"]),
         "dbeta": rel_l2(bn1.bias.grad, ref["base_model.conv1_7x7_s2_bn.bias"]),
         "conv1_dw": rel_l2(params["base_model.conv1_7x7_s2.weight"].grad, ref["base_model.conv1_7x7_s2.weight"]),
         "5b_1x1_dw": rel_l2(params["base_model.inception_5b_1x1.weight"].grad, ref["base_model.inception_5b_1x1.weight"])}
    print("binary bn partial (exact_tc): %s" % {k: "%.2e" % v for k, v in e.items()})
    assert e["fwd"] < E2E_TOL["exact_tc"] and e["running_mean"] < 1e-5 and e["running_var"] < 1e-5, e
    assert e["dgamma"] < 5e-2 and e["dbeta"] < 5e-2 and e["conv1_dw"] < 5e-2 and e["5b_1x1_dw"] < 1e-2, e


# ---- 8. data parallel bucket coverage -----------------------------------------------------------------------------------
def test_grad_sync_covers_the_classifier():
    dev = _cuda()
    from ssn_b200.dp import GradSync
    from ssn_b200.optim import FusedSGD
    K = 2
    m = _model(K, "RGB", "exact_tc")
    order = [p for p in m.parameters() if p.requires_grad]
    opt = FusedSGD(m.get_optim_policies(), lr=0.0, momentum=0.0, weight_decay=0.0, order=order)
    sync = GradSync(opt.flat_grad, order, m)
    assert sync.heads_lo == opt.flat_grad.numel() - K * 1024 - K        # classifier_fc is the head bucket
    x, target = (t.to(dev) for t in B.synth_binary_batch(2, 4, K, 3, seed=7))
    m.fused_step(x, target, loss_scale=1.0, grad_sync=sync)
    sync.finish()
    torch.cuda.synchronize()
    spans = sorted(sync.launched)
    assert len(spans) == 4 and spans[0][0] == 0 and spans[-1][1] == opt.flat_grad.numel(), spans
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:])), spans
    assert torch.isfinite(opt.flat_grad).all() and opt.flat_grad[sync.heads_lo:].abs().sum() > 0
