"""GPU parity tests: the CUDA path (through the C ABI / the reference-shaped module surface) against
the CPU oracle and the committed golden vectors.  Run on an H100: pytest -m gpu."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ssn_oracle as O
from oracle import synth


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


# ---- STPP ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag,cfg,seg", [("pyr", (1, (1, 2), 1), (2, 5, 2)), ("flat", [1, 1, 1], (2, 5, 2)),
                                         ("seg3", [1, 1, 1], (1, 1, 1)), ("seg3nan", (1, (1, 2), 1), (1, 1, 1)),
                                         ("deep", ((1, 2), (1, 2, 4), 2), (4, 8, 4))])
def test_stpp_golden(golden_dir, tag, cfg, seg):
    dev = _cuda()
    from ops.ssn_ops import StructuredTemporalPyramidPooling
    z = _load(golden_dir, "stpp.npz")
    ft = torch.tensor(z[tag + "_ft"], device=dev, requires_grad=True)
    S = sum(seg)
    mod = StructuredTemporalPyramidPooling(ft.shape[1], True, configs=cfg)
    a, c = mod(ft, torch.tensor(z[tag + "_sc"], device=dev), [seg[0], seg[0] + seg[1], S])
    # <= 2 ulp (SURVEY §8c); NaN positions must coincide
    ref_a, ref_c = z[tag + "_act"], z[tag + "_comp"]
    assert np.array_equal(np.isnan(c.detach().cpu().numpy()), np.isnan(ref_c))
    np.testing.assert_allclose(a.detach().cpu().numpy(), ref_a, rtol=3e-7, atol=1e-7)
    np.testing.assert_allclose(np.nan_to_num(c.detach().cpu().numpy()), np.nan_to_num(ref_c), rtol=3e-7, atol=1e-7)
    assert mod.feat_multiplier == int(z[tag + "_mult"])
    loss = (a * torch.tensor(z[tag + "_wa"], device=dev)).sum() + (torch.nan_to_num(c) * torch.tensor(z[tag + "_wc"], device=dev)).sum()
    loss.backward()
    got = ft.grad.cpu().numpy()
    ref = z[tag + "_dft"]
    ok = ~np.isnan(ref)
    np.testing.assert_allclose(np.nan_to_num(got[ok]), ref[ok], rtol=2e-6, atol=1e-6)


def test_stpp_large_property():
    """full-size property: STPP is linear in ft and the course part equals the mean of segments 2..6"""
    dev = _cuda()
    from ops.ssn_ops import StructuredTemporalPyramidPooling
    n, D = 4096, 1024
    g = torch.Generator().manual_seed(5)
    ft = torch.randn(n * 9, D, generator=g).to(dev)
    sc = torch.rand(n, 2, generator=g).to(dev)
    mod = StructuredTemporalPyramidPooling(D, True)
    a1, c1 = mod(ft, sc, [2, 7, 9])
    a2, c2 = mod(ft * 2.0, sc, [2, 7, 9])
    assert torch.equal(a2, a1 * 2.0) and torch.equal(c2, c1 * 2.0)
    ref = ft.view(n, 9, D)[:, 2:7].mean(1)
    assert rel_l2(a1, ref) < 1e-6
    # checksum of checksums: sum over parts of course pyramid == relation between levels
    lvl1 = c1[:, D:2 * D] * 3.0
    lvl2 = (c1[:, 2 * D:3 * D] * 3.0 * 2 + c1[:, 3 * D:4 * D] * 3.0 * 3) / 5.0
    assert rel_l2(lvl2, lvl1) < 1e-5


# ---- losses -----------------------------------------------------------------------------------------
def test_losses_golden(golden_dir):
    dev = _cuda()
    import ops.ssn_ops as R
    z = _load(golden_dir, "losses.npz")
    pred = torch.tensor(z["ohem_pred"], device=dev)
    labels = torch.tensor(z["ohem_labels"], device=dev)
    for tag, pos, ratio, gs in (("pos", 1, 1.0, 1), ("neg", -1, 0.17, 7), ("half", -1, 0.5, 4)):
        p = pred.clone().requires_grad_(True)
        l = R.OHEMHingeLoss.apply(p, labels, pos, ratio, gs)
        assert tuple(l.shape) == (1,)
        (l * 1.7).sum().backward()
        np.testing.assert_allclose(l.detach().cpu().numpy(), z["ohem_" + tag + "_loss"], rtol=1e-6)
        got, ref = p.grad.cpu().numpy(), z["ohem_" + tag + "_grad"]
        assert np.array_equal(got != 0, ref != 0)          # kept-index sets: exact
        np.testing.assert_allclose(got, ref, rtol=1e-6)
    p = pred.clone().requires_grad_(True)
    l = R.OHEMHingeLoss.apply(p, torch.tensor(z["ohem_wrap_labels"], device=dev), -1, 0.3, 7)
    l.sum().backward()
    np.testing.assert_allclose(l.detach().cpu().numpy(), z["ohem_wrap_loss"], rtol=1e-6)
    np.testing.assert_array_equal(p.grad.cpu().numpy(), z["ohem_wrap_grad"])
    p = pred.clone().requires_grad_(True)
    cl = R.CompletenessLoss()(p, labels, 1, 7)
    cl.sum().backward()
    np.testing.assert_allclose(cl.detach().cpu().numpy(), z["comp_loss"], rtol=1e-6)
    np.testing.assert_allclose(p.grad.cpu().numpy(), z["comp_grad"], rtol=1e-6)
    rp = torch.tensor(z["reg_pred"], device=dev, requires_grad=True)
    l = R.ClassWiseRegressionLoss()(rp, torch.tensor(z["reg_labels"], device=dev), torch.tensor(z["reg_targets"], device=dev))
    l.backward()
    np.testing.assert_allclose(l.item(), z["reg_loss"], rtol=1e-6)
    np.testing.assert_allclose(rp.grad.cpu().numpy(), z["reg_grad"], rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("tag,cfg", [("flat", (1, 1, 1)), ("pyr", (1, (1, 2), 1))])
def test_stpp_reorganized_golden(golden_dir, tag, cfg):
    dev = _cuda()
    from ops.ssn_ops import STPPReorgainzed
    z = _load(golden_dir, "test_path.npz")
    K = 3
    scores = torch.tensor(z[tag + "_scores"], device=dev)
    st = STPPReorgainzed(scores.shape[1], K + 1, K, 2 * K, True, True, stpp_cfg=cfg)
    a, c, r = st.forward(scores, torch.tensor(z[tag + "_ticks"]), torch.tensor(z[tag + "_sc"]))
    for got, name in ((a, "_act"), (c, "_comp"), (r, "_reg")):
        ref = z[tag + name]
        got = got.cpu().numpy()
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        np.testing.assert_allclose(np.nan_to_num(got), np.nan_to_num(ref), rtol=2e-6, atol=1e-6)


def test_stpp_reorganized_vs_oracle_big():
    dev = _cuda()
    from ops.ssn_ops import STPPReorgainzed
    g = torch.Generator().manual_seed(3)
    K, T, N = 20, 400, 300
    cfg = (1, (1, 2), 1)
    D = (K + 1) + 5 * K + 5 * 2 * K
    scores = torch.randn(T, D, generator=g)
    ticks = torch.sort(torch.randint(0, T, (N, 4), generator=g), dim=1)[0]
    sc = torch.rand(N, 2, generator=g)
    ref = O.stpp_reorganized(scores, ticks, sc, K + 1, K, 2 * K, cfg)
    mod = STPPReorgainzed(D, K + 1, K, 2 * K, True, True, stpp_cfg=cfg)
    got = mod.forward(scores.to(dev), ticks, sc)
    for a, b in zip(got, ref):
        np.testing.assert_allclose(a.cpu().numpy(), b.numpy(), rtol=1e-5, atol=1e-6)


# ---- heads --------------------------------------------------------------------------------------------
def _heads_case(dev, videos, K, M, seed):
    g = torch.Generator().manual_seed(seed)
    n = videos * 8
    course = torch.randn(n, 1024, generator=g)
    stpp = torch.randn(n, 1024 * M, generator=g)
    hd = synth.synth_heads(K, M, seed=seed, std=0.02, bias_std=0.1)
    ptype = torch.tensor([0, 1, 1, 1, 1, 1, 1, 2]).repeat(videos)
    target = torch.randint(1, K + 1, (n,), generator=g)
    target[ptype == 2] = 0
    rtarget = torch.randn(n, 2, generator=g)
    return course, stpp, hd, ptype, target, rtarget


@pytest.mark.parametrize("videos,K,M", [(4, 20, 5), (2, 4, 3), (8, 200, 5)])
def test_fused_heads_loss_vs_oracle(videos, K, M):
    dev = _cuda()
    import ssn_models
    from ssn_b200.engine import heads_loss_fused
    course, stpp, hd, ptype, target, rtarget = _heads_case(dev, videos, K, M, 7)
    # oracle
    c0 = course.clone().requires_grad_(True); s0 = stpp.clone().requires_grad_(True)
    hp = {k: v.clone().requires_grad_(True) for k, v in hd.items()}
    F = torch.nn.functional
    ra = F.linear(c0, hp["activity_fc.weight"], hp["activity_fc.bias"])
    rc = F.linear(s0, hp["completeness_fc.weight"], hp["completeness_fc.bias"])
    rr = F.linear(s0, hp["regressor_fc.weight"], hp["regressor_fc.bias"]).view(-1, K, 2)
    ai = ((ptype == 0) | (ptype == 2)).nonzero().view(-1); ci = ((ptype == 0) | (ptype == 1)).nonzero().view(-1)
    ri = (ptype == 0).nonzero().view(-1)
    loss, (la, lc, lr) = O.total_loss((ra[ai], target[ai], rc[ci], target[ci], rr[ri], target[ri], rtarget[ri]))
    loss.backward()
    # product
    act_fc = ssn_models._HeadLinear(1024, K + 1).to(dev); comp_fc = ssn_models._HeadLinear(1024 * M, K).to(dev)
    reg_fc = ssn_models._HeadLinear(1024 * M, 2 * K).to(dev)
    for fc, nm in ((act_fc, "activity_fc"), (comp_fc, "completeness_fc"), (reg_fc, "regressor_fc")):
        fc.weight.data.copy_(hd[nm + ".weight"]); fc.bias.data.copy_(hd[nm + ".bias"])
    out = heads_loss_fused(course.to(dev), stpp.to(dev), act_fc, comp_fc, reg_fc, ptype.to(dev), target.to(dev),
                           rtarget.to(dev), K, M)
    np.testing.assert_allclose(out["losses"].cpu().numpy(), [la.item(), lc.item(), lr.item(), loss.item()], rtol=2e-5)
    assert rel_l2(out["raw_act"], ra.detach()) < 1e-5 and rel_l2(out["raw_comp"], rc.detach()) < 1e-5
    assert rel_l2(out["raw_reg"], rr.detach().reshape(-1, 2 * K)) < 1e-5
    assert rel_l2(out["d_course"], c0.grad) < 1e-5 and rel_l2(out["d_stpp"], s0.grad) < 1e-5
    for k, nm in (("act", "activity_fc"), ("comp", "completeness_fc"), ("reg", "regressor_fc")):
        assert rel_l2(out["d_%s_w" % k], hp[nm + ".weight"].grad) < 1e-5, nm
        assert rel_l2(out["d_%s_b" % k], hp[nm + ".bias"].grad) < 1e-5, nm
    # kept (non-zero) gradient positions of the completeness logits are exact
    # (recovered through d_comp_b support: classes with any kept row)
    assert np.array_equal(out["d_comp_b"].cpu().numpy() != 0, hp["completeness_fc.bias"].grad.numpy() != 0)


# ---- backbone ---------------------------------------------------------------------------------------------
def _load_backbone(model_base, bb, dev):
    sd = model_base.state_dict()
    for k, v in bb.items():
        sd[k].copy_(v)
    return model_base.to(dev)


@pytest.fixture(scope="module")
def backbone_rgb():
    return synth.synth_backbone(3, seed=0)


E2E_TOL = {"exact": 1e-4, "exact_tc": 5e-4}     # whole-network bars (north_star: 1e-3)


def _prec(name):
    from ssn_b200 import _lib
    return {"exact": _lib.EXACT_FP32, "fast": _lib.FAST_FP16, "exact_tc": _lib.EXACT_TC}[name]


@pytest.mark.parametrize("precision", ["exact", "exact_tc"])
def test_backbone_exact_golden(golden_dir, backbone_rgb, precision):
    """EXACT (fp32 SIMT) and EXACT_TC (split-operand wgmma) modes, whole backbone, 18 frames: against the
    reference's own output (golden)."""
    dev = _cuda()
    import model_zoo
    from ops.ssn_ops import Identity
    z = _load(golden_dir, "ssn_e2e.npz")
    net = model_zoo.BNInception()
    net.set_precision(_prec(precision), 1024.0)
    net.fc = Identity()
    _load_backbone(net, backbone_rgb, dev).eval()
    x, *_ = synth.synth_batch(2, 4, 3, seed=0)
    frames = x.view(-1, 3, 224, 224)[:18].to(dev)
    with torch.no_grad():
        out = net(frames)
    err = rel_l2(out, torch.tensor(z["rgb_base_out18"]))
    print("backbone 18 frames (%s) rel-L2 vs reference golden: %.3e" % (precision, err))
    # tolerance: 1e-3 relative fp32 (north_star).  Measured on H100: exact 1.0e-5; exact_tc 3.2e-5 (per-layer 1e-6..3e-6 --
    # 22-bit split operands, tensor-core accumulation -- amplified by the ReLU switching of 69 random layers)
    assert err < E2E_TOL[precision], err


@pytest.mark.parametrize("precision", ["exact", "exact_tc", "fast"])
def test_backbone_per_layer(backbone_rgb, precision):
    """each op fed the ORACLE's input for that op; forward outputs and (training) backward
    gradients compared per kernel boundary.  exact: 2e-5; fast (fp16 operands, fp32 accumulate): 3e-3 rel-L2
    (measured worst ~1.2e-3 on pool_proj layers; most layers ~3e-4)."""
    dev = _cuda()
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    Fn = 2
    tol = 3e-3 if precision == "fast" else 2e-5
    x = synth.synth_frames(Fn, 3, seed=3)
    bb = {k: v.clone() for k, v in backbone_rgb.items()}
    for k in bb:
        if k.endswith(".weight") and "_bn" not in k or k.endswith(".bias") and "_bn" not in k:
            bb[k].requires_grad_(True)
    taps = {}
    xr = x.clone().requires_grad_(True)
    feat = O.backbone_forward(bb, xr, 3, taps=taps)
    taps["data"] = xr
    for t in taps.values():
        if t.requires_grad:
            t.retain_grad()
    g = torch.Generator().manual_seed(9)
    dfeat = torch.randn(feat.shape, generator=g) * 0.01
    feat.backward(dfeat)
    eng = BackboneEngine(3, Fn, _prec(precision), True, 1024.0, dev)
    names = [n for (n, *_r) in O.conv_layers(3)]
    eng.pack([bb[n + ".weight"].detach().to(dev) for n in names], [bb[n + ".bias"].detach().to(dev) for n in names],
             [bb[n + "_bn.weight"].to(dev) for n in names], [bb[n + "_bn.bias"].to(dev) for n in names],
             [bb[n + "_bn.running_mean"].to(dev) for n in names], [bb[n + "_bn.running_var"].to(dev) for n in names])
    dw = [torch.zeros_like(bb[n + ".weight"].detach()).to(dev) for n in names]
    db = [torch.zeros_like(bb[n + ".bias"].detach()).to(dev) for n in names]
    eng.bind_grads(dw, db)
    conv_idx = 0
    worst = {}
    for i, (kind, iname, oname) in enumerate(eng.ops()):
        if kind == "gpool":
            continue
        eng.write(iname, taps[iname].detach().to(dev))
        eng.run_op(i, backward=False)
        got = eng.read(oname)
        e = rel_l2(got, taps[oname].detach())
        worst["fwd " + oname] = e
        assert e < tol, ("fwd", oname, e)
        if precision == "exact_tc":
            # the fp16 hi/lo operand planes the next convolution reads carry the fp32 value to ~2^-22
            ep = rel_l2(eng.read(oname, planes=True), got)
            assert ep < 2e-6, ("planes", oname, ep)
        # backward of this op: feed oracle activations (already there) and oracle output-gradient
        gout = taps[oname].grad
        eng.write(oname, taps[oname].detach().to(dev))            # the op's true output (ReLU mask source)
        eng.write(oname, gout.to(dev), grad=True)
        if iname != "data":
            eng.write(iname, torch.zeros_like(taps[iname].detach()).to(dev), grad=True)
        eng.run_op(i, backward=True)
        if kind == "conv":
            n = names[conv_idx]
            ew = rel_l2(dw[conv_idx], bb[n + ".weight"].grad)
            eb = rel_l2(db[conv_idx], bb[n + ".bias"].grad)
            worst["wgrad " + n] = ew
            assert ew < tol * 2 and eb < tol * 2, ("wgrad", n, ew, eb)
            conv_idx += 1
    # dgrad per op: run each op's backward alone into a zeroed input-gradient and compare with the
    # oracle's autograd contribution of that op (computed by a local vjp)
    for i, (kind, iname, oname) in enumerate(eng.ops()):
        if kind == "gpool" or iname == "data":
            continue
        gout = taps[oname].grad
        xin = taps[iname].detach().clone()
        if precision == "fast" and kind == "maxpool":
            xin = xin.half().float()     # fp16 storage creates ties the fp32 oracle would route differently
        xin.requires_grad_(True)
        ref_in = _oracle_single_op(bb, kind, oname, xin)
        (gref,) = torch.autograd.grad(ref_in, xin, gout)
        eng.write(iname, taps[iname].detach().to(dev))
        eng.write(oname, taps[oname].detach().to(dev))
        eng.write(oname, gout.to(dev), grad=True)
        if kind == "maxpool":
            eng.run_op(i, backward=False)                      # regenerate argmax for this input
            eng.write(oname, gout.to(dev), grad=True)
        eng.write(iname, torch.zeros_like(xin.detach()).to(dev), grad=True)
        # force "first writer" semantics irrespective of plan flags: zeroed buffer + accumulate is the same
        eng.run_op(i, backward=True)
        got = eng.read(iname, grad=True)
        e = rel_l2(got, gref)
        worst["dgrad " + oname] = e
        assert e < tol * 2, ("dgrad", oname, e)
    print("per-layer worst (%s): %s" % (precision, sorted(worst.items(), key=lambda kv: -kv[1])[:5]))


def _oracle_single_op(bb, kind, oname, xin):
    Fnn = torch.nn.functional
    if kind == "conv":
        id_ = oname[:-3]
        spec = {n: (k, s, p) for (n, _ci, _co, k, s, p) in O.conv_layers(3)}[id_]
        z = Fnn.conv2d(xin, bb[id_ + ".weight"].detach(), bb[id_ + ".bias"].detach(), spec[1], spec[2])
        z = Fnn.batch_norm(z, bb[id_ + "_bn.running_mean"], bb[id_ + "_bn.running_var"], bb[id_ + "_bn.weight"].detach(),
                           bb[id_ + "_bn.bias"].detach(), False, 0.1, 1e-5)
        return Fnn.relu(z)
    for k_, id_, out, ins, a in O.bninception_ops(3):
        if k_ == "pool" and out == oname:
            return O._pool(xin, a)
    raise KeyError(oname)


@pytest.mark.parametrize("precision", ["exact", "exact_tc"])
def test_ssn_train_exact_vs_oracle(golden_dir, backbone_rgb, precision):
    """whole SSN, B=2 videos (144 frames), EXACT / EXACT_TC mode, through the reference-shaped module surface
    and the reference's training-loop calls (ssn_train.py:207-236): outputs, losses and every
    gradient against the oracle (itself pinned to the reference by tests/golden/ssn_e2e.npz)."""
    dev = _cuda()
    import ssn_models
    import ops.ssn_ops as R
    K = 4
    model = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    hd = synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1)
    sd = model.state_dict()
    for k, v in backbone_rgb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model = model.to(dev)
    model.train()
    gs = float(os.environ.get("SSNB_TEST_GS", "1024"))
    model.set_precision(_prec(precision), gs)
    x, sc, tgt, rtgt, ptype = synth.synth_batch(2, K, 3, seed=0)
    outs = model(x.to(dev), sc.to(dev), tgt.to(dev), rtgt.to(dev), ptype.to(dev))
    act, act_t, comp, comp_t, reg, reg_l, reg_t = outs
    la = torch.nn.CrossEntropyLoss()(act, act_t)
    lc = R.CompletenessLoss()(comp, comp_t, 1, 7)
    lr = R.ClassWiseRegressionLoss()(reg, reg_l, reg_t)
    loss = la + 0.1 * lc + 0.1 * lr
    loss.backward()
    for eng in model.base_model._engines.values():
        assert not eng.grad_overflow(), "gradient operand planes overflowed fp16 under grad_scale %g" % gs
    z = _load(golden_dir, "ssn_e2e.npz")
    for name, o in zip(("act", "act_t", "comp", "comp_t", "reg", "reg_l", "reg_t"), outs):
        ref = z["rgb_" + name]
        if ref.dtype.kind == "f":
            assert rel_l2(o.detach(), torch.tensor(ref)) < E2E_TOL[precision], name
        else:
            np.testing.assert_array_equal(o.cpu().numpy(), ref)     # index selection: bit-exact
    np.testing.assert_allclose([la.item(), lc.item(), lr.item(), loss.item()], z["rgb_losses"], rtol=E2E_TOL[precision])
    # gradients: against the oracle run on THIS machine with the same regenerated weights (the
    # golden gradients were produced with BN statistics calibrated on another CPU; 1e-6 weight
    # differences are amplified by the ReLU/max-pool switching of 69 random layers).  The per-layer
    # test above bounds every kernel at 2e-5; end to end the fp32 reduction-order differences
    # between this GPU path and the CPU oracle grow towards conv1.
    bbo = {k: v.clone() for k, v in backbone_rgb.items()}
    hdo = {k: v.clone() for k, v in hd.items()}
    for d in (bbo, hdo):
        for k in d:
            if "_bn." not in k:
                d[k].requires_grad_(True)
    oloss, _ = O.total_loss(O.ssn_train_forward(bbo, hdo, x, sc, tgt, rtgt, ptype))
    oloss.backward()
    params = dict(model.named_parameters())
    errs = {}
    for n_, p in params.items():
        if p.grad is None:
            continue
        ref = bbo[n_[len("base_model."):]].grad if n_.startswith("base_model.") else hdo[n_].grad
        errs[n_] = rel_l2(p.grad, ref)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("e2e %s grad rel-L2 vs live fp32 oracle, worst:" % precision, worst)
    # Noise floor: the same oracle in float64.  A ReLU whose pre-activation is ~1e-5 from zero flips
    # between any two fp32 evaluation orders and changes that layer's gradient by O(1/sqrt(#active));
    # the fp32 reference itself is therefore only ~1e-2 from the true gradient below the first few
    # layers.  The criterion is: this path is as close to the float64 gradient as the reference is.
    bb64 = {k: v.detach().double() for k, v in backbone_rgb.items()}
    hd64 = {k: v.detach().double() for k, v in hd.items()}
    for d in (bb64, hd64):
        for k in d:
            if "_bn." not in k:
                d[k].requires_grad_(True)
    l64, _ = O.total_loss(O.ssn_train_forward(bb64, hd64, x.double(), sc.double(), tgt, rtgt.double(), ptype))
    l64.backward()

    def agg(get):
        num = den = 0.0
        for n_ in errs:
            ref = (bb64[n_[len("base_model."):]] if n_.startswith("base_model.") else hd64[n_]).grad
            num += float((get(n_).double().cpu() - ref).pow(2).sum()); den += float(ref.pow(2).sum())
        return (num / den) ** 0.5
    ours64 = agg(lambda n_: params[n_].grad)
    ref64 = agg(lambda n_: (bbo[n_[len("base_model."):]] if n_.startswith("base_model.") else hdo[n_]).grad)
    print("e2e %s aggregate gradient rel-L2 vs float64 oracle: ours %.3e, fp32 reference %.3e" % (precision, ours64, ref64))
    # exact_tc: forward differs from fp32 by 2e-4 instead of 1e-6, so proportionally more ReLUs sit inside the flip band
    assert ours64 <= (2.0 if precision == "exact" else 4.0) * ref64 + 1e-4, (ours64, ref64)
    for n_ in ("activity_fc.weight", "completeness_fc.weight", "regressor_fc.weight"):
        assert errs[n_] < (1e-3 if precision == "exact" else 3e-3), (n_, errs[n_])

    # the fused step must reproduce the modular path
    model2 = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    model2.load_state_dict(model.state_dict())
    model2 = model2.to(dev).train()
    model2.set_precision(_prec(precision), 1024.0)
    losses = model2.fused_step(x.to(dev), sc.to(dev), tgt.to(dev), rtgt.to(dev), ptype.to(dev))
    np.testing.assert_allclose(losses.cpu().numpy(), [la.item(), lc.item(), lr.item(), loss.item()], rtol=1e-5)
    print("fused_step (%s) losses" % precision, losses.tolist())
    p2 = dict(model2.named_parameters())
    for n_, p in params.items():
        if p.grad is not None:
            assert rel_l2(p2[n_].grad, p.grad) < 1e-4, n_


@pytest.mark.parametrize("precision", ["exact", "exact_tc"])
def test_flow_forward_exact(golden_dir, precision):
    dev = _cuda()
    import ssn_models
    z = _load(golden_dir, "ssn_e2e.npz")
    K = 4
    model = ssn_models.SSN(K, 2, 5, 2, "Flow", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    bb = synth.synth_backbone(10, seed=0)
    hd = synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1)
    sd = model.state_dict()
    for k, v in bb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model = model.to(dev).train()
    model.set_precision(_prec(precision), 1024.0)
    x, sc, tgt, rtgt, ptype = synth.synth_batch(2, K, 10, seed=0)
    with torch.no_grad():
        outs = model(x.to(dev), sc.to(dev), tgt.to(dev), rtgt.to(dev), ptype.to(dev))
    for name, o in zip(("act", "act_t", "comp", "comp_t", "reg", "reg_l", "reg_t"), outs):
        ref = z["flow_" + name]
        if ref.dtype.kind == "f":
            assert rel_l2(o, torch.tensor(ref)) < E2E_TOL[precision], name
        else:
            np.testing.assert_array_equal(o.cpu().numpy(), ref)


def test_test_forward_and_prepare_test_fc(backbone_rgb):
    """test path: prepare_test_fc folding + test_forward == heads applied after STPP on a constant
    video (pool∘FC = FC∘pool), ssn_models.py:176-201, ssn_test.py:83-87."""
    dev = _cuda()
    import ssn_models
    K = 4
    model = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, test_mode=True, stpp_cfg=(1, 1, 1))
    hd = synth.synth_heads(K, 3, seed=1, std=0.02, bias_std=0.1)
    sd = model.state_dict()
    for k, v in backbone_rgb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model.prepare_test_fc()
    w_ref, b_ref = O.prepare_test_fc(hd, 3)
    np.testing.assert_array_equal(model.test_fc.weight.data.numpy(), w_ref.numpy())
    np.testing.assert_array_equal(model.test_fc.bias.data.numpy(), b_ref.numpy())
    model = model.to(dev).eval()
    x = synth.synth_frames(4, 3, seed=5).to(dev)
    with torch.no_grad():
        scores, base_out = model(x, None, None, None, None)
    ref_feat = O.backbone_forward(backbone_rgb, x.cpu(), 3)
    assert rel_l2(base_out, ref_feat) < 1e-4
    assert rel_l2(scores, torch.nn.functional.linear(ref_feat, w_ref, b_ref)) < 1e-4
    # the same inference call on the tensor-core path (forward-only engine, no gradient buffers)
    from ssn_b200 import _lib
    model.set_precision(_lib.FAST_FP16, 1024.0)
    with torch.no_grad():
        scores_f, base_f = model(x, None, None, None, None)
    assert rel_l2(base_f, ref_feat) < 5e-2 and rel_l2(scores_f, scores) < 5e-2


def test_fast_fused_vs_unfused_and_oracle(backbone_rgb):
    """FAST mode, whole backbone fwd+bwd on 18 frames: the fused schedule (sibling 1x1 fusion, conv1
    space-to-depth, stride-2 sampling, wgmma everywhere) against the same engine with fusion and
    tensor cores disabled (SIMT fp16 kernels), and both against the fp32 oracle."""
    dev = _cuda()
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    Fn = 18
    names = [n for (n, *_r) in O.conv_layers(3)]
    x = synth.synth_frames(Fn, 3, seed=11)
    g = torch.Generator().manual_seed(12)
    dfeat = torch.randn(Fn, 1024, generator=g) * 0.01

    def run(env):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            eng = BackboneEngine(3, Fn, _lib.FAST_FP16, True, 4096.0, dev)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        eng.pack([backbone_rgb[n + ".weight"].to(dev) for n in names], [backbone_rgb[n + ".bias"].to(dev) for n in names],
                 [backbone_rgb[n + "_bn.weight"].to(dev) for n in names], [backbone_rgb[n + "_bn.bias"].to(dev) for n in names],
                 [backbone_rgb[n + "_bn.running_mean"].to(dev) for n in names], [backbone_rgb[n + "_bn.running_var"].to(dev) for n in names])
        feat = eng.forward(x.to(dev))
        dw = [torch.zeros_like(backbone_rgb[n + ".weight"]).to(dev) for n in names]
        db = [torch.zeros_like(backbone_rgb[n + ".bias"]).to(dev) for n in names]
        eng.backward(dfeat.to(dev), dw, db)
        torch.cuda.synchronize()
        return feat, dw, db

    f_fast, dw_fast, db_fast = run({"SSNB_DISABLE_UMMA": "0", "SSNB_DISABLE_FUSION": "0"})
    f_unf, dw_unf, db_unf = run({"SSNB_DISABLE_UMMA": "0", "SSNB_DISABLE_FUSION": "1"})
    f_simt, dw_simt, db_simt = run({"SSNB_DISABLE_UMMA": "1"})
    bb = {k: v.clone() for k, v in backbone_rgb.items()}
    for k in bb:
        if "_bn." not in k:
            bb[k].requires_grad_(True)
    ref = O.backbone_forward(bb, x, 3)
    ref.backward(dfeat)
    # (1) fusion is a pure re-scheduling: identical forward (same MMA order => same ReLU / arg-max decisions),
    #     gradients differ only by where the fp16 rounding of the accumulated data gradient happens
    u_feat = rel_l2(f_fast, f_unf)
    u_w = max(rel_l2(a, b) for a, b in zip(dw_fast, dw_unf))
    u_b = max(rel_l2(a, b) for a, b in zip(db_fast, db_unf))
    # (2) tensor-core path vs SIMT fp16 path: same storage precision, different accumulation order
    e_feat = rel_l2(f_fast, f_simt)
    e_w = max(rel_l2(a, b) for a, b in zip(dw_fast, dw_simt))
    o_feat = rel_l2(f_fast, ref.detach())
    o_w = sorted(((rel_l2(a, bb[n + ".weight"].grad), n) for a, n in zip(dw_fast, names)), reverse=True)[:3]
    print("fast fused vs unfused: feat %.2e max dW %.2e max db %.2e | vs SIMT-fp16: feat %.2e max dW %.2e | vs fp32 oracle: feat %.2e worst dW %s"
          % (u_feat, u_w, u_b, e_feat, e_w, o_feat, o_w))
    assert u_feat < 1e-4 and u_w < 1e-2 and u_b < 1e-2
    # wgmma vs SIMT on the same fp16 operands: identical arithmetic up to accumulation order, but end to end a different
    # rounding flips ReLU / arg-max decisions below; bounded per layer by the median and loosely by the worst layer
    e_ws = sorted(rel_l2(a, b) for a, b in zip(dw_fast, dw_simt))
    print("fast wgmma vs SIMT-fp16 dW rel-L2: median %.2e, worst %.2e" % (e_ws[len(e_ws) // 2], e_ws[-1]))
    assert e_feat < 5e-3 and e_ws[len(e_ws) // 2] < 0.3 and e_ws[-1] < 0.5, (e_feat, e_ws[len(e_ws) // 2], e_ws[-1])    # measured 0.15 / 0.19
    # End-to-end gradients of FAST mode on this synthetic random-weight net are dominated by ReLU / max-pool
    # decision flips (forward differs by ~1e-2 => many flips; cf. the fp32 noise floor of ~1e-2 measured in
    # test_ssn_train_exact_vs_oracle for a 1e-5 forward difference).  The criterion is the direction and the size of
    # the whole gradient (aggregate over the 69 weight tensors) -- the same as test_fused_step_bench_shape[fast];
    # the per-kernel bound is test_backbone_per_layer[fast].
    num = den = dot = na = 0.0
    for a, n in zip(dw_fast, names):
        r = bb[n + ".weight"].grad.double()
        a = a.double().cpu()
        num += float((a - r).pow(2).sum()); den += float(r.pow(2).sum()); dot += float((a * r).sum()); na += float(a.pow(2).sum())
    agg, cos = (num / den) ** 0.5, dot / (na * den) ** 0.5
    print("fast whole-backbone dW vs fp32 oracle: aggregate rel-L2 %.3f, cosine %.4f" % (agg, cos))
    assert o_feat < 5e-2 and agg < 0.6 and cos > 0.9, (o_feat, agg, cos)


@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_flow_conv1_fwd_bwd(precision):
    """Flow modality (10-channel stacked flow, ssn_models.py:318-343): the first convolution is the only
    layer whose geometry changes; forward + weight/bias gradient per kernel boundary, and the whole
    backbone forward in FAST mode through the packed space-to-depth input path."""
    dev = _cuda()
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    Fn = 4
    bb = synth.synth_backbone(10, seed=1, calib_frames=2)
    names = [n for (n, *_r) in O.conv_layers(10)]
    x = synth.synth_frames(Fn, 10, seed=2)
    w = bb["conv1_7x7_s2.weight"].clone().requires_grad_(True)
    b = bb["conv1_7x7_s2.bias"].clone().requires_grad_(True)
    Fnn = torch.nn.functional
    z = Fnn.conv2d(x, w, b, 2, 3)
    y = Fnn.relu(Fnn.batch_norm(z, bb["conv1_7x7_s2_bn.running_mean"], bb["conv1_7x7_s2_bn.running_var"],
                                bb["conv1_7x7_s2_bn.weight"], bb["conv1_7x7_s2_bn.bias"], False, 0.1, 1e-5))
    g = torch.Generator().manual_seed(3)
    gy = torch.randn(y.shape, generator=g) * 0.01
    y.backward(gy)
    prec = _lib.EXACT_FP32 if precision == "exact" else _lib.FAST_FP16
    tol = 2e-5 if precision == "exact" else 3e-3
    eng = BackboneEngine(10, Fn, prec, True, 1024.0, dev)
    eng.pack([bb[n + ".weight"].to(dev) for n in names], [bb[n + ".bias"].to(dev) for n in names],
             [bb[n + "_bn.weight"].to(dev) for n in names], [bb[n + "_bn.bias"].to(dev) for n in names],
             [bb[n + "_bn.running_mean"].to(dev) for n in names], [bb[n + "_bn.running_var"].to(dev) for n in names])
    dw = [torch.zeros_like(bb[n + ".weight"]).to(dev) for n in names]
    db = [torch.zeros_like(bb[n + ".bias"]).to(dev) for n in names]
    eng.bind_grads(dw, db)
    eng.write("data", x.to(dev))
    eng.run_op(0, backward=False)
    assert rel_l2(eng.read("conv1_7x7_s2_bn"), y.detach()) < tol
    eng.write("conv1_7x7_s2_bn", y.detach().to(dev))
    eng.write("conv1_7x7_s2_bn", gy.to(dev), grad=True)
    eng.run_op(0, backward=True)
    assert rel_l2(dw[0], w.grad) < 2 * tol and rel_l2(db[0], b.grad) < 2 * tol
    feat = eng.forward(x.to(dev))
    ref = O.backbone_forward(bb, x, 10)
    assert rel_l2(feat, ref) < (1e-4 if precision == "exact" else 5e-2)


def _agg_rel(get_ours, ref_grads):
    num = den = 0.0
    for n_, r in ref_grads.items():
        num += float((get_ours(n_).double().cpu() - r.double()).pow(2).sum()); den += float(r.double().pow(2).sum())
    return (num / den) ** 0.5


def _cos(get_ours, ref_grads):
    dot = na = nb = 0.0
    for n_, r in ref_grads.items():
        a = get_ours(n_).double().cpu().flatten(); b = r.double().flatten()
        dot += float(a @ b); na += float(a @ a); nb += float(b @ b)
    return dot / (na * nb) ** 0.5


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_fused_step_bench_shape(precision):
    """What bench.py times: SSN.fused_step at the BASELINE configs[1] shape (4 videos x 8 proposals x 9 segments = 288
    frames, K=20, STPP (1,(1,2),1)) in the benched precision modes, against the CPU oracle on the same batch: losses, the
    fused global-pool + STPP outputs (feat / course / stpp), head logits and head gradients, and the 138 backbone
    gradients in aggregate.  Bars: exact_tc is the parity mode (north_star 1e-3 on outputs); fast is reported with the
    bars its fp16 operands can meet (DESIGN.md section 2)."""
    dev = _cuda()
    import ssn_models
    K, V = 20, 4
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    hd = synth.synth_heads(K, 5, seed=0, std=0.01, bias_std=0.05)
    model = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    sd = model.state_dict()
    for k, v in bb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model = model.to(dev).train()
    model.set_precision(_prec(precision), 4096.0)
    batch = synth.synth_batch(V, K, 3, seed=100)
    losses = model.fused_step(*[t.to(dev) for t in batch])
    torch.cuda.synchronize()
    for eng in model.base_model._engines.values():
        assert not eng.grad_overflow()
    bbo = {k: v.clone() for k, v in bb.items()}
    hdo = {k: v.clone() for k, v in hd.items()}
    for d in (bbo, hdo):
        for k in d:
            if "_bn." not in k:
                d[k].requires_grad_(True)
    x, sc, tgt, rtgt, ptype = batch
    feat_ref = O.backbone_forward(bbo, x.view(-1, 3, 224, 224), 3)
    course_ref, stpp_ref = O.stpp_forward(feat_ref, sc.view(-1, 2), [2, 7, 9], (1, (1, 2), 1))
    outs = O.ssn_train_forward(bbo, hdo, x, sc, tgt, rtgt, ptype)
    oloss, (la, lc, lr) = O.total_loss(outs)
    oloss.backward()
    lf = model.last_fused
    e = {"feat": rel_l2(lf["feat"], feat_ref.detach()), "course": rel_l2(lf["course"], course_ref.detach()),
         "stpp": rel_l2(lf["stpp"], stpp_ref.detach())}
    ref_l = np.array([la.item(), lc.item(), lr.item(), oloss.item()])
    e["loss"] = float(np.abs(losses.cpu().numpy() - ref_l).max() / np.abs(ref_l).max())
    params = dict(model.named_parameters())
    head_ref = {k: v.grad for k, v in hdo.items()}
    bb_ref = {"base_model." + k: v.grad for k, v in bbo.items() if v.grad is not None}
    e["head_grads"] = _agg_rel(lambda n_: params[n_].grad, head_ref)
    e["backbone_grads"] = _agg_rel(lambda n_: params[n_].grad, bb_ref)
    e["backbone_grads_cos"] = _cos(lambda n_: params[n_].grad, bb_ref)
    print("fused_step F=288 (%s) vs fp32 oracle: %s" % (precision, {k: "%.3e" % v for k, v in e.items()}))
    print("fused_step F=288 (%s) losses %s oracle %s" % (precision, losses.tolist(), ref_l.tolist()))
    # measured on H100: exact_tc feat 3.4e-5, loss 6e-7, head grads 2.7e-5, backbone grads 1.1e-2 (cosine 0.9999; the
    # fp32 reference itself is 7.6e-3 from the float64 gradient on this random-weight net, test_ssn_train_exact_vs_oracle);
    # fast feat 9.2e-3, loss 3e-4, head grads 3.1e-3, backbone grads 0.27 (cosine 0.964): outside the 1e-3 tolerance, reported
    bars = {"exact_tc": {"feat": 2e-4, "course": 2e-4, "stpp": 2e-4, "loss": 1e-4, "head_grads": 5e-4, "backbone_grads": 5e-2},
            "fast": {"feat": 3e-2, "course": 3e-2, "stpp": 3e-2, "loss": 3e-3, "head_grads": 2e-2, "backbone_grads": 0.6}}[precision]
    for k, b in bars.items():
        assert e[k] < b, (k, e[k], b)
    assert e["backbone_grads_cos"] > (0.999 if precision == "exact_tc" else 0.9), e["backbone_grads_cos"]


@pytest.mark.parametrize("precision", ["exact", "exact_tc"])
def test_flow_train_vs_oracle(precision):
    """whole-net Flow (2x5-channel, conv1 with 10 input channels) forward + backward through the module surface, B=2 videos
    (144 frames): the 7 outputs, the losses and all gradients against the CPU oracle (ssn_models.py:318-343 conv1 shape)."""
    dev = _cuda()
    import ssn_models
    import ops.ssn_ops as R
    K = 4
    bb = synth.synth_backbone(10, seed=0)
    hd = synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1)
    model = ssn_models.SSN(K, 2, 5, 2, "Flow", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
    sd = model.state_dict()
    for k, v in bb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model = model.to(dev).train()
    model.set_precision(_prec(precision), 1024.0)
    x, sc, tgt, rtgt, ptype = synth.synth_batch(2, K, 10, seed=0)
    outs = model(x.to(dev), sc.to(dev), tgt.to(dev), rtgt.to(dev), ptype.to(dev))
    act, act_t, comp, comp_t, reg, reg_l, reg_t = outs
    loss = torch.nn.CrossEntropyLoss()(act, act_t) + 0.1 * R.CompletenessLoss()(comp, comp_t, 1, 7) + 0.1 * R.ClassWiseRegressionLoss()(reg, reg_l, reg_t)
    loss.backward()
    bbo = {k: v.clone() for k, v in bb.items()}
    hdo = {k: v.clone() for k, v in hd.items()}
    for d in (bbo, hdo):
        for k in d:
            if "_bn." not in k:
                d[k].requires_grad_(True)
    oouts = O.ssn_train_forward(bbo, hdo, x, sc, tgt, rtgt, ptype, in_channels=10)
    oloss, _ = O.total_loss(oouts)
    oloss.backward()
    for name, o, r in zip(("act", "act_t", "comp", "comp_t", "reg", "reg_l", "reg_t"), outs, oouts):
        if r.dtype.is_floating_point:
            assert rel_l2(o.detach(), r.detach()) < E2E_TOL[precision], name
        else:
            np.testing.assert_array_equal(o.cpu().numpy(), r.numpy())
    assert abs(loss.item() - oloss.item()) < E2E_TOL[precision] * abs(oloss.item())
    params = dict(model.named_parameters())
    ref = {"base_model." + k: v.grad for k, v in bbo.items() if v.grad is not None}
    ref.update({k: v.grad for k, v in hdo.items()})
    agg, cos = _agg_rel(lambda n_: params[n_].grad, ref), _cos(lambda n_: params[n_].grad, ref)
    c1 = rel_l2(params["base_model.conv1_7x7_s2.weight"].grad, bbo["conv1_7x7_s2.weight"].grad)
    print("flow e2e (%s): aggregate gradient rel-L2 vs fp32 oracle %.3e, cosine %.6f, conv1 (10-ch) dW %.3e" % (precision, agg, cos, c1))
    # two fp32-grade evaluations of this random-weight net differ by ReLU / max-pool switching (see test_ssn_train_exact_vs_oracle)
    assert agg < (3e-2 if precision == "exact" else 1e-1) and cos > 0.995, (agg, cos)


def test_test_scores_cropmean(backbone_rgb):
    """f2: SSN.test_scores (10-crop mean folded into the folded test FC, one kernel) == the reference loop body
    `rst, _ = net(frames); rst.view(num_crop, -1, D).mean(0)` (ssn_test.py:83-84)."""
    dev = _cuda()
    import ssn_models
    K, crops, nt = 4, 10, 3
    model = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, test_mode=True, stpp_cfg=(1, (1, 2), 1))
    hd = synth.synth_heads(K, 5, seed=1, std=0.02, bias_std=0.1)
    sd = model.state_dict()
    for k, v in backbone_rgb.items():
        sd["base_model." + k].copy_(v)
    for k, v in hd.items():
        sd[k].copy_(v)
    model.prepare_test_fc()
    model = model.to(dev).eval()
    x = synth.synth_frames(crops * nt, 3, seed=6).to(dev)
    with torch.no_grad():
        rst, _ = model(x, None, None, None, None)
        ref = rst.view(crops, -1, rst.shape[1]).mean(dim=0)
        got = model.test_scores(x, crops)
    assert got.shape == ref.shape
    assert rel_l2(got, ref) < 1e-5
    w_ref, b_ref = O.prepare_test_fc(hd, 5)
    feat = O.backbone_forward(backbone_rgb, x.cpu(), 3)
    oracle = torch.nn.functional.linear(feat, w_ref, b_ref).view(crops, -1, w_ref.shape[0]).mean(dim=0)
    assert rel_l2(got, oracle) < 1e-4


def test_stpp_large_vs_oracle():
    """the vectorised STPP kernels at a bandwidth-bound size (2048 proposals) and with a deep pyramid: forward and backward
    against the oracle restatement of ops/ssn_ops.py:39-70 (part boundaries exact, values <= 1e-6)."""
    dev = _cuda()
    from ops.ssn_ops import StructuredTemporalPyramidPooling
    g = torch.Generator().manual_seed(21)
    for cfg, seg, n, D in (((1, (1, 2), 1), (2, 5, 2), 2048, 1024), (((1, 2), (1, 2, 4), 2), (4, 8, 4), 64, 256), ([1, 1, 1], (2, 5, 2), 33, 1024)):
        S = sum(seg)
        split = [seg[0], seg[0] + seg[1], S]
        ft = torch.randn(n * S, D, generator=g)
        sc = torch.rand(n, 2, generator=g)
        fr = ft.clone().requires_grad_(True)
        ra, rc = O.stpp_forward(fr, sc, split, cfg)
        wa, wc = torch.randn(ra.shape, generator=g), torch.randn(rc.shape, generator=g)
        (ra * wa).sum().add((rc * wc).sum()).backward()
        mod = StructuredTemporalPyramidPooling(D, True, configs=cfg)
        fd = ft.clone().to(dev).requires_grad_(True)
        a, c = mod(fd, sc.to(dev), split)
        ((a * wa.to(dev)).sum() + (c * wc.to(dev)).sum()).backward()
        assert torch.allclose(a.detach().cpu(), ra.detach(), rtol=1e-6, atol=1e-6) and torch.allclose(c.detach().cpu(), rc.detach(), rtol=1e-6, atol=1e-6)
        assert torch.allclose(fd.grad.cpu(), fr.grad, rtol=1e-6, atol=1e-6)


def test_fused_sgd_matches_torch(backbone_rgb):
    """f4: ssn_b200.optim.FusedSGD (one launch over flat buffers, per-group lr_mult / decay_mult of SSN.get_optim_policies,
    ssn_train.py:141-144,391-398) against torch.optim.SGD on the same parameter groups, three steps with momentum."""
    dev = _cuda()
    import ssn_models
    from ssn_b200.optim import FusedSGD
    K = 4

    def make():
        m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
        sd = m.state_dict()
        for k, v in backbone_rgb.items():
            sd["base_model." + k].copy_(v)
        return m.to(dev).train()
    torch.manual_seed(3)
    m1 = make()
    torch.manual_seed(3)
    m2 = make()
    lr, wd, mom = 0.01, 5e-4, 0.9
    pol1 = m1.get_optim_policies()
    groups = [{"params": g["params"], "lr": lr * g["lr_mult"], "weight_decay": wd * g["decay_mult"]} for g in pol1 if g["params"]]
    ref = torch.optim.SGD(groups, lr=lr, momentum=mom)
    invalidated = []
    opt = FusedSGD(m2.get_optim_policies(), lr=lr, momentum=mom, weight_decay=wd, on_step=[lambda: invalidated.append(1), m2.base_model.invalidate_packed])
    assert [len(g["params"]) for g in opt.param_groups] == [len(g["params"]) for g in groups]
    g = torch.Generator().manual_seed(4)
    p1 = [p for p in m1.parameters() if p.requires_grad]
    p2 = [p for p in m2.parameters() if p.requires_grad]
    assert len(p1) == len(p2) == 144
    for step in range(3):
        for a, b in zip(p1, p2):
            gr = torch.randn(a.shape, generator=g).to(dev)
            a.grad = gr.clone()
            if step == 1:
                b.grad = None                    # zero_grad(set_to_none=True) in the reference loop: the optimizer re-binds
                opt.rebind_grads()
            b.grad.copy_(gr)
        ref.step()
        opt.step()
        worst = max(rel_l2(b, a) for a, b in zip(p1, p2))
        assert worst < 1e-6, (step, worst)
    assert len(invalidated) == 3
    # lr schedule: adjust_learning_rate rewrites the groups' lr / weight_decay
    for gr_, go in zip(ref.param_groups, opt.param_groups):
        gr_["lr"] *= 0.1
        go["lr"] *= 0.1
    opt.refresh_groups()
    for a, b in zip(p1, p2):
        gr = torch.randn(a.shape, generator=g).to(dev)
        a.grad = gr.clone(); b.grad.copy_(gr)
    ref.step(); opt.step()
    assert max(rel_l2(b, a) for a, b in zip(p1, p2)) < 1e-6


def test_autograd_guards(backbone_rgb):
    """ADVICE round 1: (a) a second forward through the same engine before backward is detected, not silently wrong;
    (b) parameters with hooks (DDP-style) get their gradients through autograd, not the direct .grad shortcut."""
    dev = _cuda()
    import model_zoo
    from ops.ssn_ops import Identity
    net = model_zoo.BNInception()
    net.fc = Identity()
    _load_backbone(net, backbone_rgb, dev).eval()
    x1, x2 = synth.synth_frames(2, 3, seed=1).to(dev), synth.synth_frames(2, 3, seed=2).to(dev)
    o1 = net(x1)
    o2 = net(x2)
    with pytest.raises(RuntimeError, match="another forward"):
        o1.sum().backward()
    o2.sum().backward()
    direct = net.conv1_7x7_s2.weight.grad.clone()
    net.zero_grad()
    seen = []
    h = net.conv1_7x7_s2.weight.register_hook(lambda g: seen.append(float(g.abs().sum())))
    net(x2).sum().backward()
    h.remove()
    assert len(seen) == 1 and seen[0] > 0
    assert rel_l2(net.conv1_7x7_s2.weight.grad, direct) < 1e-6


def test_detect_postprocess_vs_reference(golden_dir):
    """f3: GPU detection post-processing (combined scores, class-wise temporal NMS, location regression) against the
    reference's own outputs (tests/golden/detect.npz): the survivor sets and their order are exact, values to fp32 rounding."""
    dev = _cuda()
    from ops.detection import video_detections, temporal_nms
    z = _load(golden_dir, "detect.npz")
    for tag in "abcd":
        props, act, comp, reg = (torch.tensor(z[tag + k]).to(dev) for k in ("_props", "_act", "_comp", "_reg"))
        thr = float(z[tag + "_thr"])
        K = comp.shape[1]
        det, cnt = video_detections(props, act, comp, reg, thr)
        raw, cnt2 = video_detections(props, act, comp, reg, thr, regress=False)
        assert torch.equal(cnt, cnt2)
        for c in range(K):
            ref_nms, ref_det = z["%s_nms_%d" % (tag, c)], z["%s_det_%d" % (tag, c)]
            n = int(cnt[c])
            assert n == ref_nms.shape[0], (tag, c, n, ref_nms.shape)
            got_raw, got = raw[c, :n].cpu().numpy(), det[c, :n].cpu().numpy()
            np.testing.assert_array_equal(got_raw[:, [0, 1, 3, 4]], ref_nms[:, [0, 1, 3, 4]])     # same boxes, same order
            np.testing.assert_allclose(got_raw[:, 2], ref_nms[:, 2], rtol=2e-6)
            np.testing.assert_allclose(got, ref_det, rtol=2e-6, atol=1e-6)
        # plain temporal_nms on given scores (ops/utils.py:56-82)
        boxes = torch.tensor(z["%s_nms_0" % tag] if False else np.concatenate((z[tag + "_props"], z[tag + "_combined"][:, :1]), axis=1)).to(dev)
        kept = temporal_nms(boxes, thr).cpu().numpy()
        np.testing.assert_array_equal(kept, z["%s_nms_0" % tag][:, :3])


@pytest.mark.parametrize("precision", ["exact", "exact_tc"])
def test_bn_mode_partial(backbone_rgb, precision):
    """f4: bn_mode='partial' -- the first BatchNorm2d in training mode (batch statistics, running-stat update, gradients for
    its weight / bias), everything else frozen (ssn_models.py:95-105,156-174): forward, the updated running statistics and
    the gradients of conv1 / bn1 / a deep layer against the oracle (F.batch_norm(training=True) + autograd)."""
    dev = _cuda()
    import ssn_models
    K = 4
    model = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1), bn_mode="partial")
    sd = model.state_dict()
    for k, v in backbone_rgb.items():
        sd["base_model." + k].copy_(v)
    model = model.to(dev).train()
    model.set_precision(_prec(precision), 1024.0)
    bn1 = model.base_model.conv1_7x7_s2_bn
    assert bn1.training and bn1.weight.requires_grad and not model.base_model.conv2_3x3_bn.training
    x = synth.synth_frames(18, 3, seed=21)
    g = torch.Generator().manual_seed(22)
    dfeat = torch.randn(18, 1024, generator=g) * 0.01
    out = model.base_model(x.to(dev))
    out.backward(dfeat.to(dev))
    bbo = {k: v.clone() for k, v in backbone_rgb.items()}
    for k in bbo:
        if "_bn." not in k or k.startswith("conv1_7x7_s2_bn.weight") or k.startswith("conv1_7x7_s2_bn.bias"):
            bbo[k].requires_grad_(True)
    ref = O.backbone_forward(bbo, x, 3, bn_train_first=True)
    ref.backward(dfeat)
    e_fwd = rel_l2(out.detach(), ref.detach())
    e_rm = rel_l2(bn1.running_mean, bbo["conv1_7x7_s2_bn.running_mean"])
    e_rv = rel_l2(bn1.running_var, bbo["conv1_7x7_s2_bn.running_var"])
    e_g = rel_l2(bn1.weight.grad, bbo["conv1_7x7_s2_bn.weight"].grad)
    e_b = rel_l2(bn1.bias.grad, bbo["conv1_7x7_s2_bn.bias"].grad)
    e_w1 = rel_l2(model.base_model.conv1_7x7_s2.weight.grad, bbo["conv1_7x7_s2.weight"].grad)
    e_w5 = rel_l2(model.base_model.inception_5b_1x1.weight.grad, bbo["inception_5b_1x1.weight"].grad)
    print("bn partial (%s): fwd %.2e running mean %.2e var %.2e dgamma %.2e dbeta %.2e conv1 dW %.2e 5b_1x1 dW %.2e"
          % (precision, e_fwd, e_rm, e_rv, e_g, e_b, e_w1, e_w5))
    assert int(bn1.num_batches_tracked) == 1
    assert e_fwd < E2E_TOL[precision] and e_rm < 1e-5 and e_rv < 1e-5
    # gradients below a 69-layer random-weight net: fp32 noise floor ~1e-2 (test_ssn_train_exact_vs_oracle)
    # measured (exact / exact_tc): dgamma 9e-3 / 1.8e-2, dbeta 8e-3 / 1.7e-2, conv1 dW 1e-2 / 1.6e-2, 5b_1x1 dW 1.6e-3 / 2.0e-3
    assert e_g < 5e-2 and e_b < 5e-2 and e_w1 < 5e-2 and e_w5 < 1e-2, (e_g, e_b, e_w1, e_w5)
    # frozen statistics elsewhere, and eval() freezes the first one too
    assert rel_l2(model.base_model.conv2_3x3_bn.running_mean, backbone_rgb["conv2_3x3_bn.running_mean"]) == 0.0
    model.eval()
    rm = bn1.running_mean.clone()
    with torch.no_grad():
        model.base_model(x.to(dev))
    assert torch.equal(rm, bn1.running_mean)


@pytest.mark.parametrize("precision", ["exact_tc", "fast"])
def test_bucketed_backward_matches_single_call(backbone_rgb, precision):
    """ssnb_backbone_bwd_range (the backward in buckets, for overlapping the gradient all-reduce: ssn_b200.dp.GradSync) leaves
    exactly the gradients of the single-call backward, and the buckets tile the flat gradient buffer."""
    dev = _cuda()
    import ssn_models
    from ssn_b200.optim import FusedSGD
    from ssn_b200.dp import GradSync
    K = 4

    def make():
        m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, stpp_cfg=(1, (1, 2), 1))
        sd = m.state_dict()
        for k, v in backbone_rgb.items():
            sd["base_model." + k].copy_(v)
        m = m.to(dev).train()
        m.set_precision(_prec(precision), 1024.0)
        return m
    torch.manual_seed(7)
    m1 = make()
    torch.manual_seed(7)
    m2 = make()
    batch = [t.to(dev) for t in synth.synth_batch(2, K, 3, seed=5)]
    l1 = m1.fused_step(*batch)
    order = [p for p in m2.parameters() if p.requires_grad]
    opt = FusedSGD(m2.get_optim_policies(), lr=0.0, momentum=0.0, weight_decay=0.0, order=order)
    sync = GradSync(opt.flat_grad, order, m2)
    l2 = m2.fused_step(*batch, grad_sync=sync)
    sync.finish()
    assert torch.equal(l1, l2)
    spans = sorted(sync.launched)
    assert spans[0][0] == 0 and spans[-1][1] == opt.flat_grad.numel() and all(a[1] == b[0] for a, b in zip(spans, spans[1:])), spans
    assert len(spans) == 4                                   # heads + three backbone buckets
    for (n1, p1), (_n2, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        if p1.grad is not None:
            assert torch.equal(p1.grad, p2.grad), n1         # same kernels, same order inside every bucket: bit-identical
