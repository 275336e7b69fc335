"""CPU tests of oracle/step_check.py, the float64 check of the SSN step's tail (fused pool + STPP, heads + multi-task loss,
STPP backward, momentum SGD): an fp32 torch stand-in for those kernels passes, and planted errors of the kinds a kernel bug
makes are reported at the op and quantities they were planted in, and nowhere else.  The heads stand-in is written with
autograd over the reference's loss formulation (oracle/ssn_oracle.py), independently of heads_loss64."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ssn_oracle as O
from oracle import step_check as S

SEG = (2, 5, 2)
TABLE = S.part_table((1, (1, 2), 1), [2, 7, 9])
COURSE = (2, 7)
COMP_QUANTITIES = {("heads", q) for q in ("loss_comp", "loss_total", "d_comp_w", "d_comp_b", "d_stpp")}


# ---- fp32 stand-ins for the kernels --------------------------------------------------------------------------------------
def _pool_stpp32(y5b, mask, scaling, plant=None):
    """gpool_stpp: feat = pixel mean * mask, course / stpp of feat.  plant: "pixels48" pools 48 of the 49 pixels;
    "mask_feat_only" applies the mask to feat but forms course / stpp from the unmasked pooled values"""
    px = y5b.flatten(2)
    pooled = px[..., :48].mean(2) if plant == "pixels48" else px.mean(2)
    feat = pooled * mask
    course, stpp = O.stpp_forward(pooled if plant == "mask_feat_only" else feat, scaling, [2, 7, 9])
    return feat, course, stpp


def _heads32(case, cfg=None, plant=None):
    """the heads + loss call in fp32 with autograd: F.linear heads, cross entropy, OHEM completeness and class-wise
    regression (ops/ssn_ops.py:173-258); gradients are those of loss_scale * total.  plant: "ohem_smallest" keeps the
    smallest negatives; "bias_unscaled" leaves loss_scale out of the three bias gradients; "dcourse_last_row" drops the
    last row's d_course"""
    cfg = cfg or case["cfg"]
    K, G, P, s = cfg["num_class"], cfg["comp_group"], cfg["fg_per_video"], cfg["loss_scale"]
    xc = case["course"].clone().requires_grad_(True)
    xs = case["stpp"].clone().requires_grad_(True)
    hp = {k: v.clone().requires_grad_(True) for k, v in case["heads"].items()}
    pt, tg, rt = case["prop_type"], case["target"], case["reg_target"]
    ra = F.linear(xc, hp["activity_fc.weight"], hp["activity_fc.bias"])
    rc = F.linear(xs, hp["completeness_fc.weight"], hp["completeness_fc.bias"])
    rr = F.linear(xs, hp["regressor_fc.weight"], hp["regressor_fc.bias"])
    ai, ci, ri = ((pt == 0) | (pt == 2)).nonzero().view(-1), ((pt == 0) | (pt == 1)).nonzero().view(-1), (pt == 0).nonzero().view(-1)
    la = F.cross_entropy(ra[ai], tg[ai])
    z = rc[ci, (tg[ci] - 1) % K].view(-1, G)
    lp, ln = (1 - z[:, :P]).clamp_min(0), (1 + z[:, P:]).clamp_min(0)
    pick = ln.detach().sort(1, descending=plant != "ohem_smallest").indices[:, :cfg["keep_neg"]]
    lc = (lp.sum() + ln.gather(1, pick).sum()) / cfg["comp_denom"]
    lr = O.classwise_regression_loss(rr.view(-1, K, 2)[ri], tg[ri], rt[ri])
    total = la + lc * cfg["comp_w"] + lr * cfg["reg_w"]
    (total * s).backward()
    out = {"raw_act": ra.detach(), "raw_comp": rc.detach(), "raw_reg": rr.detach(),
           "losses": torch.stack([la, lc, lr, total]).detach(), "d_course": xc.grad, "d_stpp": xs.grad}
    for k, nm in (("act", "activity_fc"), ("comp", "completeness_fc"), ("reg", "regressor_fc")):
        out["d_%s_w" % k] = hp[nm + ".weight"].grad
        out["d_%s_b" % k] = hp[nm + ".bias"].grad / (s if plant == "bias_unscaled" else 1.0)
    if plant == "dcourse_last_row":
        out["d_course"] = out["d_course"].clone()
        out["d_course"][-1] = 0
    return out


def _ref(case, cfg=None):
    return S.heads_loss64(case["course"], case["stpp"], case["heads"], case["prop_type"], case["target"], case["reg_target"],
                          cfg or case["cfg"])


# ---- fixtures ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pool_case():
    g = torch.Generator().manual_seed(5)
    F_ = 4 * 9
    y5b = torch.randn(F_, 1024, 7, 7, generator=g).clamp_min(0)
    mask = torch.bernoulli(torch.full((F_, 1024), 0.2), generator=g) / 0.2
    scaling = torch.rand(4, 2, generator=g)
    return y5b, mask, scaling


@pytest.fixture(scope="module")
def case40():
    """5 videos = 40 rows (a 32-row pass and a tail of 8), loss_scale 0.5"""
    return S.heads_case(5, 20, 5, seed=1, loss_scale=0.5)


@pytest.fixture(scope="module")
def case64():
    """64 global videos, K = 20, M = 5"""
    return S.heads_case(64, 20, 5, seed=2)


def _check_pool(pool_case, plant=None):
    y5b, mask, scaling = pool_case
    feat, course, stpp = _pool_stpp32(y5b, mask, scaling, plant)
    chk = S.Checker()
    S.check_pool_stpp(chk, "pool_stpp", y5b, mask, scaling, TABLE, 9, COURSE, feat, course, stpp)
    return chk


def _check_heads(case, out, cfg=None):
    chk = S.Checker()
    S.check_heads(chk, "heads", out, _ref(case, cfg))
    return chk


# ---- the stand-ins pass --------------------------------------------------------------------------------------------------
def test_pool_stpp_standin_passes(pool_case):
    chk = _check_pool(pool_case)
    assert [r.key for r in chk.records] == [("pool_stpp", q) for q in ("feat", "course", "stpp")]
    chk.assert_ok()
    # the reference follows the part table: the 5 parts of (1, (1, 2), 1) over 2 + 5 + 2 segments
    assert TABLE == ([0, 2, 2, 4, 7], [2, 7, 4, 7, 9], [1, 3, 3, 3, 1], [0, -1, -1, -1, 1])


def test_heads_standin_passes(case40, case64):
    for case in (case40, case64):
        chk = _check_heads(case, _heads32(case))
        assert len(chk.records) == 5 + 6 + 4
        print(chk.report())
        chk.assert_ok()
    # the same arithmetic as the reference's criteria at world 1 (the fp32 oracle pinned to the reference's golden losses)
    c = case40
    ref = _ref(c, S.heads_cfg(40, 8, 20, 5))
    pt, tg = c["prop_type"], c["target"]
    ra, rc = ref["raw_act"].float(), ref["raw_comp"].float()
    rr = ref["raw_reg"].float().view(-1, 20, 2)
    ai, ci, ri = ((pt == 0) | (pt == 2)).nonzero().view(-1), ((pt == 0) | (pt == 1)).nonzero().view(-1), (pt == 0).nonzero().view(-1)
    loss, parts = O.total_loss((ra[ai], tg[ai], rc[ci], tg[ci], rr[ri], tg[ri], c["reg_target"][ri]))
    got = ref["losses"].float()
    want = torch.stack([v.reshape(()) for v in list(parts) + [loss]]).detach()
    assert torch.allclose(got, want, rtol=1e-6), (got, want)


def test_heads_cfg_matches_the_data_parallel_split():
    from ssn_b200 import dp
    full, shard = S.heads_cfg(512, 8, 20, 5), S.heads_cfg(256, 8, 20, 5, global_videos=64, loss_scale=0.5)
    assert full["comp_denom"] == dp.completeness_denominator(64) == 129 and full["keep_neg"] == 1
    assert (shard["comp_denom"], shard["loss_scale"]) == dp.shard_loss_config(64, 2) == (64.5, 0.5)
    assert S.heads_cfg(256, 8, 20, 5)["comp_denom"] == 64


def test_stpp_vjp_and_sgd_standins_pass():
    g = torch.Generator().manual_seed(6)
    n, D = 3, 1024
    sc = torch.rand(n, 2, generator=g)
    ft = torch.randn(n * 9, D, generator=g, requires_grad=True)
    course, stpp = O.stpp_forward(ft, sc, [2, 7, 9])
    dc, ds = torch.randn(n, D, generator=g), torch.randn(n, 5 * D, generator=g)
    torch.autograd.backward([course, stpp], [dc, ds])
    chk = S.Checker()
    chk.add("stpp_bwd", "dft", ft.grad, S.stpp_vjp64(dc, ds, sc, TABLE, 9, COURSE), S.STPP_BWD_BAR, rows=True)
    # SGD: three parameter tensors with their own lr / wd, against torch.optim.SGD
    ps = [torch.randn(s, generator=g) for s in (5, 7, 3)]
    grads = [torch.randn(p.shape, generator=g) for p in ps]
    lrs, wds = [0.1, 0.2, 0.1], [5e-4, 0.0, 5e-4]
    tp = [p.clone().requires_grad_(True) for p in ps]
    opt = torch.optim.SGD([{"params": [p], "lr": lr, "weight_decay": wd} for p, lr, wd in zip(tp, lrs, wds)], lr=0.1, momentum=0.9)
    for p, gr in zip(tp, grads):
        p.grad = gr.clone()
    opt.step()
    opt.step()                         # a second step from a non-zero momentum
    buf0 = torch.cat([opt.state[p]["momentum_buffer"] for p in tp])
    p1 = torch.cat([p.detach() for p in tp])
    for p, gr in zip(tp, grads):
        p.grad = gr.clone()
    opt.step()
    seg_end = torch.tensor([5, 12, 15])
    rp, rb = S.sgd64(p1, torch.cat(grads), buf0, seg_end, torch.tensor(lrs), torch.tensor(wds), 0.9)
    S.check_sgd(chk, "sgd", seg_end, torch.cat([p.detach() for p in tp]), torch.cat([opt.state[p]["momentum_buffer"] for p in tp]), rp, rb)
    print(chk.report())
    chk.assert_ok()
    # a wrong learning rate on one segment is caught
    bad = S.Checker()
    rp2, rb2 = S.sgd64(p1, torch.cat(grads), buf0, seg_end, torch.tensor([0.1, 0.1, 0.1]), torch.tensor(wds), 0.9)
    S.check_sgd(bad, "sgd", seg_end, torch.cat([p.detach() for p in tp]), torch.cat([opt.state[p]["momentum_buffer"] for p in tp]), rp2, rb2)
    assert bad.failed() == {("sgd", "param")}, bad.report()


# ---- planted errors ------------------------------------------------------------------------------------------------------
def test_planted_pooling_over_48_pixels(pool_case):
    chk = _check_pool(pool_case, "pixels48")
    assert chk.failed() == {("pool_stpp", "feat")}, chk.report()


def test_planted_mask_on_feat_only(pool_case):
    chk = _check_pool(pool_case, "mask_feat_only")
    assert chk.failed() == {("pool_stpp", "course"), ("pool_stpp", "stpp")}, chk.report()


def test_planted_shard_completeness_denominator(case64):
    """64 global videos in two shards: each shard must divide by its share of the global denominator, (64 + int(64 * 6 * 0.17))
    / 2 = 64.5; a shard that uses its own, 32 + int(32 * 6 * 0.17) = 64, is off in the completeness loss and gradients"""
    rows = slice(0, 256)
    shard = {k: (v[rows] if torch.is_tensor(v) and k != "heads" else v) for k, v in case64.items()}
    cfg = S.heads_cfg(256, 8, 20, 5, global_videos=64, loss_scale=0.5)
    own = S.heads_cfg(256, 8, 20, 5, loss_scale=0.5)
    assert cfg["comp_denom"] == 64.5 and own["comp_denom"] == 64
    _check_heads(shard, _heads32(shard, cfg), cfg).assert_ok()
    chk = _check_heads(shard, _heads32(shard, own), cfg)
    assert chk.failed() == COMP_QUANTITIES, chk.report()


def test_planted_ohem_keeps_smallest(case40):
    chk = _check_heads(case40, _heads32(case40, plant="ohem_smallest"))
    assert chk.failed() == COMP_QUANTITIES, chk.report()


def test_planted_bias_gradients_without_loss_scale(case40):
    assert case40["cfg"]["loss_scale"] == 0.5
    chk = _check_heads(case40, _heads32(case40, plant="bias_unscaled"))
    assert chk.failed() == {("heads", "d_act_b"), ("heads", "d_comp_b"), ("heads", "d_reg_b")}, chk.report()


def test_planted_dcourse_tail_row(case40):
    """the last row of 40 is the tail of the second 32-row pass"""
    chk = _check_heads(case40, _heads32(case40, plant="dcourse_last_row"))
    assert chk.failed() == {("heads", "d_course")}, chk.report()
    (r,) = chk.failures()
    assert r.where == "row 39" and r.err == 1.0


def test_ohem_gap_and_tie_rule():
    """the float64 OHEM keeps the largest negative hinge losses, the lower index first among equal ones"""
    cfg = S.heads_cfg(8, 8, 2, 1, fg_per_video=1, comp_group=7, ohem_ratio=0.34)        # keep int(6 * 0.34) = 2
    assert cfg["keep_neg"] == 2
    pt = torch.tensor([0, 1, 1, 1, 1, 1, 1, 2])
    tg = torch.tensor([1, 1, 1, 1, 1, 1, 1, 0])
    raw = torch.zeros(8, 2, dtype=torch.float64)
    raw[1:7, 0] = torch.tensor([0.5, -0.2, 0.5, 0.1, 0.5, -3.0], dtype=torch.float64)     # hinge 1.5, 0.8, 1.5, 1.1, 1.5, 0
    assert S.ohem_gap(raw, pt, tg, cfg) == 0.0
    heads = {k: torch.zeros(s) for k, s in (("activity_fc.weight", (3, 128)), ("activity_fc.bias", (3,)),
                                            ("completeness_fc.weight", (2, 128)), ("regressor_fc.weight", (4, 128)),
                                            ("regressor_fc.bias", (4,)))}
    heads["completeness_fc.bias"] = torch.zeros(2)
    xs = torch.zeros(8, 128)
    xs[:, 0] = raw[:, 0].float()
    heads["completeness_fc.weight"][0, 0] = 1.0
    ref = S.heads_loss64(torch.zeros(8, 128), xs, heads, pt, tg, torch.zeros(8, 2), dict(cfg, feat_dim=128, comp_w=1.0))
    d = ref["d_stpp"][:, 0] * cfg["comp_denom"]
    # rows 1 and 3 (the first two of the three tied 1.5 losses) are kept; the positive row 0 (hinge 1) gets -1
    assert torch.allclose(d, torch.tensor([-1.0, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0], dtype=torch.float64), rtol=0, atol=1e-12), d
