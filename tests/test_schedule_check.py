"""CPU tests of oracle/schedule_check.py, the float64 per-launch check of the backbone schedule: its graph is the engine's,
a faithful run passes, and planted errors of the kinds a kernel bug makes are caught at the op and quantity they were
planted in.  The "engine" here is BNInception evaluated in fp32 on the CPU with folded weights (autograd for dZ) behind the
engine's read surface, so none of this needs a GPU."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import schedule_check as S
from oracle import ssn_oracle as O
from oracle import synth

FRAMES = 2
BARS = (1e-5, 1e-4)      # the EXACT starting bars: what is planted must be caught even at these


# ---- the checker's graph is the engine's --------------------------------------------------------------------------------
@pytest.mark.parametrize("in_channels", [3, 10])
def test_graph_matches_engine_plan(in_channels):
    from ssn_b200 import _lib
    cfg = _lib.Config(in_channels, 37, _lib.EXACT_TC, 1, 4096.0)
    h = C.c_void_p()
    _lib.check(_lib.lib.ssnb_create(C.byref(cfg), C.byref(h)))
    try:
        k, i, o = C.create_string_buffer(64), C.create_string_buffer(128), C.create_string_buffer(128)
        ops = []
        for n in range(_lib.lib.ssnb_num_ops(h)):
            _lib.check(_lib.lib.ssnb_op_info(h, n, k, 64, i, 128, o, 128), h)
            ops.append((k.value.decode(), i.value.decode(), o.value.decode()))
        G = S.Graph(in_channels)
        assert ops == G.engine_ops()
        v = [C.c_int() for _ in range(3)]
        for name, shape in G.shape.items():
            _lib.check(_lib.lib.ssnb_value_shape(h, name.encode(), *[C.byref(x) for x in v]), h)
            assert tuple(x.value for x in v) == shape, name
        assert [o["id"] for o in G.ops if o["kind"] == "conv"] == [r[0] for r in O.conv_layers(in_channels)]
        assert sum(len(m) for m in G.members.values()) == len(G.branch) == 8 * 4 + 2 * 3
    finally:
        _lib.lib.ssnb_destroy(h)


# ---- a CPU stand-in for the engine ----------------------------------------------------------------------------------------
class _UnmaskedRelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        return z.clamp_min(0)

    @staticmethod
    def backward(ctx, g):
        return g


class _LastMaxPool(torch.autograd.Function):
    """max pool whose backward routes to the LAST maximum of a tied window"""

    @staticmethod
    def forward(ctx, x, a):
        ctx.save_for_backward(x)
        ctx.a = a
        return O._pool(x, a)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        k, s, p = ctx.a["k"], ctx.a["stride"], ctx.a["pad"]
        n, c, h, w = x.shape
        oh, ow = g.shape[2:]
        hp, wp = (oh - 1) * s + k, (ow - 1) * s + k
        xp = F.pad(x, (p, wp - w - p, p, hp - h - p), value=-float("inf"))
        cols = F.unfold(xp, k, stride=s).view(n, c, k * k, oh * ow)
        last = k * k - 1 - cols.flip(2).argmax(2, keepdim=True)
        routed = torch.zeros_like(cols).scatter_(2, last, g.reshape(n, c, 1, oh * ow))
        return F.fold(routed.view(n, c * k * k, oh * ow), (hp, wp), k, stride=s)[:, :, p:p + h, p:p + w], None


class FakeEngine:
    """BNInception in fp32 on the CPU with BN-folded weights, read like a BackboneEngine (EXACT semantics: a conv output's
    gradient buffer holds its masked dZ).  Plants: fwd_nudge {conv id: relative nudge of the last frame}, unmasked {conv id},
    last_max {pool id}."""

    def __init__(self, params, x, dfeat, in_channels=3, fwd_nudge=None, unmasked=(), last_max=()):
        fwd_nudge = fwd_nudge or {}
        self.G = S.Graph(in_channels)
        self.frames = x.shape[0]
        self.v, self.z = {"data": x}, {}
        self.wf, self.bf, self.s = [], [], []
        d = self.v
        for kind, id_, out, ins, a in O.bninception_ops(in_channels):
            if kind == "conv":
                s = params[id_ + "_bn.weight"] / torch.sqrt(params[id_ + "_bn.running_var"] + 1e-5)
                w = (params[id_ + ".weight"] * s.view(-1, 1, 1, 1)).requires_grad_(True)
                b = ((params[id_ + ".bias"] - params[id_ + "_bn.running_mean"]) * s + params[id_ + "_bn.bias"]).requires_grad_(True)
                self.wf.append(w); self.bf.append(b); self.s.append(s)
                z = F.conv2d(d[ins[0]], w, b, a["stride"], a["pad"])
                z.retain_grad()
                self.z[out] = z
                y = _UnmaskedRelu.apply(z) if id_ in unmasked else F.relu(z)
                if id_ in fwd_nudge:
                    delta = torch.zeros_like(y)
                    delta[-1] = y[-1].detach() * fwd_nudge[id_]
                    y = y + delta
                d[out] = y
            elif kind == "pool" and id_ == "global_pool":
                self.feat = d[ins[0]].mean((2, 3))
                continue
            elif kind == "pool":
                d[out] = _LastMaxPool.apply(d[ins[0]], a) if id_ in last_max else O._pool(d[ins[0]], a)
            elif kind == "concat":
                d[out] = torch.cat([d[i] for i in ins], 1)
            else:
                continue
            d[out].retain_grad()
        self.feat.backward(dfeat)
        self.dw = [(w.grad * s.view(-1, 1, 1, 1)).detach() for w, s in zip(self.wf, self.s)]
        self.db = [(b.grad * s).detach() for b, s in zip(self.bf, self.s)]

    def ops(self):
        return self.G.engine_ops()

    def value_shape(self, name):
        return self.G.shape[name]

    def read(self, name, grad=False, planes=False):
        assert not planes, "fp32 stand-in: no operand planes"
        if name in self.G.members and grad:
            return torch.cat([self.read(m, grad=True) for m in self.G.members[name]], 1)
        if grad:
            t = self.z[name].grad if name in self.z else self.v[name].grad
        else:
            t = self.v[name]
        return t.detach().clone()


@pytest.fixture(scope="module")
def case():
    params = synth.synth_backbone(3, seed=0, calib_frames=2)
    x = synth.synth_frames(FRAMES, 3, seed=3)
    # a band of rows that is constant along the width: conv1's outputs repeat along a row there, so pool1 sees windows whose
    # maximum is tied between columns (the routing rule is exercised, and a wrong one is visible)
    x[:, :, 96:160, :] = x[:, :, 96:160, :1]
    dfeat = torch.randn(FRAMES, 1024, generator=torch.Generator().manual_seed(9)) * 0.01
    return params, x, dfeat


@pytest.fixture(scope="module")
def clean(case):
    params, x, dfeat = case
    return FakeEngine(params, x, dfeat)


def _check(eng, params, x, dfeat, dw=None, db=None):
    return S.check_schedule(eng, params, x, eng.feat.detach(), dfeat, dw or eng.dw, db or eng.db, "exact", bars=BARS)


def _failed(recs):
    return {(r.op, r.quantity) for r in S.failures(recs)}


def test_clean_run_passes(case, clean):
    params, x, dfeat = case
    recs = _check(clean, params, x, dfeat)
    G = S.Graph(3)
    n_conv, n_pool = len(G.conv_ids), sum(o["kind"] in ("maxpool", "avgpool") for o in G.ops)
    # fwd for every op; dZ for every conv; G for every pool output; dW + db for every conv
    assert len(recs) == (n_conv + n_pool + 1) + n_conv + n_pool + 2 * n_conv
    print("worst records:", *S.worst(recs), sep="\n  ")
    assert not S.failures(recs), S.failures(recs)
    # the tied windows of pool1 exist, at positive values (where the routing decides a gradient)
    y = clean.read("conv1_7x7_s2_bn")[:, :, 50:78, 4:108]
    assert bool(((y[..., 1:] == y[..., :-1]) & (y[..., 1:] > 0)).any())


def test_planted_weight_gradient_slice(case, clean):
    params, x, dfeat = case
    i = S.Graph(3).conv_ids.index("inception_4a_3x3")
    dw = list(clean.dw)
    dw[i] = dw[i].clone()
    dw[i][64:128] *= 1 + 1e-3
    recs = _check(clean, params, x, dfeat, dw=dw)
    assert _failed(recs) == {("inception_4a_3x3", "dW")}, S.failures(recs)
    (r,) = S.failures(recs)
    assert r.worst_slice == 1 and "inception_4a_3x3 dW" in repr(r)


def test_planted_forward_nudge_last_frame(case):
    params, x, dfeat = case
    eng = FakeEngine(params, x, dfeat, fwd_nudge={"inception_3b_3x3": 1e-4})
    recs = _check(eng, params, x, dfeat)
    assert _failed(recs) == {("inception_3b_3x3", "fwd")}, S.failures(recs)
    (r,) = S.failures(recs)
    assert r.worst_frame == FRAMES - 1 and r.cell[0] == FRAMES - 1


def test_planted_unmasked_dz(case):
    params, x, dfeat = case
    eng = FakeEngine(params, x, dfeat, unmasked={"inception_4c_double_3x3_1"})
    recs = _check(eng, params, x, dfeat)
    assert _failed(recs) == {("inception_4c_double_3x3_1", "dZ")}, S.failures(recs)


def test_planted_max_pool_last_maximum(case):
    params, x, dfeat = case
    eng = FakeEngine(params, x, dfeat, last_max={"pool1_3x3_s2"})
    recs = _check(eng, params, x, dfeat)
    # pool1's backward is the only contribution to conv1's output gradient (the engine folds it into conv1's mask pass)
    assert _failed(recs) == {("conv1_7x7_s2", "dZ")}, S.failures(recs)
    (r,) = S.failures(recs)
    assert r.consumers == ("pool1_3x3_s2",) and "via pool1_3x3_s2" in repr(r)


def test_planted_bias_gradient_dropped_pixel_range(case, clean):
    params, x, dfeat = case
    ids = S.Graph(3).conv_ids
    i = ids.index("inception_5a_1x1")
    dz = clean.read("inception_5a_1x1_bn", grad=True)                 # [F, C, 7, 7]
    rows = dz.permute(0, 2, 3, 1).reshape(-1, dz.shape[1])             # pixels x channels, the split-K order
    db = list(clean.db)
    db[i] = db[i] - rows[40:60].sum(0) * clean.s[i]                    # one split's partial (20 pixels) never added
    recs = _check(clean, params, x, dfeat, db=db)
    assert _failed(recs) == {("inception_5a_1x1", "db")}, S.failures(recs)


def test_planted_bias_gradient_without_bn_scale(case, clean):
    params, x, dfeat = case
    i = S.Graph(3).conv_ids.index("conv2_3x3")
    db = list(clean.db)
    db[i] = db[i] / clean.s[i]
    recs = _check(clean, params, x, dfeat, db=db)
    assert _failed(recs) == {("conv2_3x3", "db")}, S.failures(recs)


def test_max_pool_route_rule():
    """first maximum in row-major tap order, NaN wins, padding never wins; overlapping windows add"""
    x = torch.tensor([[[[1.0, 3.0, 3.0], [0.0, 3.0, 2.0], [float("nan"), 0.0, 5.0]]]], dtype=torch.float64)
    g = torch.ones(1, 1, 2, 2, dtype=torch.float64)
    d = S.maxpool_route(x, g, 2, 1, 0)
    want = torch.tensor([[[[0.0, 2.0, 0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 1.0]]]], dtype=torch.float64)
    assert torch.equal(d, want), d
    # ceil mode: the partial last window of a 3/2 pool over 4 columns
    x = torch.arange(16, dtype=torch.float64).view(1, 1, 4, 4)
    d = S.maxpool_route(x, torch.ones(1, 1, 2, 2, dtype=torch.float64), 3, 2, 0)
    assert d[0, 0, 2, 2] == 1 and d[0, 0, 2, 3] == 1 and d[0, 0, 3, 2] == 1 and d[0, 0, 3, 3] == 1 and d.sum() == 4
