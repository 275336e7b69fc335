"""CPU tests of oracle/schedule_check.py, the float64 per-launch check of the backbone schedule: its graph is the engine's,
a faithful run passes, and planted errors of the kinds a kernel bug makes are caught at the op and quantity they were
planted in.  The "engine" here is BNInception evaluated in fp32 on the CPU with folded weights (autograd for dZ) behind the
engine's read surface, so none of this needs a GPU.  The same holds for the bn_mode='partial' graph (conv1 raw, then a
training-mode BatchNorm + ReLU) and for a forward-only check."""
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
def _engine_plan(in_channels, bn1_train):
    """(ops, {value: shape}) of a CPU-planned engine, through the C ABI"""
    from ssn_b200 import _lib
    cfg = _lib.Config(in_channels, 37, _lib.EXACT_TC, 1, 4096.0, int(bn1_train))
    h = C.c_void_p()
    _lib.check(_lib.lib.ssnb_create(C.byref(cfg), C.byref(h)))
    try:
        k, i, o = C.create_string_buffer(64), C.create_string_buffer(128), C.create_string_buffer(128)
        ops = []
        for n in range(_lib.lib.ssnb_num_ops(h)):
            _lib.check(_lib.lib.ssnb_op_info(h, n, k, 64, i, 128, o, 128), h)
            ops.append((k.value.decode(), i.value.decode(), o.value.decode()))
        shapes = {}
        v = [C.c_int() for _ in range(3)]
        for name in S.Graph(in_channels, bn1_train).shape:
            _lib.check(_lib.lib.ssnb_value_shape(h, name.encode(), *[C.byref(x) for x in v]), h)
            shapes[name] = tuple(x.value for x in v)
        return ops, shapes
    finally:
        _lib.lib.ssnb_destroy(h)


@pytest.mark.parametrize("in_channels", [3, 10])
def test_bn1_graph_matches_engine_plan(in_channels):
    G = S.Graph(in_channels, bn1_train=True)
    ops, shapes = _engine_plan(in_channels, True)
    assert ops == G.engine_ops()
    assert shapes == G.shape
    assert ops[:3] == [("conv", "data", S.BN1_RAW), ("bn", S.BN1_RAW, S.BN1_OUT), ("maxpool", S.BN1_OUT, "pool1_3x3_s2")]
    assert [o["id"] for o in G.ops if o["kind"] == "bn"] == [S.BN1_OUT] and G.conv_ids == S.Graph(in_channels).conv_ids
    assert [o["id"] for o in G.ops if o.get("raw")] == [S.BN1_CONV]


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


MOMENTUM, BN_EPS = 0.1, 1e-5


class _PlantedBatchNormRelu(torch.autograd.Function):
    """relu(BatchNorm2d(z)) in training mode with one planted error: "no_xhat_term" drops xhat * sum(g * xhat) / M from the
    backward; "stats_first_frame" normalises the output with the first frame's statistics (the backward keeps the batch's)"""

    @staticmethod
    def forward(ctx, z, gamma, beta, plant):
        v = lambda t: t.view(1, -1, 1, 1)
        mu, var = z.mean((0, 2, 3)), z.var((0, 2, 3), unbiased=False)
        invstd = 1.0 / torch.sqrt(var + BN_EPS)
        if plant == "stats_first_frame":
            m0, v0 = z[:1].mean((0, 2, 3)), z[:1].var((0, 2, 3), unbiased=False)
            y = F.relu((z - v(m0)) / torch.sqrt(v(v0) + BN_EPS) * v(gamma) + v(beta))
        else:
            y = F.relu((z - v(mu)) * v(invstd) * v(gamma) + v(beta))
        ctx.save_for_backward(z, y, gamma, mu, invstd)
        ctx.plant = plant
        return y

    @staticmethod
    def backward(ctx, dy):
        z, y, gamma, mu, invstd = ctx.saved_tensors
        v = lambda t: t.view(1, -1, 1, 1)
        m = z.numel() // z.shape[1]
        g = dy * (y > 0)
        xh = (z - v(mu)) * v(invstd)
        sb, sg = g.sum((0, 2, 3)), (g * xh).sum((0, 2, 3))
        t = g - v(sb) / m
        if ctx.plant != "no_xhat_term":
            t = t - xh * v(sg) / m
        return v(gamma) * v(invstd) * t, sg, sb, None


class FakeEngine:
    """BNInception in fp32 on the CPU with BN-folded weights, read like a BackboneEngine (EXACT semantics: a conv output's
    gradient buffer holds its masked dZ).  Plants: fwd_nudge {conv id: relative nudge of the last frame}, unmasked {conv id},
    last_max {pool id}.  dfeat None: forward only (no gradient can be read, as with a training=0 engine).
    bn1: bn_mode='partial' -- conv1 raw (no fold, no ReLU), then F.batch_norm(training=True) + ReLU updating the engine's own
    copies of the running statistics; bn1_plant: one of BN1_PLANTS."""

    def __init__(self, params, x, dfeat, in_channels=3, fwd_nudge=None, unmasked=(), last_max=(), bn1=False, bn1_plant=None):
        assert bn1_plant is None or (bn1 and bn1_plant in BN1_PLANTS), bn1_plant
        fwd_nudge = fwd_nudge or {}
        self.G = S.Graph(in_channels, bn1_train=bn1)
        self.frames = x.shape[0]
        self.v, self.z = {"data": x}, {}
        self.wf, self.bf, self.s = [], [], []
        self.backward_ran = dfeat is not None
        d = self.v
        for kind, id_, out, ins, a in O.bninception_ops(in_channels):
            if kind == "conv" and bn1 and id_ == S.BN1_CONV:
                w = params[id_ + ".weight"].clone().requires_grad_(True)
                b = params[id_ + ".bias"].clone().requires_grad_(True)
                self.wf.append(w); self.bf.append(b); self.s.append(torch.ones_like(b))
                z = F.conv2d(d[ins[0]], w, b, a["stride"], a["pad"])
                z.retain_grad()
                self.z[S.BN1_RAW] = z
                d[S.BN1_RAW] = _UnmaskedRelu.apply(z) if bn1_plant == "raw_relu" else z
                d[out] = self._bn1(params, d[S.BN1_RAW], bn1_plant)
                d[out].retain_grad()
                continue
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
        if dfeat is None:
            return
        self.feat.backward(dfeat)
        self.dw = [(w.grad * s.view(-1, 1, 1, 1)).detach() for w, s in zip(self.wf, self.s)]
        self.db = [(b.grad * s).detach() for b, s in zip(self.bf, self.s)]
        if bn1:
            self.dgamma, self.dbeta = self.gamma.grad.detach().clone(), self.beta.grad.detach().clone()
            if bn1_plant == "dgamma_unmasked":          # sum dy * xhat over every pixel, not only where y > 0
                z = d[S.BN1_RAW].detach()
                xh = (z - z.mean((0, 2, 3), keepdim=True)) / torch.sqrt(z.var((0, 2, 3), unbiased=False, keepdim=True) + BN_EPS)
                self.dgamma = (d[S.BN1_OUT].grad * xh).sum((0, 2, 3))
            if bn1_plant == "conv1_dw_fold":            # the frozen BatchNorm's fold scale applied to the raw conv1's dW
                p = lambda k: params[S.BN1_OUT + k]
                self.dw[0] = self.dw[0] * (p(".weight") / torch.sqrt(p(".running_var") + BN_EPS)).view(-1, 1, 1, 1)

    def _bn1(self, params, z, plant):
        p = lambda k: params[S.BN1_OUT + k]
        self.gamma, self.beta = p(".weight").clone().requires_grad_(True), p(".bias").clone().requires_grad_(True)
        self.rm0, self.rv0 = p(".running_mean").clone(), p(".running_var").clone()
        self.rm, self.rv = self.rm0.clone(), self.rv0.clone()
        if plant in ("no_xhat_term", "stats_first_frame"):
            zd = z.detach()
            self.rm = (1 - MOMENTUM) * self.rm0 + MOMENTUM * zd.mean((0, 2, 3))
            self.rv = (1 - MOMENTUM) * self.rv0 + MOMENTUM * zd.var((0, 2, 3), unbiased=True)
            return _PlantedBatchNormRelu.apply(z, self.gamma, self.beta, plant)
        y = F.relu(F.batch_norm(z, self.rm, self.rv, self.gamma, self.beta, True, MOMENTUM, BN_EPS))
        if plant == "momentum_swapped":                 # running <- m * running + (1 - m) * batch
            zd = z.detach()
            self.rm = MOMENTUM * self.rm0 + (1 - MOMENTUM) * zd.mean((0, 2, 3))
            self.rv = MOMENTUM * self.rv0 + (1 - MOMENTUM) * zd.var((0, 2, 3), unbiased=True)
        return y

    def bn1_state(self):
        """the `bn1` argument of check_schedule"""
        st = dict(gamma=self.gamma.detach(), beta=self.beta.detach(), momentum=MOMENTUM, eps=BN_EPS,
                  running_mean0=self.rm0, running_var0=self.rv0, running_mean=self.rm, running_var=self.rv)
        if self.backward_ran:
            st.update(dgamma=self.dgamma, dbeta=self.dbeta)
        return st

    def ops(self):
        return self.G.engine_ops()

    def value_shape(self, name):
        return self.G.shape[name]

    def read(self, name, grad=False, planes=False):
        assert not planes, "fp32 stand-in: no operand planes"
        assert self.backward_ran or not grad, "forward-only engine: no gradient buffers"
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


@pytest.mark.parametrize("k,s,p,size", [(3, 2, 0, 7), (3, 2, 0, 8), (3, 1, 1, 7), (2, 1, 0, 5)])
def test_max_pool_route_matches_aten_on_ties_and_non_finite(k, s, p, size):
    """the route is float64 autograd of F.max_pool2d (ceil mode) on windows full of exact ties (+-0 among them), with two
    NaNs in one window (the LAST one takes the gradient), NaN beside +-inf, and windows of -inf only"""
    gen = torch.Generator().manual_seed(size * 10 + k + s + p)
    vals = torch.tensor([-1.0, -0.5, -0.0, 0.0, 0.5, 1.0], dtype=torch.float64)
    x = vals[torch.randint(0, len(vals), (2, 3, size, size), generator=gen)]
    nan, inf = float("nan"), float("inf")
    x[0, 0, 0, 0] = x[0, 0, 1, 1] = nan                 # two NaNs in the first window
    x[0, 1, 0, 1], x[0, 1, 1, 0] = inf, nan              # NaN after +inf
    x[0, 2, 0, 0], x[0, 2, 0, 1] = nan, -inf             # NaN before -inf
    x[1, 0, :3, :3] = -inf                               # a window of -inf only (with padding around it at p = 1)
    x[1, 1, -2:, -2:] = -inf                             # the partial last window
    x[1, 2, -1, -1], x[1, 2, -1, 0], x[1, 2, 0, -1] = nan, nan, inf   # poison in the last row and column
    x[1, 2, 2, 2] = inf
    x[1, 2, 2, 3 % size] = inf                           # tied +inf
    xr = x.clone().requires_grad_(True)
    y = F.max_pool2d(xr, k, s, p, ceil_mode=True)
    g = torch.randint(1, 9, y.shape, generator=gen).double()
    y.backward(g)
    d = S.maxpool_route(x, g, k, s, p)
    assert torch.equal(d, xr.grad), (d - xr.grad).abs().nonzero()[:8]


# ---- forward-only and bn_mode='partial' ---------------------------------------------------------------------------------
BN1_PLANTS = {      # planted error -> the one record that must fail
    "no_xhat_term": (S.BN1_CONV, "dZ"),             # BatchNorm backward without xhat * sum(g * xhat) / M
    "dgamma_unmasked": (S.BN1_OUT, "dgamma"),       # dgamma summed over dy instead of dy * (y > 0)
    "momentum_swapped": None,                       # momentum on the batch side: both running statistics
    "conv1_dw_fold": (S.BN1_CONV, "dW"),            # the raw conv1's dW still multiplied by the frozen fold scale
    "raw_relu": (S.BN1_CONV, "fwd"),                # a ReLU on the raw conv1 output
    "stats_first_frame": (S.BN1_OUT, "fwd"),        # batch statistics of the first frame only
}


def _check_bn1(eng, params, x, dfeat):
    return S.check_schedule(eng, params, x, eng.feat.detach(), dfeat, eng.dw, eng.db, "exact", bars=BARS, bn1=eng.bn1_state())


@pytest.fixture(scope="module")
def clean_bn1(case):
    params, x, dfeat = case
    return FakeEngine(params, x, dfeat, bn1=True)


def _n_fwd(G):
    return sum(o["kind"] != "gpool" for o in G.ops) + 1


def test_forward_only_passes(case):
    params, x, _dfeat = case
    for bn1 in (False, True):
        eng = FakeEngine(params, x, None, bn1=bn1)
        recs = S.check_schedule(eng, params, x, eng.feat.detach(), precision="exact", bars=BARS,
                                bn1=eng.bn1_state() if bn1 else None)
        # one fwd record per op; no gradient was read (the stand-in asserts that)
        assert len(recs) == _n_fwd(S.Graph(3, bn1)) and {r.quantity for r in recs} == {"fwd"}
        assert not S.failures(recs), S.failures(recs)


def test_bn1_clean_run_passes(case, clean_bn1):
    params, x, dfeat = case
    recs = _check_bn1(clean_bn1, params, x, dfeat)
    G = S.Graph(3, bn1_train=True)
    n_conv, n_pool = len(G.conv_ids), sum(o["kind"] in ("maxpool", "avgpool") for o in G.ops)
    # fwd for every op + 2 running statistics; dZ for every conv; G for every pool and the BatchNorm output; dgamma, dbeta;
    # dW + db for every conv
    assert len(recs) == (_n_fwd(G) + 2) + n_conv + (n_pool + 1) + 2 + 2 * n_conv
    print("worst records:", *S.worst(recs), sep="\n  ")
    assert not S.failures(recs), S.failures(recs)
    by = {(r.op, r.quantity): r for r in recs}
    assert by[(S.BN1_CONV, "dZ")].consumers == (S.BN1_OUT,) and by[(S.BN1_OUT, "G")].consumers == ("pool1_3x3_s2",)
    # the running statistics moved, and the raw output has negative values (no ReLU hides there)
    assert not torch.allclose(clean_bn1.rm, clean_bn1.rm0) and bool((clean_bn1.read(S.BN1_RAW) < 0).any())


@pytest.mark.parametrize("plant", sorted(BN1_PLANTS))
def test_bn1_planted_error(case, plant):
    params, x, dfeat = case
    eng = FakeEngine(params, x, dfeat, bn1=True, bn1_plant=plant)
    recs = _check_bn1(eng, params, x, dfeat)
    want = BN1_PLANTS[plant]
    want = {(S.BN1_OUT, "running_mean"), (S.BN1_OUT, "running_var")} if want is None else {want}
    assert _failed(recs) == want, S.failures(recs)
