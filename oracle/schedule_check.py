"""Float64 check of every launch of the backbone's forward + backward schedule.  TEST INFRASTRUCTURE ONLY.

After one `forward` + `backward` of a `BackboneEngine`, every op is checked LOCALLY: the float64 reference of the op is fed
the operands the engine's kernels actually consumed (read back through `read`), so one layer's rounding never reaches the
next and no ReLU or max-pool decision can differ between the engine and the reference.  That makes a per-launch bar as
tight as a per-layer test possible on the production schedule (fused sibling launches, last-writer masking, folded pool
backward, batched weight-gradient finalize, conv1 fed straight from the caller's NCHW input) at any frame count.

Consumed representation, per precision:
  exact     the fp32 values and gradients;
  exact_tc  the hi + lo fp16 operand planes (`read(name, planes=True)`, `read(name, grad=True, planes=True)`) for what
            the convolutions read; fp32 for what only pools and masks read;
  fast      the fp16 storage (`read` un-scales gradients by grad_scale);
  conv1 reads the caller's input x (fast: x rounded to fp16).

Checks (one `Record` each):
  fwd     conv: relu(conv64(X, W', b')); max pool: bitwise; avg pool: to the rounding of the stored result;
          global pool: the 7x7 mean of the last block's output;
          bn_mode='partial' (bn1): conv1 is conv64(X, W, b) without fold and ReLU, and its training-mode BatchNorm + ReLU
          is relu(gamma * xhat + beta) with float64 batch statistics of the consumed z;
  planes  exact_tc: the activation planes of every conv / pool output against its fp32 value;
  dZ      a conv output V: (Y > 0) * G_V against the dZ its backward consumed, where G_V is the sum over V's consumers of
          the vjp of each applied to ITS consumed output gradient (a branch of a concat takes its slice of the block
          output's G; the global pool contributes dfeat / 49);
  G       any other value: G_V against the stored gradient (a max-pool branch of a concat under its own ReLU mask, which
          the last writer of the block output's gradient may apply);
  dW, db  s * wgrad64(X, dZ) and s * sum(dZ) against what the engine returned in reference layout, s = gamma / sqrt(var + eps)
          (s = 1 for the raw conv1 of bn1, whose db, a sum that vanishes, is measured against sum |dZ|);
  bn1     conv1's dZ is the BatchNorm vjp of the consumed dy masked by the engine's own y > 0 (no further ReLU mask), with
          sum g and sum g * xhat taken over all frames first; dgamma / dbeta; running_mean / running_var: one momentum step
          from the statistics held before the forward (unbiased variance).

Forward-only (dfeat None, e.g. an engine created with training=0): the fwd and planes records only; no gradient is read.

Besides the tensor-wide rel-L2, every record keeps rel-L2 per frame and per 64-output-channel slice; the worst frame and
the worst slice are held to SLICE_FACTOR x the tensor bar, so an error confined to one tile is not averaged away.

Only the public surface of an engine is used: `ops()`, `value_shape(name)`, `read(name, grad, planes)`, the feat the
forward returned and the dw / db lists the backward filled.  Device-agnostic torch, float64, evaluated op by op and in
frame chunks so that the memory on top of the engine's workspace stays within a few GB.
"""
import math

import torch
import torch.nn.functional as F

from . import ssn_oracle as O

# tensor-wide rel-L2 bars: fwd / dZ / G, and dW / db.  Worst measured on an H100 80GB HBM3 (700 W) at F = 288, 37 and 1
# (tests/test_gpu_schedule.py): exact 1.1e-6 / 4.7e-7 (F = 37), exact_tc 3.1e-6 / 1.1e-4 (conv2_3x3 dW at F = 288),
# fast 9.9e-4 / 9.7e-5.  The bars are about 4x those, or the per-layer bars where 4x would be looser.
BARS = {"exact": (5e-6, 2e-6), "exact_tc": (1.5e-5, 2e-4), "fast": (3e-3, 2e-4)}
ROUND = {"exact": 1e-6, "exact_tc": 1e-6, "fast": 1e-3}     # avg pool: rounding of the stored result (fp32 / fp16)
FEAT_BAR = 1e-6                                               # global pool: fp32 mean of 49 stored values
PLANES_BAR = 2e-6                                             # exact_tc: hi + lo against the fp32 value (22-bit split)
# bn1 (bn_mode='partial'): bars of the training-mode BatchNorm's own records, (its fwd and conv1's dZ through its vjp,
# dgamma / dbeta), and of the running statistics after one momentum step.  Worst measured on an H100 80GB HBM3 (400 W) at
# F = 288, 37 and 1 (tests/test_gpu_schedule_modes.py): exact_tc 1.8e-7 (conv1 dZ) / 2.0e-7 (dgamma at F = 288), exact 6.2e-8 / 1.2e-7,
# running statistics 4.7e-8 (two momentum steps 6.8e-8).  The bars are about 4x those.
BN1_BARS = {"exact": (2.5e-7, 5e-7), "exact_tc": (7e-7, 8e-7)}
RUNSTAT_BAR = 2e-7
SLICE_FACTOR = 4.0
EPS = 1e-5
BN1_CONV, BN1_RAW, BN1_OUT = "conv1_7x7_s2", "conv1_7x7_s2_raw", "conv1_7x7_s2_bn"


class Record:
    """One check: op id, quantity, rel-L2 (tensor, worst frame, worst 64-channel slice), bar, where the worst error sits."""

    def __init__(self, op, quantity, err, frame_err, worst_frame, slice_err, worst_slice, cell, bar, consumers=()):
        self.op, self.quantity, self.err, self.bar = op, quantity, err, bar
        self.frame_err, self.worst_frame, self.slice_err, self.worst_slice = frame_err, worst_frame, slice_err, worst_slice
        self.cell, self.consumers = cell, tuple(consumers)

    @property
    def ok(self):
        if self.bar == 0.0:
            return self.err == 0.0
        lim = SLICE_FACTOR * self.bar
        return self.err <= self.bar and self.frame_err <= lim and self.slice_err <= lim

    @property
    def score(self):        # how close to failing: worst of the three ratios to their bars
        if self.bar == 0.0:
            return math.inf if self.err != 0.0 else 0.0
        lim = SLICE_FACTOR * self.bar
        return max(self.err / self.bar, self.frame_err / lim, self.slice_err / lim)

    def __repr__(self):
        via = " via %s" % ",".join(self.consumers) if self.consumers else ""
        return ("%s %s%s: rel-L2 %.3e (bar %.1e); worst frame %s %.3e, worst channel slice %d (channels %d..%d) %.3e; "
                "worst (frame, slice) %s" % (self.op, self.quantity, via, self.err, self.bar, self.worst_frame, self.frame_err,
                                              self.worst_slice, 64 * self.worst_slice, 64 * self.worst_slice + 63, self.slice_err,
                                              self.cell))


def _rel(num, den):
    return torch.where(den > 0, (num / den.clamp_min(1e-300)).sqrt(),
                       torch.where(num > 0, torch.full_like(num, math.inf), torch.zeros_like(num)))


class _Acc:
    """squared error and squared reference per (frame, 64-channel slice), accumulated over frame chunks"""

    def __init__(self, frames, channels, device):
        self.ns = (channels + 63) // 64
        self.num = torch.zeros(frames, self.ns, dtype=torch.float64, device=device)
        self.den = torch.zeros_like(self.num)

    def add(self, f0, got, ref, scale=None):
        """scale: what the error is relative to, in place of ref"""
        n, c = got.shape[:2]
        d = (got.double() - ref).reshape(n, c, -1)
        e = d.pow(2).sum(2)
        r = (ref if scale is None else scale).reshape(n, c, -1).pow(2).sum(2)
        pad = self.ns * 64 - c
        self.num[f0:f0 + n] += F.pad(e, (0, pad)).view(n, self.ns, 64).sum(2)
        self.den[f0:f0 + n] += F.pad(r, (0, pad)).view(n, self.ns, 64).sum(2)

    def record(self, op, quantity, bar, consumers=(), frames=True):
        err = float(_rel(self.num.sum(), self.den.sum()))
        fe = _rel(self.num.sum(1), self.den.sum(1))
        se = _rel(self.num.sum(0), self.den.sum(0))
        ce = _rel(self.num, self.den)
        wf, ws = int(fe.argmax()), int(se.argmax())
        k = int(ce.flatten().argmax())
        cell = (k // self.ns, k % self.ns) if frames else (None, k % self.ns)
        return Record(op, quantity, err, float(fe[wf]), wf if frames else None, float(se[ws]), ws, cell, bar, consumers)


# ---- the graph, as the engine names it ----------------------------------------------------------------------------------
def _pool_out(h, k, s, p):       # ceil_mode (layer_factory.py:46-50)
    o = (h + 2 * p - k + s - 1) // s + 1
    if (o - 1) * s >= h + p:
        o -= 1
    return o


class Graph:
    """BNInception from O.bninception_ops: the engine's op list, every value's shape, consumers and concat slices.
    bn1_train: bn_mode='partial', as the engine plans it: conv1 writes conv1_7x7_s2_raw (no fold, no ReLU) and an op of kind
    "bn" (training-mode BatchNorm + ReLU) turns it into conv1_7x7_s2_bn."""

    def __init__(self, in_channels=3, bn1_train=False):
        self.in_channels, self.bn1_train = in_channels, bn1_train
        self.ops = []            # dicts: kind (conv / bn / maxpool / avgpool / gpool), id, inp, out, attrs; raw convs: raw=True
        self.shape = {"data": (in_channels, 224, 224)}
        self.branch = {}         # branch value -> (block output, channel offset)
        self.members = {}        # block output -> [branch values]
        for kind, id_, out, ins, a in O.bninception_ops(in_channels):
            c, h, w = self.shape.get(ins[0], (0, 0, 0))
            if kind == "conv":
                ho = (h + 2 * a["pad"] - a["k"]) // a["stride"] + 1
                if bn1_train and id_ == BN1_CONV:
                    self.shape[BN1_RAW] = (a["cout"], ho, ho)
                    self.ops.append(dict(kind="conv", id=id_, inp=ins[0], out=BN1_RAW, a=a, raw=True))
                    self.shape[out] = (a["cout"], ho, ho)
                    self.ops.append(dict(kind="bn", id=out, inp=BN1_RAW, out=out, a={}))
                    continue
                self.shape[out] = (a["cout"], ho, ho)
                self.ops.append(dict(kind="conv", id=id_, inp=ins[0], out=out, a=a))
            elif kind == "pool" and id_ == "global_pool":
                self.ops.append(dict(kind="gpool", id=id_, inp=ins[0], out="feat", a=a))
            elif kind == "pool":
                ho = _pool_out(h, a["k"], a["stride"], a["pad"])
                self.shape[out] = (c, ho, ho)
                self.ops.append(dict(kind="maxpool" if a["mode"] == "max" else "avgpool", id=id_, inp=ins[0], out=out, a=a))
            elif kind == "concat":
                off = 0
                for v in ins:
                    self.branch[v] = (out, off)
                    off += self.shape[v][0]
                self.members[out] = list(ins)
                self.shape[out] = (off,) + self.shape[ins[0]][1:]
        self.consumers = {}
        for o in self.ops:
            self.consumers.setdefault(o["inp"], []).append(o)
        self.conv_ids = [o["id"] for o in self.ops if o["kind"] == "conv"]

    def engine_ops(self):
        """[(kind, input value, output value)] in the engine's order (what BackboneEngine.ops() returns)"""
        return [(o["kind"], o["inp"], o["out"]) for o in self.ops]


# ---- float64 pieces ------------------------------------------------------------------------------------------------------
def fold(params, conv_id, device):
    """float64 BN fold of one conv: (W', b', s) with s = gamma / sqrt(var + eps)"""
    g = lambda k: params[conv_id + k].detach().to(device=device, dtype=torch.float64)
    s = g("_bn.weight") / torch.sqrt(g("_bn.running_var") + EPS)
    w = g(".weight") * s.view(-1, 1, 1, 1)
    b = (g(".bias") - g("_bn.running_mean")) * s + g("_bn.bias")
    return w, b, s


def maxpool_route(x, g, k, s, p):
    """vjp of a ceil-mode max pool with the kernels' rule, ATen's: in row-major tap order a tap takes the gradient when it is
    greater than the maximum so far or is NaN, so the FIRST maximum wins and, in a window with NaNs, the LAST NaN; padding
    never wins (a window of -inf routes to its first real tap)"""
    n, c, h, w = x.shape
    oh, ow = g.shape[2:]
    hp, wp = (oh - 1) * s + k, (ow - 1) * s + k
    pads = (p, wp - w - p, p, hp - h - p)
    cols = F.unfold(F.pad(x, pads), k, stride=s).view(n, c, k * k, oh * ow)
    real = F.unfold(F.pad(torch.ones_like(x[:1, :1]), pads), k, stride=s).view(1, 1, k * k, oh * ow) > 0
    tap = torch.arange(k * k, device=x.device).view(1, 1, k * k, 1)
    nan = cols.isnan() & real
    num = real & ~nan
    top = torch.where(num, cols, -math.inf).amax(2, keepdim=True)
    first_max = torch.where(num & (cols == top), tap, k * k).amin(2, keepdim=True)
    last_nan = torch.where(nan, tap, -1).amax(2, keepdim=True)
    idx = torch.where(last_nan >= 0, last_nan, first_max)
    onehot = torch.zeros_like(cols).scatter_(2, idx, g.reshape(n, c, 1, oh * ow))
    dxp = F.fold(onehot.view(n, c * k * k, oh * ow), (hp, wp), k, stride=s)
    return dxp[:, :, p:p + h, p:p + w]


def _avgpool_vjp(g, in_shape, a):
    x = torch.zeros(in_shape, dtype=g.dtype, device=g.device, requires_grad=True)
    with torch.enable_grad():
        y = F.avg_pool2d(x, a["k"], a["stride"], a["pad"], ceil_mode=True)
        return torch.autograd.grad(y, x, g)[0]


# ---- the checker ---------------------------------------------------------------------------------------------------------
class _Reader:
    """the consumed representation of values / gradients, read once per group and dropped after"""

    def __init__(self, eng, precision, x):
        self.eng, self.tc, self.fast = eng, precision == "exact_tc", precision == "fast"
        self.x = x
        self.cache = {}

    def get(self, name, grad=False, planes=False):
        key = (name, grad, planes)
        if key not in self.cache:
            if name == "data":
                t = self.x.float().half().float() if self.fast else self.x.float()
            else:
                t = self.eng.read(name, grad=grad, planes=planes and self.tc)
            self.cache[key] = t
        return self.cache[key]

    def operand(self, name):            # what a convolution reads as its input
        return self.get(name, planes=name != "data")

    def dz(self, name):                 # the output gradient a convolution's backward consumed
        return self.get(name, grad=True, planes=True)

    def clear(self):
        self.cache.clear()


def check_schedule(eng, params, x, feat, dfeat=None, dw=None, db=None, precision=None, in_channels=3, chunk=16, device=None,
                   bars=None, bn1=None):
    """Check one forward (+ backward) of `eng` (see the module docstring).  params: the reference state dict (CPU or device);
    x: the forward's input; feat: what it returned; dfeat: the backward's input, None for a forward-only check; dw / db: the
    69 gradient tensors the backward filled (reference layout); bars: (fwd / dZ / G, dW / db) in place of BARS[precision]
    (and of BN1_BARS[precision]).
    bn1: for an engine created with bn1_train (bn_mode='partial'), a dict of the first BatchNorm's gamma, beta, momentum, eps,
    running_mean0 / running_var0 (held before the forward), running_mean / running_var (after it) and the dgamma / dbeta the
    backward filled.  Returns [Record] in schedule order."""
    if precision not in BARS:
        raise ValueError("precision must be one of %s" % sorted(BARS))
    backward = dfeat is not None
    G = Graph(in_channels, bn1_train=bn1 is not None)
    dev = torch.device(device) if device is not None else feat.device
    act_bar, par_bar = bars or BARS[precision]
    bn_act_bar, bn_par_bar = bars or BN1_BARS.get(precision, BARS[precision])
    frames = feat.shape[0]
    R = _Reader(eng, precision, x.to(dev))
    folded = {}
    bnstat = {}              # bn1: float64 batch statistics of the consumed z (mu, invstd, rows per channel)
    recs = []

    def W(cid):
        if cid not in folded:
            if bn1 is not None and cid == BN1_CONV:      # raw conv1: its BatchNorm runs in training mode, nothing folds, s = 1
                w, b = (params[cid + k].detach().to(device=dev, dtype=torch.float64) for k in (".weight", ".bias"))
                folded[cid] = (w, b, torch.ones_like(b))
            else:
                folded[cid] = fold(params, cid, dev)
        return folded[cid]

    def chunks():
        for f0 in range(0, frames, chunk):
            yield f0, slice(f0, min(frames, f0 + chunk))

    d64 = lambda t: t.to(device=dev, dtype=torch.float64)
    col = lambda t: d64(t).view(1, -1, 1, 1)

    def vector(op, quantity, got, ref, bar, scale=None):        # one record over a per-channel (or per-output-channel) tensor
        acc = _Acc(1, ref.shape[0], dev)
        shape = (1, ref.shape[0], -1)
        acc.add(0, d64(got).reshape(shape), ref.reshape(shape), None if scale is None else scale.reshape(shape))
        return acc.record(op, quantity, bar, frames=False)

    # ---- forward ----
    for o in G.ops:
        a = o["a"]
        if o["kind"] == "gpool":
            acc = _Acc(frames, 1024, dev)
            y = R.get(o["inp"])
            for f0, sl in chunks():
                ref = d64(y[sl]).mean((2, 3))
                acc.add(f0, d64(feat[sl]).view(-1, 1024, 1, 1), ref.view(-1, 1024, 1, 1))
            recs.append(acc.record(o["id"], "fwd", FEAT_BAR))
            R.clear()
            continue
        c = G.shape[o["out"]][0]
        acc = _Acc(frames, c, dev)
        y = R.get(o["out"])
        if o["kind"] == "conv":
            w, b, _s = W(o["id"])
            xin = R.operand(o["inp"])
            for f0, sl in chunks():
                ref = F.conv2d(d64(xin[sl]), w, b, a["stride"], a["pad"])
                acc.add(f0, d64(y[sl]), ref if o.get("raw") else F.relu(ref))
            bar = act_bar
        elif o["kind"] == "bn":
            z = R.get(o["inp"])                          # the fp32 z the statistics pass read
            n = frames * z.shape[2] * z.shape[3]
            mu = sum(d64(z[sl]).sum((0, 2, 3)) for _f0, sl in chunks()) / n
            var = sum((d64(z[sl]) - mu.view(1, -1, 1, 1)).pow(2).sum((0, 2, 3)) for _f0, sl in chunks()) / n
            invstd = 1.0 / torch.sqrt(var + bn1["eps"])
            bnstat.update(mu=mu, invstd=invstd, n=n)
            for f0, sl in chunks():
                xh = (d64(z[sl]) - mu.view(1, -1, 1, 1)) * invstd.view(1, -1, 1, 1)
                acc.add(f0, d64(y[sl]), F.relu(xh * col(bn1["gamma"]) + col(bn1["beta"])))
            bar = bn_act_bar
        else:
            xin = R.get(o["inp"])
            for f0, sl in chunks():
                pool = F.max_pool2d if o["kind"] == "maxpool" else F.avg_pool2d
                acc.add(f0, d64(y[sl]), pool(d64(xin[sl]), a["k"], a["stride"], a["pad"], ceil_mode=True))
            bar = 0.0 if o["kind"] == "maxpool" else ROUND[precision]
        recs.append(acc.record(o["id"], "fwd", bar))
        if R.tc:
            acc = _Acc(frames, c, dev)
            pl = R.get(o["out"], planes=True)
            for f0, sl in chunks():
                acc.add(f0, d64(pl[sl]), d64(y[sl]))
            recs.append(acc.record(o["id"], "planes", PLANES_BAR))
        if o["kind"] == "bn" and backward:
            m, n = float(bn1["momentum"]), bnstat["n"]
            rm = (1 - m) * d64(bn1["running_mean0"]) + m * mu
            rv = (1 - m) * d64(bn1["running_var0"]) + m * var * (n / max(n - 1, 1))
            recs.append(vector(o["id"], "running_mean", bn1["running_mean"], rm, RUNSTAT_BAR))
            recs.append(vector(o["id"], "running_var", bn1["running_var"], rv, RUNSTAT_BAR))
        R.clear()
    if not backward:
        return recs

    # ---- data gradients: one group per value whose gradient is accumulated (a block output covers its branches) ----
    producer = {o["out"]: o for o in G.ops}
    for v in reversed(list(G.shape)):
        if v == "data" or v in G.branch or v not in G.consumers:
            continue
        cons = G.consumers[v]
        members = G.members.get(v, [v])
        accs = {m: _Acc(frames, G.shape[m][0], dev) for m in members}
        bn_sums = {}
        for c in cons:
            if c["kind"] == "bn":       # the BatchNorm vjp couples all frames: sum g and sum g * xhat first
                mu, invstd = bnstat["mu"].view(1, -1, 1, 1), bnstat["invstd"].view(1, -1, 1, 1)
                sb = sg = 0.0
                for _f0, sl in chunks():
                    g = (d64(R.get(c["out"])[sl]) > 0) * d64(R.get(c["out"], grad=True)[sl])
                    sb = sb + g.sum((0, 2, 3))
                    sg = sg + (g * (d64(R.get(v)[sl]) - mu) * invstd).sum((0, 2, 3))
                bn_sums[c["id"]] = (sb, sg)
        for f0, sl in chunks():
            n = sl.stop - sl.start
            g = torch.zeros((n,) + G.shape[v], dtype=torch.float64, device=dev)
            for c in cons:
                a = c["a"]
                if c["kind"] == "conv":
                    w, _b, _s = W(c["id"])
                    g += torch.nn.grad.conv2d_input(g.shape, w, d64(R.dz(c["out"])[sl]), a["stride"], a["pad"])
                elif c["kind"] == "bn":
                    sb, sg = bn_sums[c["id"]]
                    mu, invstd, m = bnstat["mu"].view(1, -1, 1, 1), bnstat["invstd"].view(1, -1, 1, 1), bnstat["n"]
                    gy = (d64(R.get(c["out"])[sl]) > 0) * d64(R.get(c["out"], grad=True)[sl])
                    xh = (d64(R.get(v)[sl]) - mu) * invstd
                    g += col(bn1["gamma"]) * invstd * (gy - sb.view(1, -1, 1, 1) / m - xh * sg.view(1, -1, 1, 1) / m)
                elif c["kind"] == "maxpool":
                    g += maxpool_route(d64(R.get(v)[sl]), d64(R.get(c["out"], grad=True)[sl]), a["k"], a["stride"], a["pad"])
                elif c["kind"] == "avgpool":
                    g += _avgpool_vjp(d64(R.get(c["out"], grad=True)[sl]), g.shape, a)
                else:
                    g += (d64(dfeat[sl]) / 49.0).view(n, -1, 1, 1)
            for m in members:
                off = G.branch[m][1] if m in G.branch else 0
                gm = g[:, off:off + G.shape[m][0]]
                if producer[m]["kind"] == "conv":
                    accs[m].add(f0, d64(R.dz(m)[sl]), gm if producer[m].get("raw") else (d64(R.get(m)[sl]) > 0) * gm)
                elif m in G.branch:     # max-pool branch: its gradient may be masked by the block output's last writer
                    mask = d64(R.get(m)[sl]) > 0
                    accs[m].add(f0, mask * d64(R.get(m, grad=True)[sl]), mask * gm)
                else:
                    accs[m].add(f0, d64(R.get(m, grad=True)[sl]), gm)
        names = tuple(c["id"] for c in cons)
        for m in members:
            q = "dZ" if producer[m]["kind"] == "conv" else "G"
            recs.append(accs[m].record(producer[m]["id"], q, bn_act_bar if bn_sums else act_bar, names))
        for op_id, (sb, sg) in bn_sums.items():
            recs.append(vector(op_id, "dgamma", bn1["dgamma"], sg, bn_par_bar))
            recs.append(vector(op_id, "dbeta", bn1["dbeta"], sb, bn_par_bar))
        R.clear()

    # ---- weight and bias gradients ----
    for ci, o in enumerate(o for o in G.ops if o["kind"] == "conv"):
        a = o["a"]
        w, _b, s = W(o["id"])
        xin, dz = R.operand(o["inp"]), R.dz(o["out"])
        rw = torch.zeros_like(w)
        rb = torch.zeros_like(s)
        l1 = torch.zeros_like(s)
        for _f0, sl in chunks():
            z = d64(dz[sl])
            rw += torch.nn.grad.conv2d_weight(d64(xin[sl]), w.shape, z, a["stride"], a["pad"])
            rb += z.sum((0, 2, 3))
            l1 += z.abs().sum((0, 2, 3))
        rw *= s.view(-1, 1, 1, 1)
        rb *= s
        recs.append(vector(o["id"], "dW", dw[ci], rw, par_bar))       # slices of output channels
        # in front of a training-mode BatchNorm sum(dZ) vanishes (sum xhat = 0), so the raw conv1's db is a cancellation of
        # large partial sums: its error is taken relative to sum |dZ|, the scale of the rounding of any summation order
        recs.append(vector(o["id"], "db", db[ci], rb, par_bar, l1 * s if o.get("raw") else None))
        R.clear()
    return recs


def failures(recs):
    return [r for r in recs if not r.ok]


def worst(recs, n=5):
    return sorted(recs, key=lambda r: -r.score)[:n]
