"""CPU restatement of the reference's InceptionV3 forward (model_zoo/bninception/inceptionv3.yaml interpreted by
pytorch_load.py:8-61,64-67 and layer_factory.py) in torch, fp32 or fp64, plus seeded synthetic weights.
TEST INFRASTRUCTURE ONLY.

`layers(in_channels)` lists the yaml's layers in order as (id, op, out, inputs, attrs) -- Convolution, BN, ReLU, Pooling,
Concat and the InnerProduct `top_cls_fc` -- written out block by block here, independently of the engine's table in
csrc/inception_v3.cu; tests compare both against the reference's own graph (tests/golden/inception_v3.json).

Synthetic weights (`synth_weights`): kaiming-uniform convolutions with a small bias, BatchNorm affine parameters near 1 / 0,
then the running statistics are calibrated: one forward in float64 with batch statistics over `calib_frames` seeded
frames, each BatchNorm's batch mean and variance copied into its running buffers (variance clamped at 1e-3).  With those
statistics every frozen BatchNorm normalises its channel to about zero mean and unit variance on inputs like the seeded
ones, so activations stay O(1) through the 94 layers instead of exploding or vanishing.
"""
import torch
import torch.nn.functional as Fn

from .synth import synth_frames

INPUT_SIZE, FEAT_DIM = 299, 2048


def _conv_attrs(cout, kh, kw, stride, ph, pw):
    return {"kernel_h": kh, "kernel_w": kw, "num_output": cout, "pad_h": ph, "pad_w": pw, "stride_h": stride, "stride_w": stride}


def layers(in_channels=3):
    """the yaml's layer list: (id, op, out, [inputs], attrs)"""
    L = []

    def conv(name, x, cout, kh, kw, stride=1, ph=0, pw=0):
        L.append((name + "_Conv2D", "Convolution", name + "_Conv2D", [x], _conv_attrs(cout, kh, kw, stride, ph, pw)))
        L.append((name + "_batchnorm", "BN", name, [name + "_Conv2D"], {}))
        L.append((name, "ReLU", name, [name], {}))
        return name

    def pool(name, x, mode, k, stride, pad):
        L.append((name, "Pooling", name, [x], {"kernel_size": k, "mode": mode, "pad": pad, "stride": stride}))
        return name

    def concat(name, xs):
        L.append((name, "Concat", name, list(xs), {}))
        return name

    x = conv("conv", "data", 32, 3, 3, 2)
    x = conv("conv_1", x, 32, 3, 3)
    x = conv("conv_2", x, 64, 3, 3, 1, 1, 1)
    x = pool("pool", x, "max", 3, 2, 0)
    x = conv("conv_3", x, 80, 1, 1)
    x = conv("conv_4", x, 192, 3, 3)
    x = pool("pool_1", x, "max", 3, 2, 0)
    for p, proj in (("mixed", 32), ("mixed_1", 64), ("mixed_2", 64)):          # 35 x 35
        a = conv(p + "_conv", x, 64, 1, 1)
        b = conv(p + "_tower_conv_1", conv(p + "_tower_conv", x, 48, 1, 1), 64, 5, 5, 1, 2, 2)
        c = conv(p + "_tower_1_conv_2", conv(p + "_tower_1_conv_1", conv(p + "_tower_1_conv", x, 64, 1, 1), 96, 3, 3, 1, 1, 1),
                 96, 3, 3, 1, 1, 1)
        d = conv(p + "_tower_2_conv", pool(p + "_tower_2_pool", x, "ave", 3, 1, 1), proj, 1, 1)
        x = concat(p + "_join", (a, b, c, d))
    p = "mixed_3"                                                                 # 35 -> 17
    a = conv(p + "_conv", x, 384, 3, 3, 2)
    b = conv(p + "_tower_conv_2", conv(p + "_tower_conv_1", conv(p + "_tower_conv", x, 64, 1, 1), 96, 3, 3, 1, 1, 1), 96, 3, 3, 2)
    c = pool(p + "_pool", x, "max", 3, 2, 0)
    x = concat(p + "_join", (a, b, c))
    for p, c7 in (("mixed_4", 128), ("mixed_5", 160), ("mixed_6", 160), ("mixed_7", 192)):    # 17 x 17
        a = conv(p + "_conv", x, 192, 1, 1)
        t = conv(p + "_tower_conv", x, c7, 1, 1)
        t = conv(p + "_tower_conv_1", t, c7, 7, 1, 1, 3, 0)
        b = conv(p + "_tower_conv_2", t, 192, 1, 7, 1, 0, 3)
        t = conv(p + "_tower_1_conv", x, c7, 1, 1)
        for i, (kh, kw) in enumerate(((1, 7), (7, 1), (1, 7), (7, 1))):
            t = conv(p + "_tower_1_conv_%d" % (i + 1), t, 192 if i == 3 else c7, kh, kw, 1, kh // 2, kw // 2)
        d = conv(p + "_tower_2_conv", pool(p + "_tower_2_pool", x, "ave", 3, 1, 1), 192, 1, 1)
        x = concat(p + "_join", (a, b, t, d))
    p = "mixed_8"                                                                 # 17 -> 8
    a = conv(p + "_tower_conv_1", conv(p + "_tower_conv", x, 192, 1, 1), 320, 3, 3, 2)
    t = conv(p + "_tower_1_conv", x, 192, 1, 1)
    t = conv(p + "_tower_1_conv_1", t, 192, 7, 1, 1, 3, 0)
    t = conv(p + "_tower_1_conv_2", t, 192, 1, 7, 1, 0, 3)
    b = conv(p + "_tower_1_conv_3", t, 192, 3, 3, 2)
    c = pool(p + "_pool", x, "max", 3, 2, 0)
    x = concat(p + "_join", (a, b, c))
    for p, mode in (("mixed_9", "ave"), ("mixed_10", "max")):                    # 8 x 8
        a = conv(p + "_conv", x, 320, 1, 1)
        t = conv(p + "_tower_conv", x, 384, 1, 1)
        b1 = conv(p + "_tower_mixed_conv", t, 384, 3, 1, 1, 1, 0)
        b2 = conv(p + "_tower_mixed_conv_1", t, 384, 1, 3, 1, 0, 1)
        t = conv(p + "_tower_1_conv_1", conv(p + "_tower_1_conv", x, 448, 1, 1), 384, 3, 3, 1, 1, 1)
        c1 = conv(p + "_tower_1_mixed_conv", t, 384, 3, 1, 1, 1, 0)
        c2 = conv(p + "_tower_1_mixed_conv_1", t, 384, 1, 3, 1, 0, 1)
        d = conv(p + "_tower_2_conv", pool(p + "_tower_2_pool", x, mode, 3, 1, 1), 192, 1, 1)
        x = concat(p + "_join", (a, b1, b2, c1, c2, d))
    pool("top_cls_pool", x, "ave", 8, 1, 0)
    L[-1] = ("top_cls_pool", "Pooling", "top_cls_global_pool", [x], L[-1][4])
    L.append(("top_cls_fc", "InnerProduct", "fc", ["top_cls_global_pool"], {"num_output": 1000}))
    return L


def conv_layers(in_channels=3):
    """[(name, cin, cout, kh, kw, stride, pad_h, pad_w)] of the 94 convolutions, name = the blob (id without _Conv2D)"""
    ch = {"data": in_channels}
    out = []
    for id_, op, o, ins, a in layers(in_channels):
        if op == "Convolution":
            out.append((id_[:-len("_Conv2D")], ch[ins[0]], a["num_output"], a["kernel_h"], a["kernel_w"], a["stride_h"], a["pad_h"], a["pad_w"]))
            ch[o] = a["num_output"]
        elif op == "Concat":
            ch[o] = sum(ch[i] for i in ins)
        elif op != "InnerProduct":
            ch[o] = ch[ins[0]]
    return out


def state_dict_shapes(in_channels=3):
    """{key: shape} of the backbone state_dict (without the 'base_model.' prefix), the reference's keys and order"""
    sd = {}
    for name, cin, cout, kh, kw, *_ in conv_layers(in_channels):
        sd[name + "_Conv2D.weight"] = (cout, cin, kh, kw)
        sd[name + "_Conv2D.bias"] = (cout,)
        for k in ("weight", "bias", "running_mean", "running_var"):
            sd[name + "_batchnorm." + k] = (cout,)
        sd[name + "_batchnorm.num_batches_tracked"] = ()
    sd["top_cls_fc.weight"] = (1000, FEAT_DIM)
    sd["top_cls_fc.bias"] = (1000,)
    return sd


def forward(params, x, in_channels=3, dtype=torch.float64, taps=None, bn_training=False, bn_stats_out=None):
    """x [F, C, 299, 299] -> top_cls_global_pool features [F, 2048] in `dtype`.  params: backbone state_dict entries
    (no prefix).  taps (dict): every blob is stored there.  bn_training: BatchNorm with batch statistics (calibration), the
    (mean, biased var) of each written to bn_stats_out[name]."""
    p = {k: v.to(dtype) for k, v in params.items() if not k.endswith("num_batches_tracked")}
    blobs = {"data": x.to(dtype)}
    for id_, op, o, ins, a in layers(in_channels):
        if op == "Convolution":
            blobs[o] = Fn.conv2d(blobs[ins[0]], p[id_ + ".weight"], p[id_ + ".bias"], stride=a["stride_h"], padding=(a["pad_h"], a["pad_w"]))
        elif op == "BN":
            z = blobs[ins[0]]
            if bn_training:
                m, v = z.mean(dim=(0, 2, 3)), z.var(dim=(0, 2, 3), unbiased=False)
                if bn_stats_out is not None:
                    bn_stats_out[id_] = (m, v)
            else:
                m, v = p[id_ + ".running_mean"], p[id_ + ".running_var"]
            blobs[o] = Fn.batch_norm(z, m, v, p[id_ + ".weight"], p[id_ + ".bias"], False, 0.0, 1e-5)
        elif op == "ReLU":
            blobs[o] = torch.relu(blobs[ins[0]])
        elif op == "Pooling":
            f = Fn.max_pool2d if a["mode"] == "max" else Fn.avg_pool2d
            blobs[o] = f(blobs[ins[0]], a["kernel_size"], a["stride"], a["pad"], ceil_mode=True)
        elif op == "Concat":
            blobs[o] = torch.cat([blobs[i] for i in ins], 1)
        if taps is not None and op != "InnerProduct":
            taps[o] = blobs[o]
    return blobs["top_cls_global_pool"].flatten(1)


def synth_weights(in_channels=3, seed=0, calib_frames=4):
    """seeded backbone parameters keyed like the reference state_dict (no prefix; top_cls_fc excluded: it is replaced)"""
    g = torch.Generator().manual_seed(5000 + seed)
    p = {}
    for name, cin, cout, kh, kw, *_ in conv_layers(in_channels):
        bound = (6.0 / (cin * kh * kw)) ** 0.5
        c, b = name + "_Conv2D", name + "_batchnorm"
        p[c + ".weight"] = (torch.rand(cout, cin, kh, kw, generator=g) * 2 - 1) * bound
        p[c + ".bias"] = (torch.rand(cout, generator=g) * 2 - 1) * 0.1
        p[b + ".weight"] = 0.75 + 0.5 * torch.rand(cout, generator=g)
        p[b + ".bias"] = 0.3 * (torch.rand(cout, generator=g) * 2 - 1) + 0.1
        p[b + ".running_mean"] = torch.zeros(cout)
        p[b + ".running_var"] = torch.ones(cout)
    stats = {}
    with torch.no_grad():
        forward(p, synth_frames(calib_frames, in_channels, INPUT_SIZE, seed=seed + 77), in_channels, torch.float64,
                bn_training=True, bn_stats_out=stats)
    for id_, (m, v) in stats.items():
        p[id_ + ".running_mean"] = m.float()
        p[id_ + ".running_var"] = v.clamp_min(1e-3).float()
    return p


def ops(in_channels=3):
    """the engine's schedule derived from the yaml layers: (kind, in, out, k, stride, pad) per Convolution / Pooling"""
    out = []
    for id_, op, o, ins, a in layers(in_channels):
        if op == "Convolution":
            out.append(("conv", ins[0], id_[:-len("_Conv2D")], 0, a["stride_h"], 0))
        elif op == "Pooling":
            kind = "gpool" if o == "top_cls_global_pool" else ("maxpool" if a["mode"] == "max" else "avgpool")
            out.append((kind, ins[0], o, a["kernel_size"], a["stride"], a["pad"]))
    return out


def concat_slices(in_channels=3):
    """{branch blob: (join, channel offset)} for every concat input"""
    ch = {"data": in_channels}
    sl = {}
    for id_, op, o, ins, a in layers(in_channels):
        if op == "Convolution":
            ch[o] = a["num_output"]
        elif op == "Concat":
            off = 0
            for i in ins:
                sl[i] = (o, off)
                off += ch[i]
            ch[o] = off
        elif op != "InnerProduct":
            ch[o] = ch[ins[0]]
    return sl
