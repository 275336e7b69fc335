"""InceptionV3 at test time, CPU side: the oracle against the reference's golden (graph, state_dict, features, scores), the
engine's plan against the reference graph without a GPU, the module surface and the ABI mirror of ssnb_iv3_config."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import inception_v3_oracle as IV
from oracle import synth, binary_oracle as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = (("rgb", "RGB", 3, 4, 11), ("flow", "Flow", 10, 3, 12))     # as oracle/gen_golden_inception_v3.py


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLD, "inception_v3.json")) as f:
        g = json.load(f)
    return g, np.load(os.path.join(GOLD, "inception_v3.npz"))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def test_oracle_graph_equals_reference(golden):
    g, _ = golden
    mine = [[i, op, o, list(ins), a] for (i, op, o, ins, a) in IV.layers(3)]
    assert mine == g["layers"]
    assert sum(1 for l in g["layers"] if l[1] == "Convolution") == 94


def test_module_surface_matches_reference(golden):
    import model_zoo
    import ssn_models
    g, _ = golden
    net = model_zoo.InceptionV3()
    assert [n for n, _ in net.named_children()] == g["children"]
    for tag, modality, cin, K, _seed in CASES:
        m = ssn_models.SSN(K, 2, 5, 2, modality, base_model="InceptionV3", dropout=0, test_mode=True)
        assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == g["state_dict"][tag]
        want = {k[len("base_model."):]: tuple(s) for k, s in g["state_dict"][tag] if k.startswith("base_model.")}
        mine = {k: s for k, s in IV.state_dict_shapes(cin).items() if not k.startswith("top_cls_fc")}
        assert mine == want
        inp = g["input_" + tag]
        assert (m.input_size, m.input_mean, m.input_std, m.crop_size, m.scale_size) == \
            (inp["input_size"], inp["input_mean"], inp["input_std"], inp["crop_size"], inp["scale_size"])
        assert m.base_model.last_layer_name == "top_cls_fc" and m.base_model.in_channels() == cin


def test_flow_stem_is_the_mean_expanded_rgb_kernel():
    import ssn_models
    m = ssn_models.SSN(3, 2, 5, 2, "Flow", base_model="InceptionV3", dropout=0)
    c = m.base_model.conv_Conv2D
    # _construct_flow_model: a 10-channel stem whose every input channel holds the mean RGB kernel, bias kept
    assert tuple(c.weight.shape) == (32, 10, 3, 3) and c.stride == (2, 2) and c.padding == (0, 0) and c.bias is not None
    assert torch.equal(c.weight.data, c.weight.data[:, :1].expand_as(c.weight.data))
    assert m.input_mean == [128] and m.new_length == 5


@pytest.mark.parametrize("tag,modality,cin,K,seed", CASES)
def test_oracle_equals_reference_features_and_scores(golden, tag, modality, cin, K, seed):
    _, a = golden
    p = IV.synth_weights(cin, seed=0)
    x = synth.synth_frames(10, cin, IV.INPUT_SIZE, seed=seed)
    # fp32 restates the reference's arithmetic (<= 1e-5); float64 differs from the fp32 reference by the reference's own rounding
    # through 94 layers (1.7e-5 measured for RGB)
    for dtype, bar in ((torch.float64, 5e-5), (torch.float32, 1e-5)):
        with torch.no_grad():
            feat = IV.forward(p, x, cin, dtype)
        assert _rel(feat, a[tag + "_base_out"]) <= bar, (tag, dtype)
        assert _rel(feat, a[tag + "_binary_base"]) <= bar, (tag, dtype)
    import ssn_models
    m = ssn_models.SSN(K, 2, 5, 2, modality, base_model="InceptionV3", dropout=0, test_mode=True)
    sd = m.state_dict()
    with torch.no_grad():
        for k, v in synth.synth_heads(K, m.stpp.feat_multiplier, feat_dim=IV.FEAT_DIM, seed=0, std=0.02, bias_std=0.1).items():
            sd[k].copy_(v)
    m.prepare_test_fc()
    test_fc = feat.double() @ m.test_fc.weight.data.double().t() + m.test_fc.bias.data.double()
    assert _rel(test_fc, a[tag + "_test_fc"]) <= 1e-5
    cls = B.synth_classifier(2, feat_dim=IV.FEAT_DIM, seed=0)
    scores = feat.double() @ cls["classifier_fc.weight"].double().t() + cls["classifier_fc.bias"].double()
    assert _rel(scores, a[tag + "_binary_scores"]) <= 1e-5


@pytest.mark.parametrize("cin", [3, 10])
def test_engine_plan_matches_reference_graph(cin):
    from ssn_b200.inception_v3 import InceptionV3Engine, conv_table
    assert conv_table(cin) == IV.conv_layers(cin)
    eng = InceptionV3Engine(cin, 1)                  # planning needs no GPU
    ops = eng.ops()
    assert [(k, i, o, kk, s, p) for (k, i, o, _c, kk, s, p) in ops] == \
        [(k, i, o, kk if k != "conv" else 0, s, p if k != "conv" else 0) for (k, i, o, kk, s, p) in IV.ops(cin)]
    assert [c for (k, _i, _o, c, *_r) in ops if k == "conv"] == list(range(94))
    # shapes of every value and the channel offset of every concat input, against the oracle's own forward
    taps = {}
    with torch.no_grad():
        IV.forward(IV.synth_weights(cin, calib_frames=1), torch.zeros(1, cin, 299, 299), cin, torch.float32, taps=taps)
    slices = IV.concat_slices(cin)
    for name, t in taps.items():
        if name == "top_cls_global_pool" or name.endswith("_Conv2D"):        # the feat output; pre-BatchNorm blobs (folded)
            continue
        c, h, w, buf, coff = eng.value_info(name)
        assert (c, h, w) == tuple(t.shape[1:]), name
        if name in slices:
            assert (buf, coff) == slices[name], name
        elif name.endswith("_join"):
            assert (buf, coff) == (name, 0)
    assert ops[-1][0] == "gpool" and ops[-1][2] == "top_cls_global_pool" and ops[-1][4:] == (8, 1, 0)


def test_workspace_at_400_frames():
    from ssn_b200.inception_v3 import InceptionV3Engine
    # every value keeps a buffer of its own: 9.23 M fp32 elements per RGB frame (conv outputs 8.97 M, the input and the
    # pool outputs the rest), plus one arg-max byte per max-pool output element and the packed weights
    # (FAST: fp16 storage; EXACT_TC: fp32 plus the fp16 hi / lo operand planes of every value; the tensor-core modes pad the
    # input to 16 channels)
    from ssn_b200 import _lib
    for prec, (rgb, flow) in WORKSPACE_400.items():
        assert InceptionV3Engine(3, 400, prec).workspace_bytes == rgb, prec
        assert InceptionV3Engine(10, 400, prec).workspace_bytes == flow, prec


WORKSPACE_400 = {0: (19624844288, 20626151424), 1: (10910259200, 10910259200), 2: (42632786944, 42632786944)}


def test_engine_rejections_without_gpu():
    from ssn_b200 import _lib
    h = C.c_void_p()
    for cfg, msg in ((_lib.IV3Config(3, 8, 7, 0), b"unknown precision"), (_lib.IV3Config(4, 8, _lib.EXACT_FP32, 0), b"in_channels"),
                     (_lib.IV3Config(3, 0, _lib.EXACT_FP32, 0), b"frames")):
        assert _lib.lib.ssnb_iv3_create(C.byref(cfg), C.byref(h)) == 1
        assert msg in _lib.lib.ssnb_last_error(None), (msg, _lib.lib.ssnb_last_error(None))
    for prec in (_lib.FAST_FP16, _lib.EXACT_TC):             # every precision plans without a GPU
        cfg = _lib.IV3Config(10, 8, prec, 0)
        assert _lib.lib.ssnb_iv3_create(C.byref(cfg), C.byref(h)) == 0
        assert _lib.lib.ssnb_iv3_workspace_bytes(h) > 0
        _lib.lib.ssnb_iv3_destroy(h)
    assert _lib.lib.ssnb_iv3_conv_info(94, 3, None, 0, *([None] * 7)) != 0
    ok = _lib.IV3Config(3, 2, _lib.EXACT_FP32, 0)
    assert _lib.lib.ssnb_iv3_create(C.byref(ok), C.byref(h)) == 0
    assert _lib.lib.ssnb_iv3_forward(h, None, None, None) != 0
    assert _lib.lib.ssnb_iv3_run_op(h, 0, None, None) != 0            # no workspace, no weights: refused, no launch
    assert _lib.lib.ssnb_iv3_value_info(h, b"nonexistent", None, None, None, None, 0, None) != 0
    _lib.lib.ssnb_iv3_destroy(h)


def test_training_paths_raise_before_any_launch():
    import ssn_models
    import binary_model
    from ssn_b200 import _lib
    m = ssn_models.SSN(3, 2, 5, 2, "RGB", base_model="InceptionV3", dropout=0)
    with pytest.raises(NotImplementedError, match="follow-up"):
        m.fused_step(torch.zeros(1), None, None, None, None)
    with pytest.raises(ValueError, match="precision"):
        m.set_precision(7)
    m.set_precision(_lib.EXACT_TC)
    assert m.base_model.precision == _lib.EXACT_TC
    b = binary_model.BinaryClassifier(2, 5, "RGB", base_model="InceptionV3", dropout=0)
    with pytest.raises(NotImplementedError, match="follow-up"):
        b.fused_step(torch.zeros(1), None)


def test_header_mirror_of_iv3_config(tmp_path):
    from ssn_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct \{([^{}]*)\}\s*ssnb_iv3_config;", hdr).group(1), flags=re.S)
    names = [d.split()[1] for d in body.split(";") if d.strip()]
    assert names == [n for n, _ in _lib.IV3Config._fields_]
    prints = ['printf("size %zu\\n", sizeof(ssnb_iv3_config));'] + ['printf("%s %%zu\\n", offsetof(ssnb_iv3_config, %s));' % (n, n) for n in names]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "abi")], check=True)
    lay = dict(l.split() for l in subprocess.run([str(tmp_path / "abi")], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(lay["size"]) == C.sizeof(_lib.IV3Config)
    for n, _ in _lib.IV3Config._fields_:
        assert int(lay[n]) == getattr(_lib.IV3Config, n).offset
