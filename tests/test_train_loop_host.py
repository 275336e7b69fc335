"""CPU-side checks of the training loop's update block and meters: the oracle (oracle/train_loop_oracle.py) against what the
reference's own accuracy(), AverageMeter and update block computed (tests/golden/train_loop.npz), the ssnb.h structs and
signatures of the new calls mirrored in ctypes, and argument validation that fails before any launch."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import train_loop_oracle as TL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "train_loop.npz"))


@pytest.mark.parametrize("tag", ["ssn", "binary"])
def test_accuracy_and_meters_match_reference(gold, tag):
    meters = TL.new_meters(("act_acc", "fg_acc", "bg_acc"))
    for step in range(3):
        p = "%s_acc%d_" % (tag, step)
        act, tgt = torch.from_numpy(gold[p + "scores"]), torch.from_numpy(gold[p + "target"])
        TL._update_acc(meters, act, tgt)
        vals = [TL.accuracy(act, tgt),
                TL.accuracy(act.view(-1, 2, act.size(1))[:, 0, :], tgt.view(-1, 2)[:, 0]),
                TL.accuracy(act.view(-1, 2, act.size(1))[:, 1, :], tgt.view(-1, 2)[:, 1])]
        assert np.array([float(v) for v in vals], np.float32).tobytes() == gold[p + "vals"].tobytes()
    got = np.array([meters[k] for k in ("act_acc", "fg_acc", "bg_acc")], np.float64)
    assert got.tobytes() == gold[tag + "_meters"].tobytes()


@pytest.mark.parametrize("tag", ["ssn", "binary"])
@pytest.mark.parametrize("case", range(5))
def test_update_block_matches_reference(gold, tag, case):
    p = "%s_upd%d_" % (tag, case)
    iter_size, clip = gold[p + "cfg"]
    clip = None if np.isnan(clip) else float(clip)
    params = [torch.nn.Parameter(torch.from_numpy(gold[p + "param%d" % j]).clone()) for j in range(4)]
    for j, q in enumerate(params):
        q.grad = torch.from_numpy(gold[p + "grad%d" % j]).clone()
    groups = [{"params": params[:2], "lr": 0.1, "weight_decay": 5e-4}, {"params": params[2:3], "lr": 0.2, "weight_decay": 0.0}]
    opt = torch.optim.SGD(groups, lr=0.1, momentum=0.9)
    total = TL.update_block(opt.param_groups, params, int(iter_size), clip)
    assert np.float64(total) == gold[p + "total_norm"]
    for j in range(3):
        assert params[j].grad.numpy().tobytes() == gold[p + "seen%d" % j].tobytes(), j
    opt.step()
    for j in range(3):
        assert params[j].detach().numpy().tobytes() == gold[p + "param_after%d" % j].tobytes(), j
    assert params[3].grad.numpy().tobytes() == gold[p + "extra_after"].tobytes()


def test_extra_grads_struct_and_signatures_match_header(tmp_path):
    from ssn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    m = re.search(r"enum \{ SSNB_GRAD_NORM_CTAS = (\d+), SSNB_MAX_EXTRA_GRADS = (\d+) \};", hdr)
    assert m and (int(m.group(1)), int(m.group(2))) == (_lib.GRAD_NORM_CTAS, _lib.MAX_EXTRA_GRADS)
    for name, n_args in (("ssnb_grad_norm", 7), ("ssnb_grad_clip", 6), ("ssnb_sgd_step_groups_clipped", 15), ("ssnb_train_meters", 10)):
        decl = re.search(r"int %s\(([^)]*)\);" % name, hdr).group(1)
        assert len(decl.split(",")) == n_args == len(_lib.SIGNATURES[name][1]), name
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    fields = ["count", "reserved", "grad", "numel"]
    prints = ['printf("size %zu\\n", sizeof(ssnb_extra_grads));']
    prints += ['printf("%s %%zu\\n", offsetof(ssnb_extra_grads, %s));' % (f, f) for f in fields]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    exe = tmp_path / "abi"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True)
    lay = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(lay["size"]) == C.sizeof(_lib.ExtraGrads)
    assert [n for n, _ in _lib.ExtraGrads._fields_] == fields
    for f in fields:
        assert getattr(_lib.ExtraGrads, f).offset == int(lay[f]), f


def test_arguments_rejected_before_any_launch():
    """every bad argument returns SSNB_EINVAL from the host-side checks (no device is touched: this runs without one)"""
    from ssn_b200._lib import lib, ExtraGrads
    EINVAL = 1
    buf = C.create_string_buffer(64)
    p = C.cast(buf, C.c_void_p)
    too_many = ExtraGrads(count=9)
    null_extra = ExtraGrads(count=1)
    null_extra.numel[0] = 5
    assert lib.ssnb_grad_norm(p, 4, 1.0, None, None, p, None) == EINVAL            # no partials
    assert lib.ssnb_grad_norm(None, 4, 1.0, None, p, p, None) == EINVAL            # no gradient
    assert lib.ssnb_grad_norm(p, 4, 1.0, C.byref(too_many), p, p, None) == EINVAL
    assert lib.ssnb_grad_norm(p, 4, 1.0, C.byref(null_extra), p, p, None) == EINVAL
    assert b"extra gradient 0" in lib.ssnb_last_error(None)
    assert lib.ssnb_grad_clip(None, 1.0, p, 4, None, None) == EINVAL
    assert lib.ssnb_grad_clip(p, float("nan"), p, 4, None, None) == EINVAL
    assert lib.ssnb_grad_clip(p, -1.0, p, 4, None, None) == EINVAL
    assert lib.ssnb_sgd_step_groups_clipped(p, p, p, 4, p, p, p, 1, 0.9, 1.0, None, 1.0, 1, None, None) == EINVAL
    assert lib.ssnb_sgd_step_groups_clipped(p, p, p, 4, p, p, p, 0, 0.9, 1.0, p, 1.0, 1, None, None) == EINVAL
    assert lib.ssnb_sgd_step_groups_clipped(p, p, p, 4, p, p, p, 1, 0.9, 1.0, p, 1.0, 1, C.byref(too_many), None) == EINVAL
    assert lib.ssnb_train_meters(p, 0, 3, p, None, p, 1, 1.0, p, None) == EINVAL   # no rows
    assert lib.ssnb_train_meters(p, 4, 0, p, None, p, 1, 1.0, p, None) == EINVAL   # no columns
    assert lib.ssnb_train_meters(p, 4, 3, p, None, None, 1, 1.0, p, None) == EINVAL
    assert lib.ssnb_train_meters(p, 4, 3, p, None, p, 9, 1.0, p, None) == EINVAL
    assert lib.ssnb_train_meters(p, 4, 3, p, None, p, 1, 0.0, p, None) == EINVAL
    assert lib.ssnb_train_meters(p, 65537, 3, p, None, p, 1, 1.0, p, None) == EINVAL


def test_python_surface_rejects_bad_input():
    from ssn_b200.meters import StepMeters
    from ssn_b200.optim import _extra_grads
    with pytest.raises(ValueError):
        StepMeters("tsn", "cpu")
    with pytest.raises(ValueError):
        _extra_grads([torch.zeros(2)] * 9, torch.device("cpu"))
    with pytest.raises(ValueError):
        _extra_grads([torch.zeros(2, dtype=torch.float64)], torch.device("cpu"))
    m = StepMeters("binary", "cpu")
    with pytest.raises(ValueError):                 # an SSN update on binary meters
        m.update_ssn(torch.zeros(4), torch.zeros(8, 3), torch.zeros(8), torch.zeros(8), 2)
    with pytest.raises(ValueError):                 # 3 targets for 8 rows
        m.update_binary(torch.zeros(1), torch.zeros(8, 2), torch.zeros(3), 2)
    assert m.read() == {"loss": 0.0, "act_acc": 0.0, "fg_acc": 0.0, "bg_acc": 0.0}
