"""CPU tests of the frame transforms: the numpy oracle bitwise against the reference's transforms.py + PIL (tests/golden/frames.npz,
oracle/gen_golden_frames.py), the parameter draws against the reference's, the C struct layout and the host-side argument checks."""
import ctypes as C
import hashlib
import json
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import frames_oracle as F
from oracle.gen_golden_frames import frames_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "frames.npz"))
CASES = json.loads(str(GOLDEN["cases"]))


def oracle_case(case, frames):
    if case["kind"] == "train":
        return F.train_group(list(frames), case["params"], case["out"], case["mean"], [1], case["is_flow"])
    if case["kind"] == "oversample":
        return F.oversample_group(list(frames), case["out"], case["scale"], case["mean"], [1])
    return F.center_group(list(frames), case["out"], case["scale"], case["mean"], [1])


@pytest.mark.parametrize("case", [c for c in CASES if "seed" not in c], ids=lambda c: c["name"])
def test_oracle_matches_reference_small(case):
    got = oracle_case(case, GOLDEN["in_" + case["name"]])
    ref = GOLDEN["out_" + case["name"]]
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert got.tobytes() == ref.tobytes()


@pytest.mark.parametrize("case", [c for c in CASES if "seed" in c], ids=lambda c: c["name"])
def test_oracle_matches_reference_full_size(case):
    got = oracle_case(case, frames_for(case["seed"], *case["shape"]))
    assert list(got.shape) == case["out_shape"]
    assert hashlib.sha256(np.ascontiguousarray(got, np.float32).tobytes()).hexdigest() == case["sha256"]


def test_golden_covers_the_edge_cases():
    byname = {c["name"]: c for c in CASES}
    # a 31-row frame whose crop snapped up to the output size and reaches outside it
    assert any(c["params"][1] == 32 for n, c in byname.items() if n.startswith("train_snap"))
    assert any(c["kind"] == "train" and c["params"][4] for c in CASES) and any(c["kind"] == "train" and not c["params"][4] for c in CASES)
    sizes = [F.scaled_size(*GOLDEN["in_" + c["name"]].shape[1:3], c["scale"]) for c in CASES if c["kind"] == "center" and "seed" not in c]
    assert any((h - 32) % 2 for h, _ in sizes) and any((w - 32) % 2 for _, w in sizes), "no centre crop with an odd difference"


def test_sample_train_params_matches_reference_draws():
    from ops.frame_transforms import sample_train_params
    draws = json.loads(str(GOLDEN["draws"]))
    assert draws
    for d in draws:
        random.seed(d["seed"])
        got = sample_train_params([tuple(s) for s in d["sizes"]], d["scales"], fix_crop=d["fix_crop"])
        assert [list(g[:4]) + [int(g[4])] for g in got] == d["params"], d
    rng = random.Random(5)
    assert sample_train_params([(256, 340)], [1, .875, .75, .66], rng=rng) == sample_train_params([(256, 340)], [1, .875, .75, .66],
                                                                                                   rng=random.Random(5))


def test_frame_structs_match_header(tmp_path):
    from ssn_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()

    def fields(struct):
        body = re.search(r"typedef struct \{([^{}]*)\}\s*" + struct + ";", hdr).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if decl:
                names += [re.sub(r"\[.*\]", "", n).strip() for n in decl.split(None, 1)[1].split(",")]
        return names

    structs = {"ssnb_frame_cfg": _lib.FrameCfg, "ssnb_frame_group": _lib.FrameGroup}
    prints = []
    for s in structs:
        prints.append('printf("%s %%zu\\n", sizeof(%s));' % (s, s))
        prints += ['printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f) for f in fields(s)]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    exe = tmp_path / "abi"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    layout = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for s, mirror in structs.items():
        assert int(layout[s]) == C.sizeof(mirror), s
        assert [n for n, _ in mirror._fields_] == fields(s), s
        for n, _ in mirror._fields_:
            assert getattr(mirror, n).offset == int(layout["%s.%s" % (s, n)]), (s, n)


def _layout(cfg, groups):
    from ssn_b200._lib import lib
    ws, nd = C.c_size_t(0), C.c_int64(0)
    rc = lib.ssnb_frame_transform_workspace_bytes(C.byref(cfg), groups, len(groups), C.byref(ws), C.byref(nd))
    return rc, ws.value, nd.value


def _cfg(mode=0, channels=3, out=224, scale=256, mean=(104, 117, 128)):
    from ssn_b200._lib import FrameCfg
    return FrameCfg(mode, channels, out, scale, 0, len(mean), (C.c_float * 8)(*mean), (C.c_float * 8)(*([1.0] * len(mean))))


def _group(h=256, w=340, n=9, crop=(0, 0, 224, 224)):
    from ssn_b200._lib import FrameGroup
    g = FrameGroup()
    g.height, g.width, g.images = h, w, n
    g.crop_x, g.crop_y, g.crop_w, g.crop_h = crop
    return g


def test_layout_fills_offsets_and_sizes():
    from ssn_b200._lib import FrameGroup, FRAMES_OVERSAMPLE
    gs = (FrameGroup * 3)(_group(256, 340, 4), _group(360, 480, 2), _group(256, 256, 1))
    rc, ws, nd = _layout(_cfg(FRAMES_OVERSAMPLE), gs)
    assert rc == 0
    assert [g.first_image for g in gs] == [0, 4, 6]
    assert [g.dst_offset for g in gs] == [0, 10 * 4 * 3 * 224 * 224, 10 * 6 * 3 * 224 * 224]
    assert nd == 10 * 7 * 3 * 224 * 224
    assert ws >= 2 * 256 * 341 * 3 and gs[1].scratch_offset == 0       # only the 480x360 group is resized (to 341x256)


@pytest.mark.parametrize("bad", ["mode", "channels", "out", "scale", "n_mean", "mean_cycle", "crop_w", "crop_big", "height", "images"])
def test_layout_rejects_bad_arguments(bad):
    from ssn_b200._lib import lib, FrameGroup
    cfg = _cfg(mode=1 if bad == "scale" else 0, mean=(104, 117) if bad == "mean_cycle" else (104, 117, 128))
    g = _group()
    if bad == "mode":
        cfg.mode = 7
    elif bad == "channels":
        cfg.channels = 2
    elif bad == "out":
        cfg.out_size = 0
    elif bad == "scale":
        cfg.scale_size = 100
    elif bad == "n_mean":
        cfg.n_mean = 9
    elif bad == "crop_w":
        g.crop_w = 0
    elif bad == "crop_big":
        g.crop_w = 17 * 224
    elif bad == "height":
        g.height = 0
    elif bad == "images":
        g.images = 0
    if bad == "mean_cycle":
        g.images = 1                              # 3 planes do not cycle over 2 means
    rc, _, _ = _layout(cfg, (FrameGroup * 1)(g))
    assert rc == 1, lib.ssnb_last_error(None)
    assert lib.ssnb_last_error(None).startswith(b"frame_transform: ")


def test_model_frame_transforms_fill_in_the_model():
    import ssn_models
    rgb = ssn_models.SSN(5, 2, 5, 2, "RGB", base_model="BNInception", dropout=0).frame_transforms()
    assert rgb.train.keywords["mean"] == [104, 117, 128] and rgb.train.keywords["frame_channels"] == 3
    assert rgb.train.keywords["is_flow"] is False and rgb.sample_train_params.keywords["scales"] == [1, .875, .75, .66]
    assert rgb.oversample.keywords["scale_size"] == 256 and rgb.center_crop.keywords["crop_size"] == 224
    flow = ssn_models.SSN(5, 2, 5, 2, "Flow", base_model="BNInception", dropout=0).frame_transforms()
    assert flow.train.keywords["mean"] == [128] and flow.train.keywords["frame_channels"] == 10
    assert flow.train.keywords["is_flow"] is True and flow.sample_train_params.keywords["scales"] == [1, .875, .75]


def test_div_true_is_rejected():
    from ops.frame_transforms import train_frames
    import torch
    with pytest.raises(NotImplementedError):
        train_frames(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), [(8, 8, 0, 0, False)], [0.5], [0.2], 3, div=True)


def test_group_to_uint8_stacks_a_pil_group():
    PIL = pytest.importorskip("PIL.Image")
    import torch
    from ops.frame_transforms import GroupToUint8
    a = np.random.default_rng(0).integers(0, 256, (2, 5, 7, 3), dtype=np.uint8)
    out = GroupToUint8()([PIL.fromarray(x) for x in a])
    assert out.dtype == torch.uint8 and np.array_equal(out.numpy(), a)
    out = GroupToUint8()([PIL.fromarray(x[:, :, 0], "L") for x in a])
    assert out.shape == (2, 5, 7, 1) and np.array_equal(out[..., 0].numpy(), a[..., 0])


def _training_sample(video, transform):
    """what SSNDataSet.get_training_data (ssn_dataset.py:455-488) returns for one video: every proposal's frames through the
    transform, then torch.cat over the proposals, next to the per-proposal fields"""
    import torch
    out_frames = [transform(prop) for prop in video]
    return (torch.cat(out_frames), torch.from_numpy(np.array([len(p) for p in video])),
            torch.from_numpy(np.zeros((len(video), 2), np.float32)))


def _pil_videos(sizes, P, n, mode, seed):
    PIL = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(seed)
    c = 3 if mode == "RGB" else 1
    arrays = [[rng.integers(0, 256, (n, h, w, c), dtype=np.uint8) for _ in range(P)] for h, w in sizes]
    pil = [[[PIL.fromarray(x if c == 3 else x[:, :, 0], mode) for x in prop] for prop in v] for v in arrays]
    return arrays, pil


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_dataset_batch_cuts_back_into_proposal_groups(mode):
    """GroupToUint8 through the path SSNDataSet + DataLoader take (torch.cat per video, default_collate over videos):
    proposal_groups gives back each proposal's group, in order"""
    from torch.utils.data import default_collate
    from ops.frame_transforms import GroupToUint8, proposal_groups
    P, n = 4, 3 if mode == "RGB" else 6
    arrays, pil = _pil_videos([(12, 17)] * 3, P, n, mode, 1)
    batch = default_collate([_training_sample(v, GroupToUint8()) for v in pil])
    assert batch[0].shape == (3, P * n, 12, 17, 3 if mode == "RGB" else 1) and batch[0].dtype.is_floating_point is False
    groups = proposal_groups(batch[0], P)
    expect = [g for v in arrays for g in v]
    assert len(groups) == len(expect) == 3 * P
    for g, e in zip(groups, expect):
        assert np.array_equal(g.numpy(), e)


def test_ragged_collate_keeps_each_video():
    from torch.utils.data import DataLoader, default_collate
    from ops.frame_transforms import GroupToUint8, proposal_groups, collate_ragged
    P, n = 2, 3
    arrays, pil = _pil_videos([(12, 17), (17, 12), (20, 20)], P, n, "RGB", 2)
    samples = [_training_sample(v, GroupToUint8()) for v in pil]
    with pytest.raises(RuntimeError):
        default_collate(samples)                   # videos of different resolutions do not stack
    batch = next(iter(DataLoader(samples, batch_size=3, collate_fn=collate_ragged)))
    assert isinstance(batch[0], list) and batch[1].shape == (3, P) and batch[2].shape == (3, P, 2)
    groups = proposal_groups(batch[0], P)
    for g, e in zip(groups, [g for v in arrays for g in v]):
        assert np.array_equal(g.numpy(), e)
    with pytest.raises(ValueError):
        proposal_groups(batch[0], 4)
