"""The GPU frame transforms (csrc/frames.cu, ops/frame_transforms.py) bitwise against the numpy oracle of the reference's PIL
group transforms (oracle/frames_oracle.py) and against the golden cases written from the reference itself."""
import ctypes as C
import hashlib
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import frames_oracle as F
from oracle.gen_golden_frames import frames_for

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RGB_MEAN, FLOW_MEAN = [104, 117, 128], [128]
RGB_SCALES, FLOW_SCALES = [1, .875, .75, .66], [1, .875, .75]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _frames(seed, n, h, w, c):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, c), dtype=np.uint8)


def _cat(outs):
    return np.concatenate([o.reshape(-1) for o in outs])


def _same(gpu, ref):
    g = gpu.reshape(-1).cpu().numpy()
    ref = ref.reshape(-1)
    assert g.shape == ref.shape
    bad = np.flatnonzero(g.view(np.uint32) != ref.view(np.uint32))
    assert bad.size == 0, "%d of %d values differ, first at %d: %r vs %r" % (bad.size, g.size, bad[0], g[bad[0]], ref[bad[0]])


def _train_all(groups, params, is_flow, mean, fc):
    from ops.frame_transforms import train_frames
    out = train_frames([torch.from_numpy(g) for g in groups], params, mean, [1], fc, is_flow=is_flow)
    ref = _cat([F.train_group(list(g), p, 224, mean, [1], is_flow) for g, p in zip(groups, params)])
    return out, ref


@pytest.mark.parametrize("modality", ["RGB", "Flow"])
def test_every_fixed_crop_and_flip_of_a_340x256_frame(modality):
    from ops.frame_transforms import crop_pairs, fill_fix_offset
    _dev()
    flow = modality == "Flow"
    c, n = (1, 2) if flow else (3, 1)
    base = _frames(1, n, 256, 340, c)
    params = [(cw, ch, ox, oy, fl) for cw, ch in crop_pairs(340, 256, 224, FLOW_SCALES if flow else RGB_SCALES)
              for ox, oy in fill_fix_offset(True, 340, 256, cw, ch) for fl in (False, True)]
    out, ref = _train_all([base] * len(params), params, flow, FLOW_MEAN if flow else RGB_MEAN, 2 if flow else 3)
    _same(out, ref)


def test_random_offsets_fix_crop_false():
    from ops.frame_transforms import sample_train_params
    _dev()
    groups = [_frames(10 + i, 2, 256, 340, 3) for i in range(6)]
    params = sample_train_params([(256, 340)] * 6, RGB_SCALES, fix_crop=False, rng=random.Random(3))
    out, ref = _train_all(groups, params, False, RGB_MEAN, 3)
    _same(out, ref)


RAGGED = [(256, 340), (340, 256), (360, 480), (240, 320), (223, 300), (80, 100), (224, 224)]


def test_ragged_sizes_in_one_training_call():
    from ops.frame_transforms import sample_train_params
    _dev()
    groups = [_frames(20 + i, 3, h, w, 3) for i, (h, w) in enumerate(RAGGED)]
    params = sample_train_params(RAGGED, RGB_SCALES, rng=random.Random(0))
    # and explicitly the snapped 224 crop of the 223-row frame at a negative row offset: zero fill
    groups.append(groups[4])
    params.append((224, 224, 38, -1, True))
    out, ref = _train_all(groups, params, False, RGB_MEAN, 3)
    _same(out, ref)


@pytest.mark.parametrize("sizes,c", [([(256, 340), (360, 480), (340, 256), (480, 360), (256, 256), (300, 223)], 3),
                                     ([(256, 340), (360, 480)], 1)])
def test_oversample(sizes, c):
    from ops.frame_transforms import oversample_frames
    _dev()
    n = 4 if c == 1 else 2
    groups = [_frames(40 + i, n, h, w, c) for i, (h, w) in enumerate(sizes)]
    mean = FLOW_MEAN if c == 1 else RGB_MEAN
    out = oversample_frames([torch.from_numpy(g) for g in groups], mean, [1], 2 if c == 1 else 3)
    _same(out, _cat([F.oversample_group(list(g), 224, 256, mean, [1]) for g in groups]))


def test_center_crop_odd_differences():
    from ops.frame_transforms import center_crop_frames
    _dev()
    sizes = [(256, 341), (257, 340), (256, 256), (359, 480), (341, 256), (300, 223)]   # odd (scaled - 224) on either axis
    groups = [_frames(60 + i, 2, h, w, 3) for i, (h, w) in enumerate(sizes)]
    out = center_crop_frames([torch.from_numpy(g).cuda() for g in groups], RGB_MEAN, [1], 3)
    _same(out, _cat([F.center_group(list(g), 224, 256, RGB_MEAN, [1]) for g in groups]))


def test_golden_cases():
    from ops.frame_transforms import train_frames, oversample_frames, center_crop_frames
    _dev()
    gold = np.load(os.path.join(ROOT, "tests", "golden", "frames.npz"))
    for case in json.loads(str(gold["cases"])):
        frames = frames_for(case["seed"], *case["shape"]) if "seed" in case else gold["in_" + case["name"]]
        x = torch.from_numpy(frames)
        c = frames.shape[3]
        if case["kind"] == "train":
            out = train_frames(x, [case["params"]], case["mean"], [1], c, input_size=case["out"], is_flow=case["is_flow"])
        elif case["kind"] == "oversample":
            out = oversample_frames(x, case["mean"], [1], c, crop_size=case["out"], scale_size=case["scale"])
        else:
            out = center_crop_frames(x, case["mean"], [1], c, crop_size=case["out"], scale_size=case["scale"])
        got = out.cpu().numpy().reshape(-1)
        if "seed" in case:
            assert hashlib.sha256(got.tobytes()).hexdigest() == case["sha256"], case["name"]
        else:
            assert got.tobytes() == gold["out_" + case["name"]].tobytes(), case["name"]


def _plan(mode, groups, params=None, c=3):
    from ops.frame_transforms import FramePlan
    dev = _dev()
    return FramePlan(mode, [g.shape[:3] for g in groups], c, 224, 256, RGB_MEAN, [1], False, dev, params)


def test_one_call_equals_per_group_calls_and_repeats_bitwise():
    from ops.frame_transforms import sample_train_params, train_frames
    _dev()
    groups = [torch.from_numpy(_frames(80 + i, 2, h, w, 3)) for i, (h, w) in enumerate(RAGGED)]
    params = sample_train_params(RAGGED, RGB_SCALES, rng=random.Random(9))
    whole = train_frames(groups, params, RGB_MEAN, [1], 3)
    again = train_frames(groups, params, RGB_MEAN, [1], 3)
    parts = torch.cat([train_frames(g, [p], RGB_MEAN, [1], 3) for g, p in zip(groups, params)])
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))
    assert torch.equal(whole.view(torch.int32), again.view(torch.int32))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_output_and_workspace_prefilled_with_ones_are_overwritten(mode):
    groups = [_frames(90 + i, 2, h, w, 3) for i, (h, w) in enumerate([(360, 480), (256, 340), (240, 320)])]
    params = [(224, 224, 3, 5, True), (192, 224, 0, 16, False), (200, 200, 40, 20, True)] if mode == 0 else None
    plan = _plan(mode, groups, params)
    plan.workspace.fill_(0xFF)
    dst = torch.full((plan.dst_floats,), -1, dtype=torch.int32, device=plan.device).view(torch.float32)   # 0xFFFFFFFF: NaN
    src = torch.from_numpy(np.concatenate([g.reshape(-1) for g in groups])).to(plan.device)
    plan.run(src, dst)
    if mode == 0:
        ref = _cat([F.train_group(list(g), p, 224, RGB_MEAN, [1], False) for g, p in zip(groups, params)])
    elif mode == 1:
        ref = _cat([F.oversample_group(list(g), 224, 256, RGB_MEAN, [1]) for g in groups])
    else:
        ref = _cat([F.center_group(list(g), 224, 256, RGB_MEAN, [1]) for g in groups])
    _same(dst, ref)


def test_cuda_graph_replay_with_new_frames_and_parameters():
    from ops.frame_transforms import sample_train_params, train_frames
    dev = _dev()
    sizes = [(256, 340)] * 4 + [(360, 480)] * 2
    first = [_frames(100 + i, 3, h, w, 3) for i, (h, w) in enumerate(sizes)]
    plan = _plan(0, first, sample_train_params(sizes, RGB_SCALES, rng=random.Random(1)))
    src = torch.from_numpy(np.concatenate([g.reshape(-1) for g in first])).to(dev)
    dst = torch.empty(plan.dst_floats, dtype=torch.float32, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(src, dst)                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run(src, dst)
    second = [_frames(200 + i, 3, h, w, 3) for i, (h, w) in enumerate(sizes)]
    params = sample_train_params(sizes, RGB_SCALES, rng=random.Random(2))
    src.copy_(torch.from_numpy(np.concatenate([x.reshape(-1) for x in second])))
    plan.set_train_params(params)
    g.replay()
    torch.cuda.synchronize()
    eager = train_frames([torch.from_numpy(x) for x in second], params, RGB_MEAN, [1], 3)
    assert torch.equal(dst.view(torch.int32), eager.reshape(-1).view(torch.int32))


def test_rejected_arguments_launch_nothing():
    from ssn_b200._lib import lib
    groups = [_frames(300, 2, 256, 340, 3)]
    plan = _plan(0, groups, [(224, 224, 0, 0, False)])
    src = torch.from_numpy(groups[0].reshape(-1)).to(plan.device)
    dst = torch.full((plan.dst_floats,), 7.0, device=plan.device)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    before = lib.ssnb_global_launch_count()

    def call(**kw):
        a = dict(groups=plan.groups, src_bytes=src.numel(), dst_floats=dst.numel(), ws=plan.workspace.numel(), groups_dev=plan.groups_dev.data_ptr())
        a.update(kw)
        return lib.ssnb_frame_transform(C.byref(plan.cfg), a["groups"], a["groups_dev"], len(plan.groups), src.data_ptr(), a["src_bytes"],
                                        dst.data_ptr(), a["dst_floats"], plan.workspace.data_ptr(), a["ws"], stream)

    assert call(src_bytes=src.numel() - 1) == 1
    assert call(dst_floats=dst.numel() - 1) == 1
    assert call(groups_dev=None) == 1
    plan.groups[0].dst_offset = 1                  # not the layout ssnb_frame_transform_workspace_bytes assigned
    assert call() == 1
    plan.groups[0].dst_offset = 0
    plan.groups[0].crop_w = 0
    assert call() == 1
    torch.cuda.synchronize()
    assert lib.ssnb_global_launch_count() == before
    assert bool((dst == 7.0).all())


# ---- end to end: the model sees the same frames ----------------------------------------------------------------------------------
def _ssn(test_mode=False):
    import ssn_models
    from oracle import synth
    from ssn_b200 import _lib
    K = 4
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0, test_mode=test_mode)
    sd = m.state_dict()
    for k, v in synth.synth_backbone(3, seed=0, calib_frames=2).items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1).items():
        if k in sd:
            sd[k].copy_(v)
    m = m.to(_dev())
    m = m.eval() if test_mode else m.train()
    m.set_precision(_lib.EXACT_TC, 1024.0)
    return m


def test_fused_step_on_gpu_frames_equals_oracle_frames():
    from oracle import synth
    dev = _dev()
    tf = _ssn().frame_transforms()
    props = [_frames(400 + i, 9, 256, 340, 3) for i in range(16)]          # 2 videos x 8 proposals x 9 segments
    params = tf.sample_train_params([(256, 340)] * 16, rng=random.Random(4))
    x_gpu = tf.train([torch.from_numpy(p) for p in props], params)
    x_ref = torch.from_numpy(_cat([F.train_group(list(p), q, 224, RGB_MEAN, [1], False) for p, q in zip(props, params)])).to(dev)
    _same(x_gpu, x_ref.cpu().numpy())
    _, sc, tgt, rtgt, ptype = [t.to(dev) for t in synth.synth_batch(2, 4, 3, seed=5)]
    res = []
    for x in (x_gpu, x_ref):
        m = _ssn()
        losses = m.fused_step(x.reshape(2, -1, 224, 224), sc, tgt, rtgt, ptype).clone()
        res.append((losses, m.base_model.conv1_7x7_s2.weight.grad.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_test_scores_on_gpu_frames_equals_oracle_frames():
    dev = _dev()
    m = _ssn(test_mode=True)
    m.prepare_test_fc()
    tf = m.frame_transforms()
    ticks = _frames(500, 8, 360, 480, 3)
    x_gpu = tf.oversample(torch.from_numpy(ticks))
    x_ref = torch.from_numpy(F.oversample_group(list(ticks), 224, 256, RGB_MEAN, [1])).to(dev)
    _same(x_gpu, x_ref.cpu().numpy())
    a = m.test_scores(x_gpu, 10)
    b = m.test_scores(x_ref.view(-1, 3, 224, 224), 10)
    assert torch.equal(a, b)


def test_dataset_batch_through_proposal_groups_without_synchronising():
    """SSNDataSet's batch layout (each video's proposals torch.cat'ed, videos default-collated) cut back into proposal groups
    and transformed in one call: one crop / flip draw per proposal, bitwise the oracle's, and neither the call nor the
    10-crop / 1-crop calls synchronise the device"""
    from torch.utils.data import default_collate
    from ops.frame_transforms import proposal_groups, sample_train_params, train_frames, oversample_frames, center_crop_frames
    dev = _dev()
    P, n = 8, 9
    videos = [[_frames(600 + 10 * v + p, n, 256, 340, 3) for p in range(P)] for v in range(2)]
    frames = default_collate([torch.cat([torch.from_numpy(p) for p in v]) for v in videos])       # [2, P * n, H, W, C]
    groups = proposal_groups(frames, P)
    params = sample_train_params([g.shape[1:3] for g in groups], RGB_SCALES, rng=random.Random(6))
    cuda_groups = [g.to(dev) for g in groups]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        x = train_frames(groups, params, RGB_MEAN, [1], 3)
        x_dev = train_frames(cuda_groups, params, RGB_MEAN, [1], 3)
        o = oversample_frames(cuda_groups[:2], RGB_MEAN, [1], 3)
        c = center_crop_frames(groups[:2], RGB_MEAN, [1], 3)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert x.shape == (2 * P * n, 3, 224, 224)
    ref = _cat([F.train_group(list(p), q, 224, RGB_MEAN, [1], False) for p, q in zip([p for v in videos for p in v], params)])
    _same(x, ref)
    _same(x_dev, ref)
    _same(o, _cat([F.oversample_group(list(g.numpy()), 224, 256, RGB_MEAN, [1]) for g in groups[:2]]))
    _same(c, _cat([F.center_group(list(g.numpy()), 224, 256, RGB_MEAN, [1]) for g in groups[:2]]))
