"""The GPU JPEG decode (csrc/jpeg.cu, ops/jpeg.py) bitwise against what Pillow decoded (tests/golden/jpeg.npz) and against the
numpy oracle (oracle/jpeg_oracle.py) on seeded batches, and end to end through the frame transforms and the training step."""
import hashlib
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import frames_oracle as F
from oracle import jpeg_oracle as J
from oracle.gen_golden_jpeg import content, encode

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
CASES = json.loads(str(GOLDEN["cases"]))["cases"]
RGB_MEAN = [104, 117, 128]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def jpg(name):
    return GOLDEN["jpg_" + name].tobytes()


def _same(gpu, ref, what=""):
    g = gpu.cpu().numpy()
    assert g.shape == ref.shape, (what, g.shape, ref.shape)
    bad = np.flatnonzero(g.reshape(-1) != ref.reshape(-1))
    assert bad.size == 0, "%s: %d of %d bytes differ, first at %d" % (what, bad.size, g.size, bad[0])


def test_every_golden_case_in_one_call():
    from ops.jpeg import decode_jpeg
    _dev()
    groups = [[jpg(c["name"])] for c in CASES for _ in (0, 1)]
    modes = ["RGB", "L"] * len(CASES)
    out = decode_jpeg(groups, mode=modes)
    for k, (c, mode) in enumerate(zip([c for c in CASES for _ in (0, 1)], modes)):
        px = out[k][0].cpu().numpy()
        if "sha256_" + mode in c:
            assert hashlib.sha256(px.tobytes()).hexdigest() == c["sha256_" + mode], (c["name"], mode)
        else:
            _same(out[k][0], GOLDEN["px_%s_%s" % (mode, c["name"])], c["name"] + " " + mode)


def _stream(w, h, sub, kind, seed, **kw):
    return encode(content(kind, w, h, 1 if sub == "gray" else 3, seed), sub, **kw)


def test_ragged_call_equals_per_image_calls_and_the_oracle():
    from ops.jpeg import decode_jpeg
    _dev()
    rng = np.random.default_rng(3)
    specs = []
    for i in range(24):
        w, h = int(rng.integers(1, 200)), int(rng.integers(1, 150))
        sub = ["444", "422", "420", "gray"][i % 4]
        kw = dict(quality=int(rng.choice([5, 50, 75, 90, 95, 100])))
        if i % 5 == 0:
            kw["restart_marker_blocks"] = int(rng.integers(1, 4))
        if i % 7 == 0:
            kw["optimize"] = True
        specs.append((_stream(w, h, sub, ["noise", "smooth", "checker", "saturated"][i % 4], 100 + i, **kw), "RGB" if i % 3 else "L"))
    groups = [[s] * (1 + i % 3) for i, (s, _) in enumerate(specs)]
    modes = [m for _, m in specs]
    together = decode_jpeg(groups, mode=modes)
    for i, ((s, m), g) in enumerate(zip(specs, together)):
        ref = J.decode(s, m)
        alone = decode_jpeg([[s]], mode=m)[0]
        _same(alone[0], ref, "alone %d" % i)
        for k in range(g.shape[0]):
            _same(g[k], ref, "together %d.%d" % (i, k))


def test_400_frames_at_340x256_equal_the_oracle_and_repeat_bitwise():
    from ops.jpeg import decode_jpeg
    _dev()
    # 50 distinct streams (4:2:0 q95, as frame extractors write) at shuffled positions in one 400-image call
    streams = [_stream(340, 256, "420", "smooth" if i % 2 else "noise", 500 + i, quality=95) for i in range(50)]
    order = np.random.default_rng(0).permutation(np.arange(400) % 50)
    blobs = [[streams[k] for k in order]]
    a = decode_jpeg(blobs)[0]
    b = decode_jpeg(blobs)[0]
    assert a.shape == (400, 256, 340, 3)
    assert torch.equal(a, b)
    refs = [J.decode(s) for s in streams]
    for j, k in enumerate(order):
        _same(a[j], refs[k], "frame %d" % j)


@pytest.mark.parametrize("poison", [0x00, 0xA5, 0xFF])
def test_output_and_workspace_prefilled_with_poison_are_overwritten(poison):
    from ops.jpeg import JpegPlan
    dev = _dev()
    blobs = [jpg(c["name"]) for c in CASES[::5]]
    ends = np.cumsum([len(b) for b in blobs])
    plan = JpegPlan(np.frombuffer(b"".join(blobs), np.uint8), ends - [len(b) for b in blobs], ends,
                    [3 if i % 2 else 1 for i in range(len(blobs))])
    d = plan.upload(dev)
    out = torch.full((plan.out_bytes,), poison, dtype=torch.uint8, device=dev)
    ws = torch.full((plan.workspace_bytes,), poison, dtype=torch.uint8, device=dev)
    status = torch.full((len(blobs),), -7, dtype=torch.int32, device=dev)
    plan.run(d, out, status, ws)
    assert (status.cpu() == 0).all()
    for i, b in enumerate(blobs):
        im = plan.images[i]
        n = im.width * im.height * im.channels
        _same(out[im.out_offset:im.out_offset + n].view(im.height, im.width, im.channels), J.decode(b, "RGB" if i % 2 else "L"), str(i))


def _corrupt(b):
    """the scan's middle overwritten by 8 stuffed 0xFF bytes: 64 one bits, which no Huffman code of Pillow's tables reads"""
    hdr = J.parse(b)
    mid = (hdr["scan"] + len(b)) // 2
    return b[:mid] + b"\xff\x00" * 8 + b[mid + 16:]


def test_corrupt_and_truncated_segments_get_their_status_and_spare_the_rest():
    from ops.jpeg import decode_jpeg, STATUS_TEXT
    _dev()
    good = [_stream(340, 256, "420", "smooth", 700 + i, quality=95) for i in range(4)]
    bad_code = _corrupt(good[1])
    cut = good[2][:len(good[2]) * 3 // 5]
    rst = _stream(96, 64, "444", "noise", 710, quality=90, restart_marker_blocks=2)
    h = J.parse(rst)
    k = rst.index(b"\xff\xd3", h["scan"])
    rst_bad = rst[:k] + b"\xff\xd6" + rst[k + 2:]                  # RST3 where it belongs replaced by RST6
    call = [good[0], bad_code, good[3], cut, rst_bad, good[0]]
    refs = [J.decode(s, with_status=True) for s in call]
    assert [r[1] for r in refs] == [0, J.BAD_CODE, 0, J.TRUNCATED, J.BAD_RESTART, 0]
    groups, status = decode_jpeg([[s] for s in call], check=False)
    assert status.cpu().tolist() == [r[1] for r in refs]
    for i, (g, (px, _)) in enumerate(zip(groups, refs)):
        _same(g[0], px, "image %d" % i)                # corrupt images too: zeros from the first bad block, as the oracle
    with pytest.raises(ValueError, match=r"decode_jpeg: image 1 \(group 1, image 0\): " + STATUS_TEXT[J.BAD_CODE]):
        decode_jpeg([[s] for s in call])
    with pytest.raises(ValueError, match=r"image 1 \(group 0, image 1\): " + STATUS_TEXT[J.TRUNCATED]):
        decode_jpeg([[good[0], cut]])


# ---- end to end: bytes -> decode -> frame transforms -> the model ------------------------------------------------------------------
def _ssn():
    import ssn_models
    from oracle import synth
    from ssn_b200 import _lib
    K = 4
    m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0)
    sd = m.state_dict()
    for k, v in synth.synth_backbone(3, seed=0, calib_frames=2).items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1).items():
        if k in sd:
            sd[k].copy_(v)
    m = m.to(_dev()).train()
    m.set_precision(_lib.EXACT_TC, 1024.0)
    return m


def test_bytes_through_decode_proposal_groups_train_and_oversample_frames():
    from ops.frame_transforms import proposal_groups, oversample_frames
    from ops.jpeg import GroupToJpegBytes, collate_jpeg
    dev = _dev()
    tf = _ssn().frame_transforms()
    P, n = 2, 9
    files = [[_stream(340, 256, "420", "smooth", 900 + 20 * v + k, quality=95) for k in range(P * n)] for v in range(2)]
    # the data set: one packed tensor per proposal, torch.cat per video; the loader: collate_jpeg
    samples = [(torch.cat([GroupToJpegBytes()(f[p * n:(p + 1) * n]) for p in range(P)]), torch.tensor(v)) for v, f in enumerate(files)]
    frames, _ = collate_jpeg(samples)
    decoded = tf.decode(frames)
    groups = proposal_groups(decoded, props_per_video=P)
    ref_groups = [np.stack([J.decode(s) for s in f[p * n:(p + 1) * n]]) for f in files for p in range(P)]
    params = tf.sample_train_params([(256, 340)] * len(groups), rng=random.Random(2))
    x = tf.train(groups, params)
    ref = np.concatenate([F.train_group(list(g), q, 224, RGB_MEAN, [1], False).reshape(-1) for g, q in zip(ref_groups, params)])
    assert x.cpu().numpy().reshape(-1).view(np.uint32).tolist() == ref.view(np.uint32).tolist()
    o = oversample_frames(decoded[0][:4], RGB_MEAN, [1], 3)
    ref_o = F.oversample_group(list(ref_groups[0][:4]), 224, 256, RGB_MEAN, [1])
    assert o.cpu().numpy().tobytes() == ref_o.tobytes()
    # Flow: x, y planes decoded as L
    flow = [_stream(340, 256, "gray", "smooth", 950 + k, quality=90) for k in range(10)]
    fl = decode_jpeg_l(flow)
    _same(fl, np.stack([J.decode(s, "L") for s in flow]), "flow")


def decode_jpeg_l(blobs):
    import ssn_models
    tf = ssn_models.SSN(4, 2, 5, 2, "Flow", base_model="BNInception", dropout=0).frame_transforms()
    return tf.decode([blobs])[0]


def test_fused_step_on_decoded_frames_equals_oracle_frames():
    from oracle import synth
    dev = _dev()
    tf = _ssn().frame_transforms()
    files = [[_stream(340, 256, "420", "smooth", 1000 + 9 * g + k, quality=95) for k in range(9)] for g in range(16)]
    decoded = tf.decode(files)
    ref = [np.stack([J.decode(s) for s in f]) for f in files]
    params = tf.sample_train_params([(256, 340)] * 16, rng=random.Random(4))
    x_gpu = tf.train(decoded, params)
    x_ref = tf.train([torch.from_numpy(r) for r in ref], params)
    assert torch.equal(x_gpu, x_ref)
    _, sc, tgt, rtgt, ptype = [t.to(dev) for t in synth.synth_batch(2, 4, 3, seed=5)]
    res = []
    for x in (x_gpu, x_ref):
        m = _ssn()
        losses = m.fused_step(x.reshape(2, -1, 224, 224), sc, tgt, rtgt, ptype).clone()
        res.append((losses, m.base_model.conv1_7x7_s2.weight.grad.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
