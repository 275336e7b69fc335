"""JPEG encode with restart intervals on the H100 (csrc/jpeg_encode.cu), byte for byte against Pillow: every golden fixture, a
ragged call of about 200 images in both modes under both options against Pillow and against the same call permuted,
thinned and alone, restart 0 through the new entry against the existing entry, repeats over 0xFF-filled buffers and a
CUDA-graph replay, decode_jpeg of the marked files (one thread per interval) against Pillow, the marker-free files and
jpeg_roundtrip, and write_frame_jpegs / write_flow_jpegs from CUDA against the Pillow path."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_encode_oracle as E
from oracle import jpeg_restart_oracle as R
from oracle.gen_golden_jpeg_restart import image, pillow

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_restart.npz"))
SPECS = [(m, k, int(h), int(w), int(s), int(q), int(b), int(r)) for m, k, h, w, s, q, b, r in GOLD["specs"]]
DEV = torch.device("cuda:0")
OPTIONS = [dict(restart_marker_blocks=1), dict(restart_marker_blocks=7), dict(restart_marker_rows=1), dict(restart_marker_rows=2)]


def _cuda(img):
    return torch.from_numpy(np.ascontiguousarray(img)).to(DEV)


def _rb_rr(kw):
    return kw.get("restart_marker_blocks", 0), kw.get("restart_marker_rows", 0)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_golden_fixtures(mode):
    from ops.jpeg import encode_jpeg
    calls = {}
    for i, (m, kind, h, w, seed, q, rb, rr) in enumerate(SPECS):
        if m == mode:
            calls.setdefault((q, rb, rr), []).append(i)
    for (q, rb, rr), idx in sorted(calls.items()):             # one ragged call per quality and option
        got = encode_jpeg([_cuda(image(*SPECS[i][:5])) for i in idx], mode=mode, quality=q, restart_marker_blocks=rb,
                          restart_marker_rows=rr)
        for i, g in zip(idx, got):
            assert g == GOLD["jpg_" + str(GOLD["names"][i])].tobytes(), str(GOLD["names"][i])


def _ragged(mode, n, seed):
    rng = np.random.default_rng(seed)
    C_ = E.MODES[mode]
    special = [(1, 1), (720, 1280), (17, 9), (37, 23), (256, 340), (360, 480), (8, 65), (1, 1280), (720, 1), (16, 16)]
    out = []
    for i in range(n):
        h, w = special[i] if i < len(special) else (int(rng.integers(1, 200)), int(rng.integers(1, 260)))
        kind = ["noise", "flow", "ramp", "checker", "const128"][i % 5]
        out.append(E.fixture(kind, h, w, C_, seed * 1000 + i))
    return out


@pytest.mark.parametrize("mode,quality", [("L", 95), ("RGB", 90)])
def test_ragged_call_equals_pillow_permuted_thinned_and_alone(mode, quality):
    from ops.jpeg import encode_jpeg
    imgs = _ragged(mode, 200, 5 if mode == "L" else 6)
    xs = [_cuda(a) for a in imgs]
    perm = np.random.default_rng(0).permutation(len(imgs))
    for kw in OPTIONS:
        got = encode_jpeg(xs, mode=mode, quality=quality, **kw)
        assert len(got) == len(imgs)
        for i, (a, g) in enumerate(zip(imgs, got)):
            assert g == pillow(a, mode, quality, *_rb_rr(kw)), (kw, i, a.shape)
        pg = encode_jpeg([xs[j] for j in perm], mode=mode, quality=quality, **kw)
        assert all(pg[k] == got[j] for k, j in enumerate(perm)), kw
        thin = encode_jpeg(xs[1::3], mode=mode, quality=quality, **kw)
        assert thin == got[1::3], kw
        for i in range(0, len(imgs), 7):
            assert encode_jpeg([xs[i]], mode=mode, quality=quality, **kw)[0] == got[i], (kw, i)


def test_restart_zero_through_the_new_entry_equals_the_existing_entry():
    from ops.jpeg import JpegEncodePlan
    from ssn_b200._lib import lib
    for mode in ("L", "RGB"):
        imgs = _ragged(mode, 60, 9)
        xs = [_cuda(a) for a in imgs]
        plan = JpegEncodePlan([a.shape[:2] for a in imgs], mode, 95, DEV)      # the new entry with both options 0
        plan.run(xs)
        new = plan.files()
        out = torch.full_like(plan.out, 0xFF)
        ws = torch.full_like(plan.workspace, 0xFF)
        lengths = torch.zeros_like(plan.lengths)
        src = torch.cat([x.reshape(-1) for x in xs])
        rc = lib.ssnb_jpeg_encode(plan._code, 95, src.data_ptr(), src.numel(), plan.images, plan.images_dev.data_ptr(), len(imgs),
                                  out.data_ptr(), out.numel(), lengths.data_ptr(), ws.data_ptr(), ws.numel(),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        lens = lengths.cpu().numpy()
        old = [out[int(o):int(o) + int(n)].cpu().numpy().tobytes() for o, n in zip(plan.slots, lens)]
        assert new == old == [pillow(a, mode, 95) for a in imgs], mode


@pytest.mark.parametrize("kw", [dict(restart_marker_blocks=3), dict(restart_marker_rows=1)])
def test_repeat_poisoned_buffers_and_graph_replay(kw):
    from ops.jpeg import JpegEncodePlan
    imgs = _ragged("RGB", 40, 3)
    want = [pillow(a, "RGB", 75, *_rb_rr(kw)) for a in imgs]
    plan = JpegEncodePlan([a.shape[:2] for a in imgs], "RGB", 75, DEV, **kw)
    xs = [_cuda(a) for a in imgs]
    plan.run(xs)
    assert plan.files() == want
    plan.run(xs)
    assert plan.files() == want
    plan.workspace.fill_(0xFF)
    plan.out.fill_(0xFF)
    plan.lengths.fill_(-1)
    plan.run(xs)
    assert plan.files() == want
    other = [E.fixture("noise", a.shape[0], a.shape[1], 3, 77 + i) for i, a in enumerate(imgs)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(xs)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run(xs)
    for x, o in zip(xs, other):
        x.copy_(_cuda(o))
    plan.out.fill_(0xFF)
    plan.workspace.fill_(0xFF)
    g.replay()
    assert plan.files() == [pillow(o, "RGB", 75, *_rb_rr(kw)) for o in other]
    for x, a in zip(xs, imgs):
        x.copy_(_cuda(a))
    g.replay()
    assert plan.files() == want


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_decode_of_marked_files(mode):
    from PIL import Image
    from ops.jpeg import JpegPlan, decode_jpeg, encode_jpeg, jpeg_roundtrip, _group
    sizes = [(256, 340), (37, 23), (17, 9), (360, 480), (1, 1), (8, 72)]
    C_ = E.MODES[mode]
    for h, w in sizes:
        arr = np.stack([E.fixture(k, h, w, C_, s) for s, k in enumerate(("noise", "flow", "ramp", "const128"))])
        x = _cuda(arr)
        plain = decode_jpeg([encode_jpeg(x, mode=mode, quality=95)], mode=mode)[0]
        rt = jpeg_roundtrip(x, mode=mode, quality=95)
        assert torch.equal(plain, rt), (mode, h, w)
        for kw in OPTIONS:
            files = encode_jpeg(x, mode=mode, quality=95, **kw)
            dec = decode_jpeg([files], mode=mode)[0]
            want = np.stack([np.asarray(Image.open(io.BytesIO(f)).convert(mode)).reshape(arr.shape[1:]) for f in files])
            assert dec.cpu().numpy().tobytes() == want.tobytes(), (mode, h, w, kw)
            assert torch.equal(dec, plain) and torch.equal(dec, rt), (mode, h, w, kw)
            buf, starts, ends = _group(files)
            plan = JpegPlan(buf, starts, ends, [C_] * len(files))
            Rv = R.interval(mode, h, w, *_rb_rr(kw))
            mx, my, _ = E.geometry(mode, h, w)
            for info in plan.images:
                assert info.restart_interval == Rv and info.intervals == -(-(mx * my) // Rv), (mode, h, w, kw)


@pytest.mark.parametrize("kw", OPTIONS)
def test_write_flow_and_frame_jpegs_from_cuda_equal_host(tmp_path, kw):
    from ops.optical_flow import write_flow_jpegs, write_frame_jpegs
    planes = np.stack([E.fixture("flow", 40, 56, 1, s) for s in range(10)])
    frames = np.stack([E.fixture("noise" if s % 2 else "ramp", 40, 56, 3, s) for s in range(7)])
    g, h = tmp_path / "g", tmp_path / "h"
    dev_f = write_flow_jpegs(_cuda(planes), [str(g / "a"), str(g / "b")], offsets=[0, 4, 7], **kw)
    host_f = write_flow_jpegs(planes, [str(h / "a"), str(h / "b")], offsets=[0, 4, 7], **kw)
    dev_r = write_frame_jpegs(_cuda(frames), [str(g / "a"), str(g / "b")], offsets=[0, 4, 7], **kw)
    host_r = write_frame_jpegs(frames, [str(h / "a"), str(h / "b")], offsets=[0, 4, 7], **kw)
    assert len(dev_f) == 10 and len(dev_r) == 7
    for d, hp in zip(dev_f + dev_r, host_f + host_r):
        assert os.path.relpath(d, g) == os.path.relpath(hp, h)
        assert open(d, "rb").read() == open(hp, "rb").read(), d
    assert b"\xff\xdd" in open(dev_r[0], "rb").read()
