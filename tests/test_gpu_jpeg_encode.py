"""JPEG encode on the H100 (csrc/jpeg_encode.cu) byte for byte against Pillow: every golden fixture, ragged calls of 500+
images per mode, each image alone against the batch, repeats over a 0xFF-filled workspace and output and a CUDA-graph
replay, the round trip through decode_jpeg, and write_flow_jpegs / write_frame_jpegs from CUDA against host arrays."""
import io
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_encode_oracle as E
from oracle.gen_golden_jpeg_encode import image, pillow

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode.npz"))
SPECS = [(m, k, int(h), int(w), int(s), int(q)) for m, k, h, w, s, q in GOLD["specs"]]
DEV = torch.device("cuda:0")


def _cuda(img):
    return torch.from_numpy(np.ascontiguousarray(img)).to(DEV)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_golden_fixtures(mode):
    from ops.jpeg import encode_jpeg
    by_q = {}
    for i, (m, kind, h, w, seed, q) in enumerate(SPECS):
        if m == mode:
            by_q.setdefault(q, []).append(i)
    for q, idx in sorted(by_q.items()):              # one ragged call per quality
        got = encode_jpeg([_cuda(image(*SPECS[i][:5])) for i in idx], mode=mode, quality=q)
        for i, g in zip(idx, got):
            assert g == GOLD["jpg_" + str(GOLD["names"][i])].tobytes(), str(GOLD["names"][i])


def _ragged(mode, n, seed):
    rng = np.random.default_rng(seed)
    C = E.MODES[mode]
    special = [(1, 1), (1, 2000), (2000, 1), (16, 16), (17, 33), (256, 340), (360, 480), (8, 65)]
    out = []
    for i in range(n):
        h, w = special[i] if i < len(special) else (int(rng.integers(1, 120)), int(rng.integers(1, 160)))
        kind = ["noise", "flow", "ramp", "checker", "const255"][i % 5]
        out.append(E.fixture(kind, h, w, C, seed * 1000 + i))
    return out


@pytest.mark.parametrize("mode,quality", [("L", 95), ("RGB", 90)])
def test_ragged_call_equals_pillow_and_each_image_alone(mode, quality):
    from ops.jpeg import encode_jpeg
    imgs = _ragged(mode, 520, 1 if mode == "L" else 2)
    got = encode_jpeg([_cuda(a) for a in imgs], mode=mode, quality=quality)
    assert len(got) == len(imgs)
    for i, (a, g) in enumerate(zip(imgs, got)):
        assert g == pillow(a, mode, quality), (i, a.shape)
    for i, a in enumerate(imgs):
        assert encode_jpeg([_cuda(a)], mode=mode, quality=quality)[0] == got[i], i


def test_repeat_poisoned_buffers_and_graph_replay():
    from ops.jpeg import JpegEncodePlan
    imgs = _ragged("RGB", 40, 3)
    want = [pillow(a, "RGB", 75) for a in imgs]
    plan = JpegEncodePlan([a.shape[:2] for a in imgs], "RGB", 75, DEV)
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
    # capture on new pixels of the same sizes, then replay on others copied into the captured inputs
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
    g.replay()
    assert plan.files() == [pillow(o, "RGB", 75) for o in other]
    for x, a in zip(xs, imgs):
        x.copy_(_cuda(a))
    g.replay()
    assert plan.files() == want


def test_batched_tensor_and_round_trip_through_decode():
    from PIL import Image
    from ops.jpeg import decode_jpeg, encode_jpeg
    planes = np.stack([E.fixture("flow", 256, 340, 1, s) for s in range(6)])
    frames = np.stack([E.fixture("ramp", 256, 340, 3, 0), E.fixture("noise", 256, 340, 3, 1), E.fixture("flow", 256, 340, 3, 2)])
    for arr, mode in ((planes, "L"), (frames, "RGB")):
        files = encode_jpeg(_cuda(arr), mode=mode, quality=95)
        assert files == [pillow(a, mode, 95) for a in arr]
        dec = decode_jpeg([files], mode=mode)[0].cpu().numpy()
        want = np.stack([np.asarray(Image.open(io.BytesIO(f)).convert(mode)).reshape(arr.shape[1:]) for f in files])
        assert dec.tobytes() == want.tobytes()


def test_write_flow_and_frame_jpegs_from_cuda_equal_host(tmp_path):
    from ops.optical_flow import write_flow_jpegs, write_frame_jpegs
    planes = np.stack([E.fixture("flow", 40, 56, 1, s) for s in range(10)])
    frames = np.stack([E.fixture("noise" if s % 2 else "ramp", 40, 56, 3, s) for s in range(7)])
    dev_f = write_flow_jpegs(_cuda(planes), [str(tmp_path / "g" / "a"), str(tmp_path / "g" / "b")], offsets=[0, 4, 7])
    host_f = write_flow_jpegs(planes, [str(tmp_path / "h" / "a"), str(tmp_path / "h" / "b")], offsets=[0, 4, 7])
    dev_r = write_frame_jpegs(_cuda(frames), [str(tmp_path / "g" / "a"), str(tmp_path / "g" / "b")], offsets=[0, 4, 7])
    host_r = write_frame_jpegs(frames, [str(tmp_path / "h" / "a"), str(tmp_path / "h" / "b")], offsets=[0, 4, 7])
    for d, h in zip(dev_f + dev_r, host_f + host_r):
        assert os.path.relpath(d, tmp_path / "g") == os.path.relpath(h, tmp_path / "h")
        assert open(d, "rb").read() == open(h, "rb").read(), d
    assert len(dev_f) == 10 and len(dev_r) == 7
