"""Frame resize on the H100 (csrc/frame_resize.cu) bitwise against cv2.resize(INTER_LINEAR): every golden fixture; 200
ragged videos of random sizes from 1 x 1 to 1920 x 1080 against the oracle and, where cv2 imports, cv2 frame by frame;
each video's output against the same call permuted and thinned; a repeat, a 0xFF-filled output and CUDA-graph replay on
new pixels; and DenseFlow's extraction end to end: videos of three sizes through one resize_frames, one tvl1_flow and
flow_planes against each video resized and solved alone, and write_frame_jpegs of the resized frames against Pillow's
files of cv2's frames."""
import io
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import frame_resize_oracle as R
from oracle import gen_golden_frame_resize as G

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


def _ragged(rng, n_videos, max_hw=(1080, 1920), max_frames=40):
    """n_videos random uint8 videos: sides log-uniform in 1 .. max, so most are small and a few near 1080p"""
    out = []
    for _ in range(n_videos):
        h, w = (int(np.exp(rng.uniform(0, np.log(m + 1)))) for m in max_hw)
        h, w = min(max(h, 1), max_hw[0]), min(max(w, 1), max_hw[1])
        out.append(rng.integers(0, 256, (int(rng.integers(1, max_frames + 1)), h, w, 3), dtype=np.uint8))
    return out


def test_every_golden_fixture():
    from ops.optical_flow import resize_frames
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frame_resize.npz"))
    by_dst = {}
    for spec in G.fixtures():
        by_dst.setdefault(spec[4:], []).append(spec)
    for (dh, dw), specs in by_dst.items():
        imgs = [G.image(*s[:4]) for s in specs]
        frames, off = resize_frames([_cuda(a[None]) for a in imgs], width=dw, height=dh)
        assert list(off) == list(range(len(specs) + 1))
        got = frames.cpu().numpy()
        for s, a, o in zip(specs, imgs, got):
            n = G.name(*s)
            assert zlib.crc32(a.tobytes()) == int(g["crc_" + n]), ("input drifted", n)
            assert zlib.crc32(o.tobytes()) == int(g["ocrc_" + n]), n
            if "out_" + n in g.files:
                assert o.tobytes() == g["out_" + n].tobytes(), n
        # and each fixture alone
        for s, a, o in zip(specs[::7], imgs[::7], got[::7]):
            assert resize_frames([_cuda(a[None])], width=dw, height=dh)[0][0].cpu().numpy().tobytes() == o.tobytes(), G.name(*s)


def test_ragged_videos_against_the_oracle_and_cv2():
    from ops.optical_flow import resize_frames
    rng = np.random.default_rng(0)
    videos = _ragged(rng, 198)
    videos.insert(17, rng.integers(0, 256, (1, 1, 1, 3), dtype=np.uint8))
    videos.insert(101, rng.integers(0, 256, (3, 1080, 1920, 3), dtype=np.uint8))
    cv2 = _cv2()
    for dh, dw in ((72, 96), (256, 340)):
        sub = videos if (dh, dw) == (72, 96) else videos[::8]
        frames, off = resize_frames([_cuda(v) for v in sub], width=dw, height=dh)
        got = frames.cpu().numpy()
        assert list(off) == list(np.cumsum([0] + [len(v) for v in sub]))
        for k, v in enumerate(sub):
            mine = got[off[k]:off[k + 1]]
            assert mine.tobytes() == R.resize(v, dw, dh).tobytes(), (k, v.shape, dh, dw)
            if cv2 is not None:
                assert mine.tobytes() == np.stack([cv2.resize(f, (dw, dh), interpolation=cv2.INTER_LINEAR) for f in v]).tobytes(), \
                    (k, v.shape, dh, dw)


def test_each_video_independent_of_the_call():
    from ops.optical_flow import resize_frames
    rng = np.random.default_rng(1)
    videos = [_cuda(v) for v in _ragged(rng, 40, max_hw=(720, 1280), max_frames=6)]
    frames, off = resize_frames(videos)
    full = [frames[off[k]:off[k + 1]].cpu().numpy().tobytes() for k in range(len(videos))]
    perm = rng.permutation(len(videos))
    frames, off = resize_frames([videos[k] for k in perm])
    for j, k in enumerate(perm):
        assert frames[off[j]:off[j + 1]].cpu().numpy().tobytes() == full[k], ("permuted", k)
    keep = sorted(rng.choice(len(videos), 9, replace=False))
    frames, off = resize_frames([videos[k] for k in keep])
    for j, k in enumerate(keep):
        assert frames[off[j]:off[j + 1]].cpu().numpy().tobytes() == full[k], ("thinned", k)
    for k in (0, len(videos) - 1):
        assert resize_frames([videos[k]])[0].cpu().numpy().tobytes() == full[k], ("alone", k)


def test_repeat_filled_output_and_graph_replay():
    from ops.optical_flow import ResizePlan
    rng = np.random.default_rng(2)
    shapes = [(3, 240, 320), (2, 360, 640), (4, 100, 77), (1, 1, 1), (2, 720, 1280)]
    first = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    other = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    want = R.resize_videos(first, 340, 256).tobytes()
    want_other = R.resize_videos(other, 340, 256).tobytes()
    plan = ResizePlan(shapes, device=DEV)
    assert list(plan.offsets) == [0, 3, 5, 9, 10, 12]
    xs = [_cuda(a) for a in first]
    assert plan.run(xs).cpu().numpy().tobytes() == want
    assert plan.run(xs).cpu().numpy().tobytes() == want
    plan.frames.fill_(0xFF)
    assert plan.run().cpu().numpy().tobytes() == want
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(xs)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = plan.run(xs)
    for x, o in zip(xs, other):
        x.copy_(_cuda(o))
    plan.frames.fill_(0xFF)
    g.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == want_other
    for x, a in zip(xs, first):
        x.copy_(_cuda(a))
    g.replay()
    torch.cuda.synchronize()
    assert out.cpu().numpy().tobytes() == want


def _scene(n, h, w, seed):
    """n frames of a smooth texture drifting about a pixel per frame, uint8 [n, h, w, 3]"""
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    ph = np.random.default_rng(seed).uniform(0, 6.3, 6)
    fr = []
    for k in range(n):
        xs, ys = x * 340.0 / w - 1.1 * k, y * 256.0 / h + 0.7 * k
        v = [128 + 60 * np.sin(xs * 0.07 + ph[c]) * np.cos(ys * 0.05 + ph[c + 3]) + 40 * np.sin((xs + ys) * 0.02 + c) for c in range(3)]
        fr.append(np.clip(np.rint(np.stack(v, -1)), 0, 255))
    return np.stack(fr).astype(np.uint8)


def test_extraction_end_to_end(tmp_path):
    """decoded frames of three source sizes -> one resize_frames -> one tvl1_flow -> flow_planes equals each video resized
    and solved alone; write_frame_jpegs of the resized frames writes the bytes Pillow writes for cv2's resized frames"""
    from PIL import Image
    from ops.optical_flow import resize_frames, tvl1_flow, flow_planes, pair_offsets, write_frame_jpegs
    videos = [_scene(3, 240, 320, 0), _scene(2, 360, 640, 1), _scene(3, 100, 77, 2)]
    frames, off = resize_frames([_cuda(v) for v in videos])
    planes = flow_planes(tvl1_flow(frames, off)).cpu().numpy()
    pairs = pair_offsets(off)
    for k, v in enumerate(videos):
        alone, _ = resize_frames([_cuda(v)])
        assert alone.cpu().numpy().tobytes() == frames[off[k]:off[k + 1]].cpu().numpy().tobytes(), k
        assert flow_planes(tvl1_flow(alone)).cpu().numpy().tobytes() == planes[2 * pairs[k]:2 * pairs[k + 1]].tobytes(), k
    cv2 = _cv2()
    ref = [np.stack([cv2.resize(f, (340, 256), interpolation=cv2.INTER_LINEAR) for f in v]) if cv2 is not None else R.resize(v, 340, 256)
           for v in videos]
    dirs = [str(tmp_path / ("v%d" % k)) for k in range(len(videos))]
    paths = write_frame_jpegs(frames, dirs, offsets=off)
    assert len(paths) == int(off[-1])
    i = 0
    for k, r in enumerate(ref):
        for f in r:
            b = io.BytesIO()
            Image.fromarray(f).save(b, format="JPEG", quality=95)
            assert open(paths[i], "rb").read() == b.getvalue(), paths[i]
            i += 1
