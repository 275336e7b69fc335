"""The JPEG round trip on the H100 (csrc/jpeg_roundtrip.cu) bitwise against decode_jpeg(encode_jpeg(...)) and against Pillow's
save -> open -> convert: the host test's grid of sizes, contents and qualities in ragged calls; each image's result against
the same call permuted and thinned; CUDA-graph replay; refusals that launch nothing; and both streams end to end, TV-L1 flow
planes and RGB frames through flow_images / frame_images against the same data through files, JpegBytesLoader and
decode_jpeg, into the frame transforms."""
import io
import os
import random

import numpy as np
import pytest
import torch

from oracle import jpeg_encode_oracle as E

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SIZES = [(1, 1), (9, 7), (8, 8), (17, 15), (16, 16), (15, 17), (256, 340), (256, 341), (360, 480)]
KINDS = ["ramp", "noise", "const128", "checker"]
QUALITIES = [1, 50, 75, 95, 100]
RGB_MEAN, FLOW_MEAN = [104, 117, 128], [128]


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _pillow(img, mode, quality):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(img[..., 0] if mode == "L" else img, mode).save(f, format="JPEG", quality=quality)
    f.seek(0)
    return np.asarray(Image.open(f).convert(mode)).reshape(img.shape)


def _grid(mode):
    C = E.MODES[mode]
    return [E.fixture(kind, h, w, C, seed=h * 131 + w + k) for h, w in SIZES for k, kind in enumerate(KINDS)]


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("quality", QUALITIES)
def test_grid_equals_decode_of_encode_and_pillow(mode, quality):
    from ops.jpeg import decode_jpeg, encode_jpeg, jpeg_roundtrip
    imgs = _grid(mode)
    xs = [_cuda(a) for a in imgs]
    got = [g.cpu().numpy() for g in jpeg_roundtrip(xs, mode=mode, quality=quality)]
    files = encode_jpeg(xs, mode=mode, quality=quality)
    dec = decode_jpeg([[f] for f in files], mode=mode)
    for i, (a, g, d) in enumerate(zip(imgs, got, dec)):
        assert g.shape == a.shape and g.dtype == np.uint8
        assert g.tobytes() == d[0].cpu().numpy().tobytes(), (i, a.shape, "decode_jpeg(encode_jpeg)")
        assert g.tobytes() == _pillow(a, mode, quality).tobytes(), (i, a.shape, "Pillow")


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_batched_tensor_and_random_ragged_sizes(mode):
    from ops.jpeg import jpeg_roundtrip
    C = E.MODES[mode]
    batch = np.stack([E.fixture(k, 256, 340, C, seed=s) for s, k in enumerate(["noise", "ramp", "flow", "checker", "noise"])])
    out = jpeg_roundtrip(_cuda(batch), mode=mode, quality=90)
    assert tuple(out.shape) == batch.shape and out.dtype == torch.uint8 and out.is_cuda
    assert out.cpu().numpy().tobytes() == np.stack([_pillow(a, mode, 90) for a in batch]).tobytes()
    rng = np.random.default_rng(5)
    imgs = [E.fixture(["noise", "flow", "ramp"][i % 3], int(rng.integers(1, 300)), int(rng.integers(1, 400)), C, seed=i)
            for i in range(60)] + [E.fixture("noise", 1, 2000, C, 1), E.fixture("noise", 2000, 1, C, 2)]
    got = jpeg_roundtrip([_cuda(a) for a in imgs], mode=mode, quality=85)
    for i, (a, g) in enumerate(zip(imgs, got)):
        assert g.cpu().numpy().tobytes() == _pillow(a, mode, 85).tobytes(), (i, a.shape)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_an_image_does_not_depend_on_the_rest_of_the_call(mode):
    from ops.jpeg import jpeg_roundtrip
    imgs = _grid(mode)
    whole = [g.cpu().numpy().tobytes() for g in jpeg_roundtrip([_cuda(a) for a in imgs], mode=mode, quality=75)]
    rng = random.Random(1)
    for _ in range(3):
        idx = rng.sample(range(len(imgs)), rng.randint(1, len(imgs)))       # permuted, some dropped
        part = jpeg_roundtrip([_cuda(imgs[i]) for i in idx], mode=mode, quality=75)
        for i, g in zip(idx, part):
            assert g.cpu().numpy().tobytes() == whole[i], i
    for i in (0, len(imgs) - 1):
        assert jpeg_roundtrip([_cuda(imgs[i])], mode=mode, quality=75)[0].cpu().numpy().tobytes() == whole[i]


def test_graph_capture_and_replay():
    from ops.jpeg import JpegRoundtripPlan
    imgs = [E.fixture("ramp", h, w, 3, seed=i) for i, (h, w) in enumerate(SIZES)]
    other = [E.fixture("noise", h, w, 3, seed=50 + i) for i, (h, w) in enumerate(SIZES)]
    plan = JpegRoundtripPlan([a.shape[:2] for a in imgs], "RGB", 95, DEV)
    xs = [_cuda(a) for a in imgs]
    eager = [g.cpu().numpy().tobytes() for g in plan.run(xs)]
    assert eager == [_pillow(a, "RGB", 95).tobytes() for a in imgs]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(xs)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        views = plan.run(xs)
    for x, o in zip(xs, other):
        x.copy_(_cuda(o))
    plan.out.fill_(0xFF)
    g.replay()
    torch.cuda.synchronize()
    assert [v.cpu().numpy().tobytes() for v in views] == [_pillow(o, "RGB", 95).tobytes() for o in other]
    for x, a in zip(xs, imgs):
        x.copy_(_cuda(a))
    g.replay()
    torch.cuda.synchronize()
    assert [v.cpu().numpy().tobytes() for v in views] == eager


def test_refusals_launch_nothing():
    import ctypes as C
    from ssn_b200._lib import lib, JpegEncodeImage
    from ops.jpeg import jpeg_roundtrip
    buf = torch.zeros(2 * 16 * 24 * 3, dtype=torch.uint8, device=DEV)
    imgs = (JpegEncodeImage * 1)()
    imgs[0].src_offset, imgs[0].height, imgs[0].width = 0, 16, 24
    dev = torch.frombuffer(bytearray(bytes(imgs)), dtype=torch.uint8).to(DEV)
    torch.cuda.synchronize()
    n0 = lib.ssnb_global_launch_count()
    half = 16 * 24 * 3
    for args in ((3, 95, buf.data_ptr(), half, imgs, dev.data_ptr(), 1, buf.data_ptr() + half // 2, half),     # out overlaps src
                 (3, 0, buf.data_ptr(), half, imgs, dev.data_ptr(), 1, buf.data_ptr() + half, half),          # quality 0
                 (2, 95, buf.data_ptr(), half, imgs, dev.data_ptr(), 1, buf.data_ptr() + half, half),         # mode 2
                 (3, 95, buf.data_ptr(), half - 1, imgs, dev.data_ptr(), 1, buf.data_ptr() + half, half),     # src too small
                 (3, 95, buf.data_ptr(), half, imgs, None, 1, buf.data_ptr() + half, half)):                  # NULL images_dev
        assert lib.ssnb_jpeg_roundtrip(*args, C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 1
    with pytest.raises(ValueError):
        jpeg_roundtrip([buf[:half].view(16, 24, 3)], mode="L")
    with pytest.raises(ValueError):
        jpeg_roundtrip([buf[:half].view(16, 24, 3)], quality=101)
    with pytest.raises(ValueError):
        jpeg_roundtrip([buf[:half].view(16, 24, 3).float()])
    assert lib.ssnb_global_launch_count() == n0
    # the accepted call launches one kernel
    out = jpeg_roundtrip([buf[:half].view(16, 24, 3)])
    assert lib.ssnb_global_launch_count() == n0 + 1 and out[0].shape == (16, 24, 3)


def _video(n, h, w, seed):
    """n frames of a smooth seeded texture drifting by about a pixel per frame"""
    from oracle import tvl1_oracle as T
    ys, xs = np.meshgrid(np.arange(float(h)), np.arange(float(w)), indexing="ij")
    return np.stack([np.stack([np.rint(T.texture(xs - 0.9 * k + 3 * c, ys + 0.5 * k, seed + c)) for c in range(3)], -1)
                     for k in range(n)]).clip(0, 255).astype(np.uint8)


def _read_back(d, modality, tmpl, count):
    from ops.jpeg import JpegBytesLoader, decode_jpeg

    class Loader(JpegBytesLoader):
        pass

    ld = Loader()
    ld.modality, ld.image_tmpl = modality, tmpl
    blobs = [b for idx in range(1, count + 1) for b in ld._load_image(d, idx)]
    return decode_jpeg([blobs], mode="L" if modality == "Flow" else "RGB")[0]


def test_flow_stream_end_to_end_equals_the_files(tmp_path):
    from ops.frame_transforms import oversample_frames
    from ops.optical_flow import flow_images, flow_planes, tvl1_flow, write_flow_jpegs
    frames = _cuda(_video(6, 96, 128, 3))
    planes = flow_planes(tvl1_flow(frames, iterations=30))
    mem = flow_images(planes)
    assert tuple(mem.shape) == tuple(planes.shape) and not torch.equal(mem, planes)      # the JPEG loss is there
    write_flow_jpegs(planes, str(tmp_path / "v"))
    files = _read_back(str(tmp_path / "v"), "Flow", "flow_{}_{:05d}.jpg", 5)
    assert mem.cpu().numpy().tobytes() == files.cpu().numpy().tobytes()
    a = oversample_frames([mem[2 * k:2 * k + 4] for k in range(3)], FLOW_MEAN, [1], 2)
    b = oversample_frames([files[2 * k:2 * k + 4] for k in range(3)], FLOW_MEAN, [1], 2)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_rgb_stream_end_to_end_equals_the_files(tmp_path):
    from ops.frame_transforms import oversample_frames, sample_train_params, train_frames
    from ops.optical_flow import frame_images, write_frame_jpegs
    video = np.concatenate([_video(5, 256, 340, 7), E.fixture("noise", 256, 340, 3, 9)[None]])
    frames = _cuda(video)
    mem = frame_images(frames, quality=95)
    write_frame_jpegs(frames, str(tmp_path / "v"), quality=95)
    files = _read_back(str(tmp_path / "v"), "RGB", "img_{:05d}.jpg", len(video))
    assert mem.cpu().numpy().tobytes() == files.cpu().numpy().tobytes()
    groups_m, groups_f = [mem[k:k + 1] for k in range(len(video))], [files[k:k + 1] for k in range(len(video))]
    params = sample_train_params([(256, 340)] * len(video), [1, .875, .75, .66], rng=random.Random(2))
    a = train_frames(groups_m, params, RGB_MEAN, [1], 3)
    b = train_frames(groups_f, params, RGB_MEAN, [1], 3)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    a = oversample_frames(groups_m[:2], RGB_MEAN, [1], 3)
    b = oversample_frames(groups_f[:2], RGB_MEAN, [1], 3)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
