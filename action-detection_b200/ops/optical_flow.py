"""TV-L1 optical flow on the GPU: the Flow stream's x / y planes from RGB frames, many frame pairs per call (csrc/optical_flow.cu).

The reference README ("Extract Frames and Optical Flow Images") makes these planes with DenseFlow, which runs OpenCV's CUDA
OpticalFlowDual_TVL1 on one frame pair at a time and writes flow_{x,y}_%05d.jpg.  Here the same solver, with the rules
oracle/tvl1_oracle.py writes down, runs on all pairs of many videos in one call:

    frames = decode_jpeg(byte_groups, mode='RGB')               # uint8 [n, H, W, 3] per video, one size for all
    flow = tvl1_flow(torch.cat(frames), offsets)                # fp32 [P, 2, H, W], pair k of a video = (frame k, frame k + 1)

Videos of different sizes are first brought to one size as DenseFlow's extract_gpu --new_width 340 --new_height 256 does
(cv::resize, INTER_LINEAR; bitwise cv2.resize, csrc/frame_resize.cu):

    frames, offsets = resize_frames(decoded_videos)             # uint8 [sum n, 256, 340, 3], offsets [V + 1]
    flow = tvl1_flow(frames, offsets)
    planes = flow_planes(flow)                                  # uint8 [2P, H, W, 1]: x, y, x, y, ... as JpegBytesLoader keeps them
    x = model.frame_transforms().oversample(planes[2 * k:2 * k + 2 * model.new_length])   # a Flow tick, as from decoded JPEGs
    write_flow_jpegs(planes, video_dirs, offsets=offsets)      # or the files SSNDataSet reads, encoded on the GPU
    write_frame_jpegs(torch.cat(frames), video_dirs, offsets=offsets)   # and the RGB side, img_{:05d}.jpg

or, without the files, the pixels the data sets would read back from them (the JPEG round trip, computed on the GPU):

    x = model.frame_transforms().oversample(flow_images(planes)[2 * k:2 * k + 2 * model.new_length])
    rgb = frame_images(torch.cat(frames))                       # what decode_jpeg returns for img_{:05d}.jpg

No CPU path: the frames must be CUDA tensors.  Parity with a built DenseFlow or OpenCV CUDA is not checked by this project.
"""
import ctypes as C
import os

import numpy as np
import torch

from ssn_b200._lib import lib, check, TVL1Params, ResizeVideo

DEFAULTS = dict(tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300, scale_step=0.8, gamma=0.0,
                fixed_iterations=False)


def tvl1_params(**params):
    """-> TVL1Params with OpenCV's defaults; 'lambda' may be given as lambda_ or as **{'lambda': ...}"""
    if "lambda" in params:
        params["lambda_"] = params.pop("lambda")
    unknown = set(params) - set(DEFAULTS)
    if unknown:
        raise TypeError("unknown TV-L1 parameter(s): %s" % sorted(unknown))
    q = dict(DEFAULTS, **params)
    return TVL1Params(float(q["tau"]), float(q["lambda_"]), float(q["theta"]), float(q["epsilon"]), float(q["scale_step"]),
                      float(q["gamma"]), int(q["nscales"]), int(q["warps"]), int(q["iterations"]), int(bool(q["fixed_iterations"])))


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def pair_offsets(offsets):
    """frame offsets [V + 1] -> pair offsets [V + 1]: video v's pairs are rows pairs[v] .. pairs[v + 1] - 1 of the flow"""
    off = np.asarray(offsets, np.int64)
    return off - np.arange(len(off), dtype=np.int64)


class TVL1Plan:
    """One call's shapes, parameters and workspace, so the solver can be run again (or captured in a CUDA graph) on new frames
    of the same layout: plan.run(frames) writes plan.flow and plan.iterations."""

    def __init__(self, offsets, height, width, device, **params):
        self.prm = tvl1_params(**params)
        self.offsets = np.ascontiguousarray(np.asarray(offsets, np.int64))
        self.V, self.H, self.W = len(self.offsets) - 1, int(height), int(width)
        self._off = self.offsets.ctypes.data_as(C.POINTER(C.c_int64))
        ws = lib.ssnb_tvl1_workspace_bytes(self.prm, self._off, self.V, self.H, self.W)
        if ws == 0:
            check(lib.ssnb_tvl1_flow(self.prm, None, self._off, None, self.V, self.H, self.W, None, None, None, 0, None), None, "tvl1_flow")
        self.levels = lib.ssnb_tvl1_levels(self.prm, self.H, self.W)
        self.P = int(self.offsets[-1]) - self.V
        dev = torch.device(device)
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=dev)
        self.offsets_dev = torch.from_numpy(self.offsets).to(dev)
        self.flow = torch.empty(self.P, 2, self.H, self.W, dtype=torch.float32, device=dev)
        self.iterations = torch.empty(self.P, self.levels, self.prm.warps, dtype=torch.int32, device=dev)

    def run(self, frames):
        if not (torch.is_tensor(frames) and frames.is_cuda and frames.dtype == torch.uint8):
            raise RuntimeError("tvl1_flow needs CUDA uint8 RGB frames [n, H, W, 3] (no CPU path)")
        if tuple(frames.shape) != (int(self.offsets[-1]), self.H, self.W, 3):
            raise ValueError("frames must be [%d, %d, %d, 3], got %s" % (int(self.offsets[-1]), self.H, self.W, tuple(frames.shape)))
        frames = frames.contiguous()
        with torch.cuda.device(self.flow.device):
            check(lib.ssnb_tvl1_flow(self.prm, frames.data_ptr(), self._off, self.offsets_dev.data_ptr(), self.V, self.H, self.W,
                                     self.flow.data_ptr(), self.iterations.data_ptr(), self.workspace.data_ptr(), self.workspace.numel(),
                                     _stream()), None, "tvl1_flow")
        return self.flow


def tvl1_flow(frames, offsets=None, return_iterations=False, **params):
    """uint8 RGB frames [sum N, H, W, 3] on the GPU (decode_jpeg's output, concatenated), frame offsets [V + 1] (default: one
    video) -> fp32 flow [sum (N - 1), 2, H, W] on the device: pair k of video v is (frame k, frame k + 1), u then v in pixels.
    params: tau, lambda (or lambda_), theta, nscales, warps, epsilon, iterations, scale_step, gamma, fixed_iterations, OpenCV's
    defaults.  return_iterations: also the int32 [P, levels, warps] iterations each warp ran (level 0 the finest)."""
    if not (torch.is_tensor(frames) and frames.is_cuda):
        raise RuntimeError("tvl1_flow needs CUDA uint8 RGB frames [n, H, W, 3] (no CPU path)")
    if frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError("frames must be uint8 [n, H, W, 3]")
    if offsets is None:
        offsets = [0, frames.shape[0]]
    plan = TVL1Plan(offsets, frames.shape[1], frames.shape[2], frames.device, **params)
    flow = plan.run(frames)
    return (flow, plan.iterations) if return_iterations else flow


def flow_planes(flow, bound=20.0):
    """fp32 flow [P, 2, H, W] on the GPU -> uint8 planes [2P, H, W, 1] (x, y, x, y, ...), DenseFlow's convertFlowToImage with
    this bound: what decode_jpeg(..., mode='L') returns for its flow_x / flow_y files, before the JPEG round trip."""
    if not (torch.is_tensor(flow) and flow.is_cuda and flow.dtype == torch.float32):
        raise RuntimeError("flow_planes needs a CUDA fp32 flow [P, 2, H, W]")
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise ValueError("flow must be [P, 2, H, W]")
    flow = flow.contiguous()
    P, _, H, W = flow.shape
    out = torch.empty(2 * P, H, W, 1, dtype=torch.uint8, device=flow.device)
    with torch.cuda.device(flow.device):
        check(lib.ssnb_flow_planes(flow.data_ptr(), P, H, W, float(bound), out.data_ptr(), _stream()), None, "flow_planes")
    return out


def _video_dirs(dirs, counts, what):
    """one directory, or one per video whose item counts the offsets give -> a directory per video"""
    if isinstance(dirs, (str, os.PathLike)):
        dirs = [dirs]
    dirs = list(dirs)
    if len(dirs) != len(counts):
        raise ValueError("one directory per video, and offsets that match the %s" % what)
    return dirs


def _encoded(images, mode, quality, restart):
    """CUDA uint8 [N, H, W, C] -> the files' bytes from the GPU encoder; anything else -> None (the Pillow path).  restart:
    the restart keywords, as encode_jpeg and Image.save take them (checked here for both paths)."""
    from ops.jpeg import encode_jpeg, _enc_restart
    _enc_restart(restart["restart_marker_blocks"], restart["restart_marker_rows"])
    if torch.is_tensor(images) and images.is_cuda:
        return encode_jpeg(images, mode=mode, quality=quality, **restart)
    return None


def write_flow_jpegs(planes, dirs, prefix="flow_", quality=95, offsets=None, restart_marker_blocks=0, restart_marker_rows=0):
    """Write flow_planes' output as DenseFlow does, one directory per video: {prefix}x_{:05d}.jpg and {prefix}y_{:05d}.jpg
    numbered from 1 like img_{:05d}.jpg.  CUDA planes are encoded on the GPU (ops.jpeg.encode_jpeg, one call for all planes),
    host planes through Pillow; the files are the same bytes either way.  dirs: one directory, or one per video with the
    frame offsets the flow was computed with.  restart_marker_blocks / restart_marker_rows: Pillow's restart intervals
    (encode_jpeg), which let decode_jpeg split each file; the decoded planes do not change.  -> the paths written, x then y
    per pair."""
    from PIL import Image
    if torch.is_tensor(planes) and planes.is_cuda:
        if planes.dtype != torch.uint8 or planes.dim() != 4 or planes.shape[3] != 1 or planes.shape[0] % 2:
            raise ValueError("planes must be uint8 [2P, H, W, 1]")
        n = planes.shape[0]
    else:
        arr = planes.cpu().numpy() if torch.is_tensor(planes) else np.asarray(planes)
        if arr.dtype != np.uint8 or arr.ndim != 4 or arr.shape[3] != 1 or arr.shape[0] % 2:
            raise ValueError("planes must be uint8 [2P, H, W, 1]")
        n = arr.shape[0]
    pairs = pair_offsets(offsets if offsets is not None else [0, n // 2 + 1])
    if pairs[-1] != n // 2:
        raise ValueError("one directory per video, and offsets that match the planes' %d pairs" % (n // 2))
    dirs = _video_dirs(dirs, np.diff(pairs), "planes' %d pairs" % (n // 2))
    restart = dict(restart_marker_blocks=int(restart_marker_blocks), restart_marker_rows=int(restart_marker_rows))
    files = _encoded(planes, "L", quality, restart)
    paths = []
    for v, d in enumerate(dirs):
        os.makedirs(d, exist_ok=True)
        for k in range(int(pairs[v + 1] - pairs[v])):
            for c, axis in enumerate("xy"):
                path = os.path.join(d, "%s%s_%05d.jpg" % (prefix, axis, k + 1))
                i = 2 * (pairs[v] + k) + c
                if files is not None:
                    with open(path, "wb") as f:
                        f.write(files[i])
                else:
                    Image.fromarray(arr[i, :, :, 0]).save(path, quality=quality, **restart)
                paths.append(path)
    return paths


def write_frame_jpegs(frames, dirs, prefix="img_", quality=95, offsets=None, restart_marker_blocks=0, restart_marker_rows=0):
    """Write RGB frames as DenseFlow does, one directory per video: {prefix}{:05d}.jpg numbered from 1, the files SSNDataSet
    reads for RGB.  frames uint8 [N, H, W, 3]: CUDA frames are encoded on the GPU in one call, host frames through Pillow,
    the same bytes either way.  dirs: one directory, or one per video with the frame offsets [V + 1] (as tvl1_flow takes
    them).  restart_marker_blocks / restart_marker_rows: Pillow's restart intervals (encode_jpeg), which let decode_jpeg
    split each file; the decoded frames do not change.  -> the paths written, in frame order."""
    from PIL import Image
    if torch.is_tensor(frames) and frames.is_cuda:
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
            raise ValueError("frames must be uint8 [N, H, W, 3]")
        n = frames.shape[0]
    else:
        arr = frames.cpu().numpy() if torch.is_tensor(frames) else np.asarray(frames)
        if arr.dtype != np.uint8 or arr.ndim != 4 or arr.shape[3] != 3:
            raise ValueError("frames must be uint8 [N, H, W, 3]")
        n = arr.shape[0]
    off = np.asarray(offsets if offsets is not None else [0, n], np.int64)
    if off.ndim != 1 or len(off) < 2 or off[0] != 0 or off[-1] != n or (np.diff(off) < 0).any():
        raise ValueError("one directory per video, and offsets that match the %d frames" % n)
    dirs = _video_dirs(dirs, np.diff(off), "%d frames" % n)
    restart = dict(restart_marker_blocks=int(restart_marker_blocks), restart_marker_rows=int(restart_marker_rows))
    files = _encoded(frames, "RGB", quality, restart)
    paths = []
    for v, d in enumerate(dirs):
        os.makedirs(d, exist_ok=True)
        for k in range(int(off[v + 1] - off[v])):
            path = os.path.join(d, "%s%05d.jpg" % (prefix, k + 1))
            i = int(off[v]) + k
            if files is not None:
                with open(path, "wb") as f:
                    f.write(files[i])
            else:
                Image.fromarray(arr[i]).save(path, quality=quality, **restart)
            paths.append(path)
    return paths


def flow_images(planes, quality=95):
    """The in-memory counterpart of write_flow_jpegs: CUDA uint8 planes [2P, H, W, 1] (flow_planes' output, x then y per pair,
    the order JpegBytesLoader keeps) -> uint8 [2P, H, W, 1] on the device, bitwise what decode_jpeg(..., mode='L') returns for
    the flow_x / flow_y files write_flow_jpegs writes at this quality (ops.jpeg.jpeg_roundtrip; no file is written)."""
    from ops.jpeg import jpeg_roundtrip
    if not (torch.is_tensor(planes) and planes.is_cuda):
        raise RuntimeError("flow_images needs CUDA uint8 planes [2P, H, W, 1] (no CPU path)")
    if planes.dtype != torch.uint8 or planes.dim() != 4 or planes.shape[3] != 1 or planes.shape[0] % 2:
        raise ValueError("planes must be uint8 [2P, H, W, 1]")
    return jpeg_roundtrip(planes, mode="L", quality=quality)


def frame_images(frames, quality=95):
    """The in-memory counterpart of write_frame_jpegs: CUDA uint8 RGB frames [N, H, W, 3] -> uint8 [N, H, W, 3] on the device,
    bitwise what decode_jpeg(..., mode='RGB') returns for the img_{:05d}.jpg files write_frame_jpegs writes at this quality
    (ops.jpeg.jpeg_roundtrip; no file is written)."""
    from ops.jpeg import jpeg_roundtrip
    if not (torch.is_tensor(frames) and frames.is_cuda):
        raise RuntimeError("frame_images needs CUDA uint8 frames [N, H, W, 3] (no CPU path)")
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError("frames must be uint8 [N, H, W, 3]")
    return jpeg_roundtrip(frames, mode="RGB", quality=quality)


MAX_SIDE = 65500


class ResizePlan:
    """One resize call's table and buffers, so it can be run again (or captured in a CUDA graph) on new frames of the same
    videos' sizes.  shapes: (frames, height, width) per video.  plan.inputs[v] is video v's uint8 [n_v, H_v, W_v, 3] view of
    the packed source plan.src; plan.run(videos) copies the videos there first, plan.run() resizes what plan.src holds into
    plan.frames, uint8 [sum n_v, height, width, 3].  plan.offsets are the frame offsets [V + 1] of tvl1_flow and write_*_jpegs."""

    def __init__(self, shapes, width=340, height=256, device="cuda"):
        shapes = [tuple(int(x) for x in s) for s in shapes]
        if not shapes:
            raise ValueError("resize_frames needs at least one video")
        self.width, self.height = int(width), int(height)
        if not (1 <= self.width <= MAX_SIDE and 1 <= self.height <= MAX_SIDE):
            raise ValueError("destination height and width must be 1 .. %d" % MAX_SIDE)
        self.table = (ResizeVideo * len(shapes))()
        src_bytes, frames = 0, 0
        for e, (n, h, w) in zip(self.table, shapes):
            if n < 1:
                raise ValueError("each video needs at least one frame")
            if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
                raise ValueError("frame height and width must be 1 .. %d" % MAX_SIDE)
            e.src_offset, e.first_frame, e.height, e.width, e.frames = src_bytes, frames, h, w, n
            src_bytes += n * h * w * 3
            frames += n
        self.shapes = shapes
        self.offsets = np.cumsum([0] + [n for n, _, _ in shapes]).astype(np.int64)
        dev = torch.device(device)
        self.src = torch.empty(src_bytes, dtype=torch.uint8, device=dev)
        self.inputs = [self.src[e.src_offset:e.src_offset + n * h * w * 3].view(n, h, w, 3) for e, (n, h, w) in zip(self.table, shapes)]
        self.table_dev = torch.frombuffer(bytearray(bytes(self.table)), dtype=torch.uint8).to(dev)
        self.frames = torch.empty(frames, self.height, self.width, 3, dtype=torch.uint8, device=dev)

    def run(self, videos=None):
        if videos is not None:
            videos = list(videos)
            if len(videos) != len(self.inputs):
                raise ValueError("the plan has %d videos, got %d" % (len(self.inputs), len(videos)))
            for v, (x, dst) in enumerate(zip(videos, self.inputs)):
                if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.uint8):
                    raise RuntimeError("resize_frames needs CUDA uint8 RGB frames [n, H, W, 3] (no CPU path)")
                if tuple(x.shape) != tuple(dst.shape):
                    raise ValueError("video %d must be %s, got %s" % (v, tuple(dst.shape), tuple(x.shape)))
                dst.copy_(x)
        with torch.cuda.device(self.frames.device):
            check(lib.ssnb_frame_resize(self.src.data_ptr(), self.src.numel(), self.table, self.table_dev.data_ptr(), len(self.table),
                                        self.height, self.width, self.frames.data_ptr(), self.frames.numel(), _stream()),
                  None, "frame_resize")
        return self.frames


def resize_frames(videos, width=340, height=256):
    """DenseFlow's per-frame cv::resize(frame, image, Size(width, height)) (extract_gpu --new_width / --new_height), bitwise
    cv2.resize(frame, (width, height), interpolation=cv2.INTER_LINEAR), for many videos of any sizes in one call.
    videos: a list of CUDA uint8 [n_v, H_v, W_v, 3] (RGB or BGR alike; decode_jpeg's output) -> (frames uint8
    [sum n_v, height, width, 3] on the device, frame offsets int64 [V + 1]), the frames and offsets tvl1_flow,
    write_frame_jpegs and frame_images take."""
    if torch.is_tensor(videos):
        videos = [videos]
    videos = list(videos)
    for x in videos:
        if not (torch.is_tensor(x) and x.is_cuda):
            raise RuntimeError("resize_frames needs CUDA uint8 RGB frames [n, H, W, 3] (no CPU path)")
        if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
            raise ValueError("each video must be uint8 [n, H, W, 3]")
    if not videos:
        raise ValueError("resize_frames needs at least one video")
    plan = ResizePlan([x.shape[:3] for x in videos], width, height, videos[0].device)
    return plan.run(videos), plan.offsets
