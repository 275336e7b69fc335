"""Frame transforms on the GPU: the reference's PIL group transforms (transforms.py) followed by Stack(roll=True),
ToTorchFormatTensor(div=False) and GroupNormalize, computed by libssn_b200.so (csrc/frames.cu) and bitwise equal to them.

The DataLoader carries uint8 frames (GroupToUint8 as the dataset's transform); the training loop draws the crop parameters
with sample_train_params, which consumes Python's `random` exactly as GroupMultiScaleCrop + GroupRandomHorizontalFlip do, and
one call per batch turns every group into the fp32 frames `model(...)` takes:

    params = sample_train_params([f.shape[1:3] for f in groups], scales)
    x = train_frames(groups, params, mean, std, frame_channels)      # [frames, C, 224, 224] on the GPU

Frames are uint8 [n, H, W, C] (C = 3 RGB, 1 for the L images of Flow), a [G, n, H, W, C] batch of equal groups, or a list of
[n, H, W, C] groups of different sizes.  CPU frames are copied in (pinned); CUDA frames are used where they are.  Only the
div=False normalisation of BNInception is supported.
"""
import ctypes as C
import random

import numpy as np
import torch

from ssn_b200._lib import lib, check, FrameCfg, FrameGroup, FRAMES_TRAIN, FRAMES_OVERSAMPLE, FRAMES_CENTER


def fill_fix_offset(more_fix_crop, image_w, image_h, crop_w, crop_h):
    """GroupMultiScaleCrop.fill_fix_offset (transforms.py:183-206)"""
    w_step = (image_w - crop_w) // 4
    h_step = (image_h - crop_h) // 4
    ret = [(0, 0), (4 * w_step, 0), (0, 4 * h_step), (4 * w_step, 4 * h_step), (2 * w_step, 2 * h_step)]
    if more_fix_crop:
        ret += [(0, 2 * h_step), (4 * w_step, 2 * h_step), (2 * w_step, 4 * h_step), (2 * w_step, 0 * h_step),
                (1 * w_step, 1 * h_step), (3 * w_step, 1 * h_step), (1 * w_step, 3 * h_step), (3 * w_step, 3 * h_step)]
    return ret


def crop_pairs(image_w, image_h, input_size, scales, max_distort=1):
    """the (crop_w, crop_h) candidates of GroupMultiScaleCrop._sample_crop_size (transforms.py:155-168)"""
    base_size = min(image_w, image_h)
    crop_sizes = [int(base_size * x) for x in scales]
    crop_h = [input_size if abs(x - input_size) < 3 else x for x in crop_sizes]
    crop_w = [input_size if abs(x - input_size) < 3 else x for x in crop_sizes]
    return [(w, h) for i, h in enumerate(crop_h) for j, w in enumerate(crop_w) if abs(i - j) <= max_distort]


def sample_train_params(sizes, scales, input_size=224, max_distort=1, fix_crop=True, more_fix_crop=True, rng=random):
    """One (crop_w, crop_h, offset_w, offset_h, flip) per group of the given (H, W) sizes, drawing from `rng` (the random
    module by default) in the reference's order: random.choice(pairs), random.choice(offsets) or randint(w), randint(h), then
    random.random() < 0.5 for the flip (transforms.py:56,170-181)."""
    out = []
    for h, w in sizes:
        cw, ch = rng.choice(crop_pairs(w, h, input_size, scales, max_distort))
        if fix_crop:
            ow, oh = rng.choice(fill_fix_offset(more_fix_crop, w, h, cw, ch))
        else:
            ow = rng.randint(0, w - cw)
            oh = rng.randint(0, h - ch)
        out.append((cw, ch, ow, oh, rng.random() < 0.5))
    return out


def _groups(frames):
    if isinstance(frames, (list, tuple)):
        groups = list(frames)
    elif frames.dim() == 5:
        groups = list(frames.unbind(0))
    else:
        groups = [frames]
    for g in groups:
        if g.dim() != 4 or g.dtype != torch.uint8 or g.shape[3] not in (1, 3):
            raise ValueError("frames must be uint8 [n, H, W, C] with C = 3 (RGB) or 1 (L)")
        if g.shape[3] != groups[0].shape[3]:
            raise ValueError("every group must have the same channel count")
    return groups


class FramePlan:
    """A validated call: the host group table, its device copy and the output / workspace sizes.  run() enqueues the library
    call only, so it can be captured in a CUDA graph; copy new frames into `src` and new parameters into `groups_dev`
    (set_train_params) before a replay."""

    def __init__(self, mode, shapes, channels, out_size, scale_size, mean, std, invert_even, device, params=None):
        if len(mean) > 8 or len(std) != len(mean) and len(std) != 1:
            raise ValueError("1..8 mean values and as many std values, or one")
        std = list(std) * len(mean) if len(std) == 1 else list(std)
        self.cfg = FrameCfg(mode, channels, out_size, scale_size, int(bool(invert_even)), len(mean), (C.c_float * 8)(*mean),
                            (C.c_float * 8)(*std))
        self.groups = (FrameGroup * len(shapes))()
        off = 0
        for g, (n, h, w) in zip(self.groups, shapes):
            g.src_offset, g.height, g.width, g.images = off, h, w, n
            off += n * h * w * channels
        self.src_bytes = off
        if params is not None:
            self._set_params(params)
        ws, nd = C.c_size_t(0), C.c_int64(0)
        check(lib.ssnb_frame_transform_workspace_bytes(C.byref(self.cfg), self.groups, len(shapes), C.byref(ws), C.byref(nd)), None,
              "frame_transform_workspace_bytes")
        self.device = device
        self.dst_floats = nd.value
        self.workspace = torch.empty(max(ws.value, 1), dtype=torch.uint8, device=device)
        self.groups_dev = torch.empty(C.sizeof(self.groups), dtype=torch.uint8, device=device)
        self._upload()

    def _set_params(self, params):
        if len(params) != len(self.groups):
            raise ValueError("one (crop_w, crop_h, offset_w, offset_h, flip) per group")
        for g, (cw, ch, ox, oy, fl) in zip(self.groups, params):
            g.crop_w, g.crop_h, g.crop_x, g.crop_y, g.flip = int(cw), int(ch), int(ox), int(oy), int(bool(fl))

    def _upload(self):
        # a fresh pinned buffer per upload: the copy is asynchronous on the current stream, and the caching host allocator
        # keeps the buffer until that copy has run
        host = torch.empty(C.sizeof(self.groups), dtype=torch.uint8, pin_memory=True)
        C.memmove(host.data_ptr(), C.addressof(self.groups), C.sizeof(self.groups))
        with torch.cuda.device(self.device):
            self.groups_dev.copy_(host, non_blocking=True)

    def set_train_params(self, params):
        """new crop windows and flips, validated and copied into groups_dev (on the current stream)"""
        self._set_params(params)
        check(lib.ssnb_frame_transform_workspace_bytes(C.byref(self.cfg), self.groups, len(self.groups), None, None), None,
              "frame_transform_workspace_bytes")
        self._upload()

    def run(self, src, dst):
        with torch.cuda.device(self.device):
            check(lib.ssnb_frame_transform(C.byref(self.cfg), self.groups, self.groups_dev.data_ptr(), len(self.groups), src.data_ptr(),
                                           src.numel(), dst.data_ptr(), dst.numel(), self.workspace.data_ptr(), self.workspace.numel(),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "frame_transform")
        return dst


def _src(groups, device):
    if all(g.is_cuda for g in groups):
        return torch.cat([g.reshape(-1) for g in groups]).to(device)
    host = torch.cat([g.reshape(-1).cpu() for g in groups]).pin_memory()
    return host.to(device, non_blocking=True)


def _transform(mode, frames, frame_channels, out_size, scale_size, mean, std, invert_even, params=None, device=None, div=False):
    if div:
        raise NotImplementedError("only ToTorchFormatTensor(div=False) normalisation (BNInception) is implemented")
    groups = _groups(frames)
    if device is None:
        device = next((g.device for g in groups if g.is_cuda), torch.device("cuda", torch.cuda.current_device()))
    channels = groups[0].shape[3]
    if invert_even is None:             # GroupOverSample inverts the flipped L images at even positions
        invert_even = channels == 1
    plan = FramePlan(mode, [tuple(g.shape[:3]) for g in groups], channels, out_size, scale_size, mean, std, invert_even, device, params)
    dst = torch.empty(plan.dst_floats, dtype=torch.float32, device=device)
    plan.run(_src(groups, device), dst)
    return dst.view(-1, frame_channels, out_size, out_size)


def train_frames(frames, params, mean, std, frame_channels, input_size=224, is_flow=False, device=None, div=False):
    """GroupMultiScaleCrop + GroupRandomHorizontalFlip (params from sample_train_params, one per group) + Stack(roll=True) +
    ToTorchFormatTensor(div=False) + GroupNormalize(mean, std) -> CUDA fp32 [frames, frame_channels, input_size, input_size]"""
    return _transform(FRAMES_TRAIN, frames, frame_channels, input_size, 0, mean, std, is_flow, params, device, div)


def oversample_frames(frames, mean, std, frame_channels, crop_size=224, scale_size=256, device=None, div=False):
    """GroupOverSample(crop_size, scale_size) + the same tail: per group, 10 crops in the reference's crop-major order (each
    window's images plain, then flipped), the order SSN.test_scores expects"""
    return _transform(FRAMES_OVERSAMPLE, frames, frame_channels, crop_size, scale_size, mean, std, None, None, device, div)


def center_crop_frames(frames, mean, std, frame_channels, crop_size=224, scale_size=256, device=None, div=False):
    """GroupScale(scale_size) + GroupCenterCrop(crop_size) + the same tail (1-crop test, validation)"""
    return _transform(FRAMES_CENTER, frames, frame_channels, crop_size, scale_size, mean, std, False, None, device, div)


class GroupToUint8:
    """SSNDataSet(transform=...) on the host: a group of PIL images (RGB, or L for Flow) -> one uint8 tensor [n, H, W, C], so
    the DataLoader carries uint8 frames and the crops, flips and normalisation run on the GPU.  SSNDataSet.get_training_data
    concatenates a video's proposals (torch.cat, ssn_dataset.py:486), so a training sample holds [P * n, H, W, C]:
    proposal_groups() cuts a batch back into one group per proposal."""

    def __call__(self, img_group):
        return torch.from_numpy(np.stack([np.asarray(im).reshape(im.size[1], im.size[0], -1) for im in img_group]))


def proposal_groups(frames, props_per_video):
    """The proposal groups of a training batch: frames is the collated [B, P * n, H, W, C] tensor (videos of one resolution,
    default_collate) or the list of per-video [P * n, H, W, C] tensors from collate_ragged (videos of different resolutions).
    -> list of B * P tensors [n, H, W, C] in video-major, proposal order: the groups GroupMultiScaleCrop saw, one draw each."""
    videos = frames.unbind(0) if torch.is_tensor(frames) else frames
    out = []
    for v in videos:
        if v.shape[0] % props_per_video:
            raise ValueError("a video's %d frames do not split into %d proposals" % (v.shape[0], props_per_video))
        out += list(v.reshape(props_per_video, -1, *v.shape[1:]).unbind(0))
    return out


def collate_ragged(batch):
    """DataLoader collate_fn for SSNDataSet samples whose videos differ in resolution: default_collate cannot stack their
    frames, so the frames stay a list of per-video tensors and every other field is collated as usual."""
    from torch.utils.data import default_collate
    rest = default_collate([b[1:] for b in batch])
    return [[b[0] for b in batch]] + list(rest)
