"""JPEG decode on the GPU: the data sets' frame loading, Image.open(path).convert('RGB') for RGB frames and .convert('L') for the
x / y planes of Flow (SSNDataSet._load_image, ssn_dataset.py:187-194; BinaryDataSet._load_image, load_binary_score.py:198-205),
computed by libssn_b200.so (csrc/jpeg.cu) and bitwise equal to Pillow over libjpeg-turbo.

The DataLoader workers read the files' bytes (JpegBytesLoader as the data set's _load_image, GroupToJpegBytes as its transform,
collate_jpeg as the loader's collate_fn) and one call per batch decodes every frame into the uint8 [n, H, W, C] groups that
ops.frame_transforms takes:

    frames = decode_jpeg(byte_groups, mode='RGB')          # list of CUDA uint8 [n, H, W, 3]
    x = train_frames(proposal_groups(frames, P), params, mean, std, frame_channels)

Huffman-coded sequential 8-bit JPEG only (what video frame extractors write): grayscale or YCbCr at 4:4:4, 4:2:2 or 4:2:0, any
size, with or without restart intervals.  Other streams are refused before anything runs on the GPU, with the image and the
reason; there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np
import torch

from ssn_b200._lib import lib, JpegInput, JpegImageInfo

STATUS_TEXT = {1: "entropy-coded data truncated", 2: "invalid Huffman code", 3: "AC coefficient run past the end of the block",
               4: "restart marker missing or out of sequence"}
_CHANNELS = {"RGB": 3, "L": 1}


def pack_jpeg_group(blobs):
    """A group of JPEG files' bytes -> one uint8 tensor: int64 n, n int64 lengths, then the bytes.  Tensors of several groups
    concatenated with torch.cat (SSNDataSet.get_training_data does so per video, ssn_dataset.py:486) read back as one group."""
    blobs = [bytes(b) for b in blobs]
    head = np.array([len(blobs)] + [len(b) for b in blobs], np.int64).tobytes()
    return torch.frombuffer(bytearray(head + b"".join(blobs)), dtype=torch.uint8)


def unpack_jpeg_group(packed):
    """pack_jpeg_group's tensor (or several concatenated) -> (uint8 buffer, int64 offsets [n + 1]) of one group"""
    buf = packed.cpu().numpy() if torch.is_tensor(packed) else np.asarray(packed, np.uint8)
    buf = buf.reshape(-1)
    starts, ends, p = [], [], 0
    while p < buf.size:
        n = int(buf[p:p + 8].view(np.int64)[0])
        lens = buf[p + 8:p + 8 * (n + 1)].view(np.int64)
        p += 8 * (n + 1)
        for ln in lens.tolist():
            starts.append(p)
            p += ln
            ends.append(p)
    if p != buf.size:
        raise ValueError("not a packed JPEG group (pack_jpeg_group)")
    return buf, np.array(starts, np.int64), np.array(ends, np.int64)


def _group(g):
    """one group -> (uint8 buffer, starts, ends): a list of bytes-like objects, a (buffer, offsets [n + 1]) pair, or a packed
    tensor from pack_jpeg_group"""
    if isinstance(g, tuple) and len(g) == 2 and (torch.is_tensor(g[0]) or isinstance(g[0], np.ndarray)):
        buf = g[0].cpu().numpy() if torch.is_tensor(g[0]) else np.asarray(g[0], np.uint8)
        off = np.asarray(g[1], np.int64)
        if buf.dtype != np.uint8 or off.ndim != 1 or off.size < 1 or (np.diff(off) < 0).any() or off[0] < 0 or off[-1] > buf.size:
            raise ValueError("a (buffer, offsets) group needs a uint8 buffer and n + 1 ascending offsets inside it")
        return buf.reshape(-1), off[:-1], off[1:]
    if torch.is_tensor(g) or isinstance(g, np.ndarray):
        return unpack_jpeg_group(g)
    parts = [bytes(b) for b in g]
    ends = np.cumsum([len(b) for b in parts], dtype=np.int64)
    return np.frombuffer(b"".join(parts), np.uint8), ends - np.array([len(b) for b in parts], np.int64), ends


class JpegPlan:
    """The host plan of one call: every image parsed (the library refuses unsupported streams here, before any launch), the
    device table and the sizes.  Holds the call's bytes as one uint8 numpy buffer; `images` gives each image's
    ssnb_jpeg_image_info."""

    def __init__(self, buf, starts, ends, channels):
        self.buf = np.ascontiguousarray(buf, np.uint8)
        n = len(starts)
        self.inputs = (JpegInput * n)()
        for e, s, t, c in zip(self.inputs, starts, ends, channels):
            e.offset, e.bytes, e.channels = int(s), int(t - s), int(c)
        self.handle = C.c_void_p()
        bad = C.c_int(-1)
        rc = lib.ssnb_jpeg_plan_create(self.buf.ctypes.data, self.buf.size, self.inputs, n, C.byref(self.handle), C.byref(bad))
        if rc != 0:
            msg = (lib.ssnb_last_error(None) or b"").decode()
            self.handle = None
            raise JpegRefused(bad.value, msg.split(": ", 2)[-1] if bad.value >= 0 else msg, rc)
        tb, ws, ob = C.c_size_t(), C.c_size_t(), C.c_int64()
        lib.ssnb_jpeg_plan_sizes(self.handle, C.byref(tb), C.byref(ws), C.byref(ob))
        self.table_bytes, self.workspace_bytes, self.out_bytes = tb.value, ws.value, ob.value
        self.images = []
        for i in range(n):
            info = JpegImageInfo()
            lib.ssnb_jpeg_plan_image(self.handle, i, C.byref(info))
            self.images.append(info)

    def __del__(self):
        if getattr(self, "handle", None):
            lib.ssnb_jpeg_plan_destroy(self.handle)
            self.handle = None

    def upload(self, device):
        """the device table and the bytes in one pinned host buffer, copied to `device` in one asynchronous copy"""
        host = torch.empty(self.table_bytes + self.buf.size, dtype=torch.uint8, pin_memory=True)
        if lib.ssnb_jpeg_plan_write_table(self.handle, host.data_ptr(), self.table_bytes) != 0:
            raise RuntimeError((lib.ssnb_last_error(None) or b"").decode())
        host[self.table_bytes:].numpy()[:] = self.buf
        with torch.cuda.device(device):
            return host.to(device, non_blocking=True)

    def run(self, dev, out, status, workspace):
        """enqueue the decode on the current stream: dev from upload(), out uint8 [out_bytes], status int32 [n], workspace uint8"""
        with torch.cuda.device(dev.device):
            rc = lib.ssnb_jpeg_decode(self.handle, dev.data_ptr(), dev.data_ptr() + self.table_bytes, dev.numel() - self.table_bytes,
                                      out.data_ptr(), out.numel(), status.data_ptr(), workspace.data_ptr(), workspace.numel(),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError("libssn_b200 jpeg_decode failed (code %d): %s" % (rc, (lib.ssnb_last_error(None) or b"").decode()))


class JpegRefused(ValueError):
    """A stream the decoder does not support, or a malformed header: `image` is its index in the call."""

    def __init__(self, image, reason, code):
        super().__init__("image %d: %s" % (image, reason))
        self.image, self.reason, self.code = image, reason, code


def _where(i, sizes):
    g = int(np.searchsorted(np.cumsum(sizes), i, side="right"))
    return g, i - int(sum(sizes[:g]))


def decode_jpeg(blobs, mode="RGB", device=None, check=True):
    """Decode groups of JPEG files on the GPU: blobs is a list of groups, each a list of bytes-like objects, a (uint8 buffer,
    offsets [n + 1]) pair or a pack_jpeg_group tensor; mode 'RGB' or 'L' for the whole call or one per group.  Returns one CUDA
    uint8 tensor [n, H, W, C] per group (C = 3 for 'RGB', 1 for 'L'; a group's images must share their size), bitwise equal to
    np.asarray(Image.open(f).convert(mode)).

    The bytes go to the device in one copy through pinned memory and the decode is enqueued on the current stream.  A stream
    the decoder does not support raises ValueError naming the image before anything is launched.  With check=True the call
    then waits for the decode and raises ValueError naming the first image whose entropy-coded data is corrupt or truncated;
    check=False returns (groups, status) instead, status int32 [images] on the device (0: decoded, else the STATUS_TEXT
    code), without waiting."""
    groups = [_group(g) for g in blobs]
    if not groups:
        return ([], None) if not check else []
    modes = [mode] * len(groups) if isinstance(mode, str) else list(mode)
    if len(modes) != len(groups) or any(m not in _CHANNELS for m in modes):
        raise ValueError("mode must be 'RGB' or 'L', or one of them per group")
    sizes = [len(g[1]) for g in groups]
    if min(sizes) < 1:
        raise ValueError("every group needs at least one image")
    base = np.cumsum([0] + [g[0].size for g in groups])
    buf = np.concatenate([g[0] for g in groups])
    starts = np.concatenate([g[1] + b for g, b in zip(groups, base)])
    ends = np.concatenate([g[2] + b for g, b in zip(groups, base)])
    channels = np.repeat([_CHANNELS[m] for m in modes], sizes)
    try:
        plan = JpegPlan(buf, starts, ends, channels)
    except JpegRefused as e:
        g, j = _where(e.image, sizes)
        raise ValueError("decode_jpeg: image %d (group %d, image %d): %s" % (e.image, g, j, e.reason)) from None
    shapes, first = [], 0
    for g, n in enumerate(sizes):
        ims = plan.images[first:first + n]
        if len({(im.height, im.width) for im in ims}) != 1:
            raise ValueError("decode_jpeg: group %d holds images of different sizes %s" % (g, sorted({(im.height, im.width) for im in ims})))
        shapes.append((n, ims[0].height, ims[0].width, _CHANNELS[modes[g]]))
        first += n
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    dev = plan.upload(device)
    out = torch.empty(max(plan.out_bytes, 1), dtype=torch.uint8, device=device)
    workspace = torch.empty(max(plan.workspace_bytes, 1), dtype=torch.uint8, device=device)
    status = torch.empty(len(plan.images), dtype=torch.int32, device=device)
    plan.run(dev, out, status, workspace)
    res, first = [], 0
    for g, shp in enumerate(shapes):
        off = plan.images[first].out_offset
        res.append(out[off:off + int(np.prod(shp))].view(shp))
        first += shp[0]
    if not check:
        return res, status
    st = status.cpu().numpy()
    if st.any():
        i = int(np.flatnonzero(st)[0])
        g, j = _where(i, sizes)
        raise ValueError("decode_jpeg: image %d (group %d, image %d): %s" % (i, g, j, STATUS_TEXT[int(st[i])]))
    return res


def _read(path):
    with open(path, "rb") as f:
        return f.read()


class JpegBytesLoader:
    """The data sets' _load_image (SSNDataSet, ssn_dataset.py:187-194; BinaryDataSet, load_binary_score.py:198-205) reading each
    frame file's bytes instead of opening it with PIL: [rgb] for RGB and RGBDiff, [x, y] for Flow, the order the reference
    stacks the planes in.  Put it first among the bases so it overrides the data set's own:

        class SSNBytesDataSet(JpegBytesLoader, SSNDataSet): pass
        dataset = SSNBytesDataSet(..., transform=GroupToJpegBytes())

    Everything else the data set does, its random draws included, is unchanged."""

    def _load_image(self, directory, idx):
        if self.modality == 'RGB' or self.modality == 'RGBDiff':
            return [_read(os.path.join(directory, self.image_tmpl.format(idx)))]
        elif self.modality == 'Flow':
            return [_read(os.path.join(directory, self.image_tmpl.format('x', idx))),
                    _read(os.path.join(directory, self.image_tmpl.format('y', idx)))]


class GroupToJpegBytes:
    """The data set's transform with JpegBytesLoader, the counterpart of GroupToUint8: a group of frame files' bytes -> one
    packed uint8 tensor (pack_jpeg_group).  get_training_data's torch.cat of a video's proposals gives one tensor per video,
    which decode_jpeg reads as one group of P * n images."""

    def __call__(self, blobs):
        return pack_jpeg_group(blobs)


def collate_jpeg(batch):
    """DataLoader collate_fn for samples whose frames are packed JPEG bytes: the packed tensors differ in length, so they stay a
    list (one group per video for decode_jpeg) and every other field is collated as usual."""
    from torch.utils.data import default_collate
    rest = default_collate([b[1:] for b in batch])
    return [[b[0] for b in batch]] + list(rest)
