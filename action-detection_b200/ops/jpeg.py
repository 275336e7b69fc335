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

encode_jpeg is the other direction, the files of the extraction step (DenseFlow's img_%05d.jpg and flow_{x,y}_%05d.jpg):
CUDA uint8 images -> the bytes Pillow's Image.save(f, quality=q) writes, computed by csrc/jpeg_encode.cu.  JpegEncodePlan
keeps one call's buffers so the encode can be repeated or captured in a CUDA graph.  restart_marker_blocks /
restart_marker_rows write Pillow's restart intervals, so that decode_jpeg splits each file into independent intervals:

    files = encode_jpeg(frames, mode='RGB', quality=95, restart_marker_rows=1)    # 16 intervals per 340 x 256 frame

jpeg_roundtrip joins the two without the files: CUDA uint8 images -> what decode_jpeg returns for the files encode_jpeg
writes of them (csrc/jpeg_roundtrip.cu, no Huffman coding), so decoded video frames or flow planes become the exact inputs
the data sets would read from the extraction step's files.  JpegRoundtripPlan keeps one call's buffers for repeats and
CUDA graphs.
"""
import ctypes as C
import os

import numpy as np
import torch

from ssn_b200._lib import lib, JpegInput, JpegImageInfo, JpegEncodeImage, JPEG_ENC_L, JPEG_ENC_RGB

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


# ------------------------------------------------------------------------------------------------------------------ encode

_ENC_MODES = {"L": (JPEG_ENC_L, 1), "RGB": (JPEG_ENC_RGB, 3)}


def jpeg_encode_capacity(mode, height, width, restart_marker_blocks=0, restart_marker_rows=0):
    """the bytes the encoder reserves for one image's file (its worst case; 0 for a bad mode, size or restart option)"""
    return int(lib.ssnb_jpeg_encode_restart_capacity(_ENC_MODES[mode][0] if mode in _ENC_MODES else 0, int(height), int(width),
                                                     int(restart_marker_blocks), int(restart_marker_rows)))


def _enc_mode(mode):
    if mode not in _ENC_MODES:
        raise ValueError("encode_jpeg: mode must be 'RGB' or 'L'")
    return _ENC_MODES[mode]


def _enc_restart(restart_marker_blocks, restart_marker_rows):
    """the restart options as ints; ValueError for those the library refuses (both set, negative, blocks above 65535)"""
    b, r = int(restart_marker_blocks), int(restart_marker_rows)
    if b < 0 or r < 0:
        raise ValueError("encode_jpeg: restart_marker_blocks and restart_marker_rows must be >= 0")
    if b and r:
        raise ValueError("encode_jpeg: restart_marker_blocks and restart_marker_rows cannot both be set")
    if b > 65535:
        raise ValueError("encode_jpeg: restart_marker_blocks must be <= 65535 (DRI's 16 bits)")
    return b, r


def _pixel_buffer(images, sizes, channels, mode, what):
    """CUDA uint8 [N, H, W, C] or a list of [H, W, C] of the given sizes -> one contiguous uint8 buffer"""
    ts = [images] if torch.is_tensor(images) else list(images)
    if not all(torch.is_tensor(t) and t.is_cuda for t in ts):
        raise RuntimeError("%s needs CUDA uint8 images (no CPU path)" % what)
    if any(t.dtype != torch.uint8 for t in ts):
        raise ValueError("%s: images must be uint8" % what)
    if torch.is_tensor(images):
        if images.dim() != 4 or images.shape[3] != channels:
            raise ValueError("%s: images must be [N, H, W, %d] for mode %r" % (what, channels, mode))
        shapes = [tuple(images.shape[1:3])] * images.shape[0]
    else:
        if any(t.dim() != 3 or t.shape[2] != channels for t in ts):
            raise ValueError("%s: each image must be [H, W, %d] for mode %r" % (what, channels, mode))
        shapes = [tuple(t.shape[:2]) for t in ts]
    if shapes != sizes:
        raise ValueError("%s: the images' sizes differ from the plan's" % what)
    if torch.is_tensor(images):
        return images.contiguous().reshape(-1)
    return torch.cat([t.reshape(-1) for t in ts])


class JpegEncodePlan:
    """One encode call's sizes, mode, quality and restart option with its device buffers: the image table, the workspace, the
    output slots (image i's file starts at out[slots[i]]) and the int64 lengths.  plan.run(images) only enqueues, so it can be
    repeated or captured in a CUDA graph on new pixels of the same sizes; plan.files() waits and returns one bytes object per
    image."""

    def __init__(self, sizes, mode="RGB", quality=95, device=None, restart_marker_blocks=0, restart_marker_rows=0):
        self.mode, self.quality = mode, int(quality)
        self._code, self.channels = _enc_mode(mode)
        self.restart_marker_blocks, self.restart_marker_rows = _enc_restart(restart_marker_blocks, restart_marker_rows)
        rst = (self.restart_marker_blocks, self.restart_marker_rows)
        self.sizes = [(int(h), int(w)) for h, w in sizes]
        n = len(self.sizes)
        if n < 1:
            raise ValueError("encode_jpeg: no image")
        self.images = (JpegEncodeImage * n)()
        off = 0
        for e, (h, w) in zip(self.images, self.sizes):
            e.src_offset, e.height, e.width = off, h, w
            off += max(h, 0) * max(w, 0) * self.channels
        self.src_bytes = off
        ws, ob = C.c_size_t(), C.c_int64()
        if lib.ssnb_jpeg_encode_restart_sizes(self._code, self.quality, *rst, self.images, n, C.byref(ws), C.byref(ob)) != 0:
            raise ValueError("encode_jpeg: " + (lib.ssnb_last_error(None) or b"").decode().split(": ", 1)[-1])
        caps = [lib.ssnb_jpeg_encode_restart_capacity(self._code, h, w, *rst) for h, w in self.sizes]
        self.slots = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.images_dev = torch.frombuffer(bytearray(bytes(self.images)), dtype=torch.uint8).to(dev)
        self.workspace = torch.empty(ws.value, dtype=torch.uint8, device=dev)
        self.out = torch.empty(ob.value, dtype=torch.uint8, device=dev)
        self.lengths = torch.zeros(n, dtype=torch.int64, device=dev)

    def _pixels(self, images):
        """CUDA uint8 [N, H, W, C] or a list of [H, W, C] of the plan's sizes -> one contiguous uint8 buffer"""
        return _pixel_buffer(images, self.sizes, self.channels, self.mode, "encode_jpeg")

    def run(self, images):
        """enqueue the encode of `images` on the current stream; returns (out, lengths) on the device"""
        src = self._pixels(images)
        if src.device != self.out.device:
            raise ValueError("encode_jpeg: images on %s, plan on %s" % (src.device, self.out.device))
        self._src = src                       # kept alive until the next run
        with torch.cuda.device(self.out.device):
            rc = lib.ssnb_jpeg_encode_restart(self._code, self.quality, self.restart_marker_blocks, self.restart_marker_rows, src.data_ptr(),
                                              src.numel(), self.images, self.images_dev.data_ptr(), len(self.sizes), self.out.data_ptr(),
                                              self.out.numel(), self.lengths.data_ptr(), self.workspace.data_ptr(), self.workspace.numel(),
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError("libssn_b200 jpeg_encode failed (code %d): %s" % (rc, (lib.ssnb_last_error(None) or b"").decode()))
        return self.out, self.lengths

    def files(self):
        """wait for the last run and return each image's file as bytes (one device-to-host copy of the files' bytes)"""
        lens = self.lengths.cpu().numpy()
        flat = torch.cat([self.out[int(o):int(o) + int(l)] for o, l in zip(self.slots, lens)]).cpu().numpy().tobytes()
        ends = np.cumsum(lens)
        return [flat[e - l:e] for e, l in zip(ends.tolist(), lens.tolist())]


def encode_jpeg(images, mode="RGB", quality=95, restart_marker_blocks=0, restart_marker_rows=0):
    """Encode CUDA uint8 images on the GPU: [N, H, W, C] or a list of ragged [H, W, C], C = 3 for 'RGB' and 1 for 'L'.  Returns
    one bytes object per image, equal to what Image.fromarray(img).save(f, format='JPEG', quality=quality) writes (Pillow over
    libjpeg-turbo; cv2.imencode writes the same bytes): baseline, 4:2:0 for 'RGB', no optimize, no metadata.  quality 1 .. 100.

    restart_marker_blocks = n (a restart interval of n MCUs, 1 .. 65535; cv2's IMWRITE_JPEG_RST_INTERVAL) or
    restart_marker_rows = r (r MCU rows per interval, min(r * MCUs per row, 65535) MCUs per image) give the bytes of Pillow's
    save with the same keyword.  The decoded pixels are those of the file without markers; decode_jpeg decodes each interval
    in a thread of its own.  Setting both, or a negative value, raises ValueError."""
    restart = _enc_restart(restart_marker_blocks, restart_marker_rows)
    if torch.is_tensor(images):
        if not images.is_cuda:
            raise RuntimeError("encode_jpeg needs CUDA uint8 images (no CPU path)")
        if images.dim() != 4:
            raise ValueError("encode_jpeg: images must be [N, H, W, C] or a list of [H, W, C]")
        sizes, device = [tuple(images.shape[1:3])] * images.shape[0], images.device
    else:
        images = list(images)
        if not images:
            return []
        if not all(torch.is_tensor(t) and t.is_cuda for t in images):
            raise RuntimeError("encode_jpeg needs CUDA uint8 images (no CPU path)")
        if any(t.dim() != 3 for t in images):
            raise ValueError("encode_jpeg: images must be [N, H, W, C] or a list of [H, W, C]")
        sizes, device = [tuple(t.shape[:2]) for t in images], images[0].device
    if len(sizes) == 0:
        return []
    plan = JpegEncodePlan(sizes, mode, quality, device, *restart)
    plan.run(images)
    return plan.files()


# ------------------------------------------------------------------------------------------------------------- round trip

def _sizes_of(images, what):
    """[N, H, W, C] or a list of [H, W, C] CUDA tensors -> ([(H, W)] per image, device); CPU tensors raise"""
    if torch.is_tensor(images):
        if not images.is_cuda:
            raise RuntimeError("%s needs CUDA uint8 images (no CPU path)" % what)
        if images.dim() != 4:
            raise ValueError("%s: images must be [N, H, W, C] or a list of [H, W, C]" % what)
        return [tuple(images.shape[1:3])] * images.shape[0], images.device
    if not all(torch.is_tensor(t) and t.is_cuda for t in images):
        raise RuntimeError("%s needs CUDA uint8 images (no CPU path)" % what)
    if any(t.dim() != 3 for t in images):
        raise ValueError("%s: images must be [N, H, W, C] or a list of [H, W, C]" % what)
    return [tuple(t.shape[:2]) for t in images], (images[0].device if images else None)


class JpegRoundtripPlan:
    """One round-trip call's sizes, mode and quality with its device image table and output buffer (image i's result at
    out[offsets[i]:offsets[i + 1]], images back to back).  plan.run(images) only enqueues, so it can be repeated or captured
    in a CUDA graph on new pixels of the same sizes; it returns the results as views of plan.out."""

    def __init__(self, sizes, mode="RGB", quality=95, device=None):
        if mode not in _ENC_MODES:
            raise ValueError("jpeg_roundtrip: mode must be 'RGB' or 'L'")
        self.mode, self.quality = mode, int(quality)
        self._code, self.channels = _ENC_MODES[mode]
        if not 1 <= self.quality <= 100:
            raise ValueError("jpeg_roundtrip: quality must be 1 .. 100")
        self.sizes = [(int(h), int(w)) for h, w in sizes]
        n = len(self.sizes)
        if n < 1:
            raise ValueError("jpeg_roundtrip: no image")
        if any(not (1 <= h <= 65500 and 1 <= w <= 65500) for h, w in self.sizes):
            raise ValueError("jpeg_roundtrip: height and width must be 1 .. 65500")
        self.images = (JpegEncodeImage * n)()
        self.offsets = np.zeros(n + 1, np.int64)
        for i, (e, (h, w)) in enumerate(zip(self.images, self.sizes)):
            e.src_offset, e.height, e.width = int(self.offsets[i]), h, w
            self.offsets[i + 1] = self.offsets[i] + h * w * self.channels
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.images_dev = torch.frombuffer(bytearray(bytes(self.images)), dtype=torch.uint8).to(dev)
        self.out = torch.empty(int(self.offsets[-1]), dtype=torch.uint8, device=dev)

    def run(self, images):
        """enqueue the round trip of `images` ([N, H, W, C] or a list of [H, W, C] of the plan's sizes) on the current stream;
        -> uint8 [N, H, W, C] for a tensor, else a list of [H, W, C], views of plan.out"""
        src = _pixel_buffer(images, self.sizes, self.channels, self.mode, "jpeg_roundtrip")
        if src.device != self.out.device:
            raise ValueError("jpeg_roundtrip: images on %s, plan on %s" % (src.device, self.out.device))
        self._src = src                       # kept alive until the next run
        with torch.cuda.device(self.out.device):
            rc = lib.ssnb_jpeg_roundtrip(self._code, self.quality, src.data_ptr(), src.numel(), self.images, self.images_dev.data_ptr(),
                                         len(self.sizes), self.out.data_ptr(), self.out.numel(),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError("libssn_b200 jpeg_roundtrip failed (code %d): %s" % (rc, (lib.ssnb_last_error(None) or b"").decode()))
        if torch.is_tensor(images):
            return self.out.view(len(self.sizes), *self.sizes[0], self.channels)
        return [self.out[int(a):int(b)].view(h, w, self.channels) for a, b, (h, w) in zip(self.offsets[:-1], self.offsets[1:], self.sizes)]


def jpeg_roundtrip(images, mode="RGB", quality=95):
    """The pixels the data sets' loaders read back from JPEG files of CUDA uint8 images, computed without the files: [N, H, W,
    C] or a list of ragged [H, W, C], C = 3 for 'RGB' and 1 for 'L'.  Returns the same structure, uint8 on the same device,
    bitwise equal to decode_jpeg(encode_jpeg(images, mode, quality), mode), i.e. to
    np.asarray(Image.open(BytesIO(f)).convert(mode)) of the file f that Image.fromarray(img).save(f, format='JPEG',
    quality=quality) writes: 4:2:0 for 'RGB'.  quality 1 .. 100.  Enqueued on the current stream; nothing waits."""
    if not torch.is_tensor(images):
        images = list(images)
    sizes, device = _sizes_of(images, "jpeg_roundtrip")
    if not sizes:
        return images.new_empty(images.shape) if torch.is_tensor(images) else []
    return JpegRoundtripPlan(sizes, mode, quality, device).run(images)
