"""numpy restatement of the reference's frame transforms (transforms.py:41-206, 256-288) and of the PIL 8-bit BILINEAR resize they
call, for the GPU tests to compare against bit for bit.  It deliberately does not import PIL: tests/golden/frames.npz, written
from the real transforms.py and PIL by oracle/gen_golden_frames.py, checks this module, and this module checks the GPU.

Images are uint8 numpy arrays [H, W, C] (C = 3 for RGB, 1 for L).  Every composition returns what the reference hands to the
model: the fp32 tensor after Stack(roll=True), ToTorchFormatTensor(div=False) and GroupNormalize, [planes, out, out].
"""
import numpy as np

PREC = 22


def pil_coeffs(in_size, out_size):
    """libImaging/Resample.c precompute_coeffs (bilinear) + normalize_coeffs_8bpc: per output index (xmin, int32 weights).
    Python floats are IEEE doubles and every operation below rounds once, as the C code does without FMA contraction."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ss = 1.0 / filterscale
    out = []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size)
        ws = []
        for x in range(xmax - xmin):
            t = abs((x + xmin - center + 0.5) * ss)
            ws.append(1.0 - t if t < 1.0 else 0.0)
        ww = 0.0
        for w in ws:
            ww += w
        if ww != 0.0:
            ws = [w / ww for w in ws]
        out.append((xmin, np.array([int(-0.5 + w * (1 << PREC)) if w < 0 else int(0.5 + w * (1 << PREC)) for w in ws], np.int64)))
    return out


def _pass(img, axis, out_size):
    """one fixed-point pass along axis (1: horizontal, 0: vertical) -> uint8"""
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    res = np.empty((out_size,) + src.shape[1:], np.uint8)
    for o, (xmin, k) in enumerate(pil_coeffs(src.shape[0], out_size)):
        acc = np.full(src.shape[1:], 1 << (PREC - 1), np.int64)
        for j, kj in enumerate(k):
            acc += src[xmin + j] * kj
        res[o] = np.where(acc >= (1 << PREC << 8), 255, np.where(acc <= 0, 0, acc >> PREC))
    return np.moveaxis(res, 0, axis)


def resize(img, w, h):
    """Image.resize((w, h), BILINEAR): horizontal pass, then vertical; an unchanged axis is skipped"""
    H, W = img.shape[:2]
    if (w, h) == (W, H):
        return img.copy()
    if w != W:
        img = _pass(img, 1, w)
    if h != H:
        img = _pass(img, 0, h)
    return img


def crop(img, x, y, w, h):
    """Image.crop((x, y, x + w, y + h)): zeros outside the image"""
    H, W, C = img.shape
    out = np.zeros((h, w, C), np.uint8)
    x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + w, W), min(y + h, H)
    if x1 > x0 and y1 > y0:
        out[y0 - y:y1 - y, x0 - x:x1 - x] = img[y0:y1, x0:x1]
    return out


def scaled_size(h, w, size):
    """torchvision Resize(size) output (h, w): the shorter edge becomes size, long = int(size * long / short)"""
    short, long_ = (w, h) if w <= h else (h, w)
    new_long = int(size * long_ / short)
    return (new_long, size) if w <= h else (size, new_long)


def group_scale(img, size):
    h, w = scaled_size(img.shape[0], img.shape[1], size)
    return img if (h, w) == img.shape[:2] else resize(img, w, h)


def flip(img, invert):
    out = img[:, ::-1]
    return 255 - out if invert else out


def stack_normalize(images, mean, std):
    """Stack(roll=True) + ToTorchFormatTensor(div=False) + GroupNormalize: [planes, h, w] fp32, RGB planes in BGR order"""
    planes = np.concatenate([np.ascontiguousarray(im[:, :, ::-1]).transpose(2, 0, 1) for im in images], 0).astype(np.float32)
    n = planes.shape[0]
    rep_mean = list(mean) * (n // len(mean))
    rep_std = list(std) * (n // len(std))
    for p, (m, s) in enumerate(zip(rep_mean, rep_std)):
        planes[p] = (planes[p] - np.float32(m)) / np.float32(s)
    return planes


def fill_fix_offset(more_fix_crop, image_w, image_h, crop_w, crop_h):
    w_step = (image_w - crop_w) // 4
    h_step = (image_h - crop_h) // 4
    ret = [(0, 0), (4 * w_step, 0), (0, 4 * h_step), (4 * w_step, 4 * h_step), (2 * w_step, 2 * h_step)]
    if more_fix_crop:
        ret += [(0, 2 * h_step), (4 * w_step, 2 * h_step), (2 * w_step, 4 * h_step), (2 * w_step, 0 * h_step),
                (1 * w_step, 1 * h_step), (3 * w_step, 1 * h_step), (1 * w_step, 3 * h_step), (3 * w_step, 3 * h_step)]
    return ret


def train_group(images, params, out_size, mean, std, is_flow):
    """GroupMultiScaleCrop (crop, then resize) + GroupRandomHorizontalFlip with params = (crop_w, crop_h, off_w, off_h, flip)"""
    cw, ch, ox, oy, flipped = params
    res = [resize(crop(im, ox, oy, cw, ch), out_size, out_size) for im in images]
    if flipped:
        res = [flip(im, is_flow and i % 2 == 0) for i, im in enumerate(res)]
    return stack_normalize(res, mean, std)


def oversample_group(images, out_size, scale_size, mean, std):
    """GroupOverSample(out_size, scale_size): per window all images plain, then all flipped (L images at even positions
    inverted)"""
    images = [group_scale(im, scale_size) for im in images]
    h, w = images[0].shape[:2]
    res = []
    for ox, oy in fill_fix_offset(False, w, h, out_size, out_size):
        crops = [crop(im, ox, oy, out_size, out_size) for im in images]
        res += crops
        res += [flip(c, im.shape[2] == 1 and i % 2 == 0) for i, (c, im) in enumerate(zip(crops, images))]
    return stack_normalize(res, mean, std)


def center_group(images, out_size, scale_size, mean, std):
    """GroupScale(scale_size) + GroupCenterCrop(out_size): offset int(round((h - th) / 2.0)), half to even"""
    images = [group_scale(im, scale_size) for im in images]
    h, w = images[0].shape[:2]
    oy, ox = int(round((h - out_size) / 2.0)), int(round((w - out_size) / 2.0))
    return stack_normalize([crop(im, ox, oy, out_size, out_size) for im in images], mean, std)
