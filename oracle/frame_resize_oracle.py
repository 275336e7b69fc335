"""numpy restatement of OpenCV 4's cv2.resize(img, (dst_w, dst_h), interpolation=cv2.INTER_LINEAR) on uint8 [H, W, C]
frames: DenseFlow's cv::resize(frame, image, Size(new_width, new_height)) before the flow (extract_gpu --new_width 340
--new_height 256).  Every function cites the part of modules/imgproc/src/resize.cpp it follows; csrc/frame_resize.cu
computes the same integers.  The yardstick is cv2 4.13 (tests/golden/frame_resize.npz holds its outputs); the OpenCV 2.4
inside a DenseFlow build is not checked.

Paths, in the order OpenCV takes them:
    copy        cv::resize: dsize == ssize -> src.copyTo(dst)
    area fast   hal::resize: INTER_LINEAR with scale_x == scale_y == 2 exactly -> INTER_AREA -> resizeAreaFast_ with
                ResizeAreaFastVec: (a + b + c + d + 2) >> 2 over each 2 x 2 block
    linear      hal::resize's coefficient tables, then resizeGeneric_ with HResizeLinear<uchar, int, short, 2048> and
                VResizeLinear with VResizeLinearVec_32s8u (OpenCV's universal-intrinsics vertical pass)
The copy and the area path equal the linear rule bit for bit (see linear_equals_special_paths in the tests), which is why
the GPU kernel has only the linear rule.
"""
import numpy as np

COEF_BITS = 11
COEF_SCALE = 1 << COEF_BITS          # INTER_RESIZE_COEF_SCALE
MAX_SIDE = 65500


def axis_coords(src, dst):
    """hal::resize's per-axis loop (non-area mode): scale = 1 / inv_scale with inv_scale = dst / src (cv::resize computes
    inv_scale_x = (double)dsize.width / ssize.width); f = (float)((d + 0.5) * scale - 0.5) with the product and the difference
    rounded in double; s = cvFloor(f); f -= s.  -> s int64 [dst], f float32 [dst]"""
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    return s.astype(np.int64), (f - s).astype(np.float32)


def fixed_weights(f):
    """ialpha / ibeta: saturate_cast<short>(cbuf[k] * INTER_RESIZE_COEF_SCALE) for cbuf = {1 - f, f} in float32; cvRound
    rounds half to even.  -> (w0, w1) int64"""
    f = np.asarray(f, np.float32)
    w0 = np.rint((np.float32(1) - f) * np.float32(COEF_SCALE))
    w1 = np.rint(f * np.float32(COEF_SCALE))
    return np.clip(w0, -32768, 32767).astype(np.int64), np.clip(w1, -32768, 32767).astype(np.int64)


def column_taps(W, dst_w):
    """hal::resize's x loop with its border clamps: sx < ksize2 - 1 (= 0) gives fx = 0, sx = 0; sx + ksize2 >= W gives
    fx = 0, sx = W - 1 (and xmax, from which HResizeLinear writes S[sx] * ONE, the same value as weights 2048 / 0).
    -> (sx, sx1, a0, a1): the two source columns and their weights"""
    sx, fx = axis_coords(W, dst_w)
    left = sx < 0
    sx, fx = np.where(left, 0, sx), np.where(left, np.float32(0), fx).astype(np.float32)
    right = sx >= W - 1
    sx, fx = np.where(right, W - 1, sx), np.where(right, np.float32(0), fx).astype(np.float32)
    a0, a1 = fixed_weights(fx)
    return sx, np.minimum(sx + 1, W - 1), a0, a1


def row_taps(H, dst_h):
    """hal::resize's y loop keeps sy and fy as computed (no clamp of the weights); resizeGeneric_'s invoker clips each row
    tap with clip(sy + k, 0, H), so above row 0 and below row H - 1 both taps read the same row with the unclamped weights.
    -> (sy0, sy1, b0, b1)"""
    sy, fy = axis_coords(H, dst_h)
    b0, b1 = fixed_weights(fy)
    return np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1), b0, b1


def horizontal(img, sx, sx1, a0, a1):
    """HResizeLinear<uchar, int, short, 2048>: D[dx] = S[sx] * a0 + S[sx + cn] * a1 in int32 (HResizeLinearVec_8u32s computes
    the same products).  img uint8 [..., H, W, C] -> int64 [..., H, dst_w, C]"""
    return img[..., sx, :].astype(np.int64) * a0[:, None] + img[..., sx1, :].astype(np.int64) * a1[:, None]


def vertical(h0, h1, b0, b1):
    """VResizeLinearVec_32s8u: v_pack(S >> 4) to int16, v_mul_hi by the int16 beta ((x * b) >> 16), the two products added,
    v_rshr_pack_u<2> ((v + 2) >> 2 saturated to uint8).  cv2 4.13 applies it to every element of a 3-channel uint8 row; the
    scalar FixedPtCast rule (h0 b0 + h1 b1 + 2^21) >> 22 of VResizeLinear's tail is not reached there."""
    p0 = np.clip(h0 >> 4, -32768, 32767)
    p1 = np.clip(h1 >> 4, -32768, 32767)
    v = ((p0 * b0) >> 16) + ((p1 * b1) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def linear(img, dst_w, dst_h):
    """resizeGeneric_ with the linear tables: uint8 [..., H, W, C] -> uint8 [..., dst_h, dst_w, C] (each frame alone)"""
    H, W = img.shape[-3:-1]
    h = horizontal(img, *column_taps(W, dst_w))
    sy0, sy1, b0, b1 = row_taps(H, dst_h)
    return vertical(h[..., sy0, :, :], h[..., sy1, :, :], b0[:, None, None], b1[:, None, None])


def is_area_fast_2x(H, W, dst_h, dst_w):
    """hal::resize: is_area_fast (scale_x, scale_y integers to DBL_EPSILON) with iscale_x == iscale_y == 2 turns
    INTER_LINEAR into INTER_AREA"""
    sx, sy = 1.0 / (dst_w / W), 1.0 / (dst_h / H)
    return abs(sx - 2) < np.finfo(np.float64).eps and abs(sy - 2) < np.finfo(np.float64).eps


def area_fast_2x(img, dst_w, dst_h):
    """resizeAreaFast_ with ResizeAreaFastVec (fast_mode: scale 2 x 2, cn 1 / 3 / 4): (a + b + c + d + 2) >> 2 per channel
    over the block's 2 x 2 source pixels"""
    x = img[..., :2 * dst_h, :2 * dst_w, :].astype(np.int64)
    s = x[..., 0::2, 0::2, :] + x[..., 0::2, 1::2, :] + x[..., 1::2, 0::2, :] + x[..., 1::2, 1::2, :]
    return ((s + 2) >> 2).astype(np.uint8)


def check_args(img, dst_w, dst_h):
    if img.dtype != np.uint8 or img.ndim not in (3, 4):
        raise ValueError("frames must be uint8 [H, W, C] or [n, H, W, C]")
    for n in (img.shape[-3], img.shape[-2], dst_w, dst_h):
        if not 1 <= n <= MAX_SIDE:
            raise ValueError("height and width must be 1 .. %d" % MAX_SIDE)


def resize(img, dst_w, dst_h):
    """cv2.resize(img, (dst_w, dst_h), interpolation=cv2.INTER_LINEAR) for uint8 [H, W, C] (or each frame of [n, H, W, C]):
    the path OpenCV takes"""
    img = np.asarray(img)
    check_args(img, dst_w, dst_h)
    H, W = img.shape[-3:-1]
    if (H, W) == (dst_h, dst_w):
        return img.copy()
    if is_area_fast_2x(H, W, dst_h, dst_w):
        return area_fast_2x(img, dst_w, dst_h)
    return linear(img, dst_w, dst_h)


def resize_videos(videos, dst_w, dst_h):
    """a list of uint8 [n_v, H_v, W_v, 3] -> uint8 [sum n_v, dst_h, dst_w, 3], what ssnb_frame_resize writes"""
    return np.concatenate([resize(np.asarray(v), dst_w, dst_h) for v in videos])
