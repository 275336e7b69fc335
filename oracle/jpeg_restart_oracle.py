"""Restart intervals in the baseline JPEG encode: what Image.save(f, quality=q, restart_marker_blocks=n) and
Image.save(f, quality=q, restart_marker_rows=r) write through libjpeg-turbo (cv2.imencode with IMWRITE_JPEG_RST_INTERVAL = n
writes the blocks form byte for byte).  Every stage before the entropy coding is oracle/jpeg_encode_oracle.py's, unchanged:
restart markers change only the layout of the entropy-coded data, never a quantised coefficient.  The rules, with the
libjpeg-turbo function each follows:

  interval()   jcmaster.c per_scan_setup: restart_interval = n MCUs (blocks), or MIN(r * MCUs_per_row, 65535) (rows),
               computed per image from its own width.  0 for both: no interval (the file encode_jpeg_oracle.encode writes).
  header()     jcmarker.c write_scan_header: a DRI segment (FF DD 00 04, the interval big-endian) after the last DHT and
               before SOS whenever the interval is non-zero, even when it covers the whole image and no RST follows.
  entropy()    jchuff.c encode_mcu_huff / emit_restart / flush_bits: interval k holds MCUs [kR, min((k + 1) R, mcus)).
               Before every interval but the first the previous one is padded to a byte with 1-bits (the pad byte is
               stuffed like any other), FF D0 + ((k - 1) mod 8) is written unstuffed, and every DC predictor is reset to 0.
               Dummy blocks keep their rule (DC of the block before, so a difference of 0); an interval starts at an MCU's
               first luma block, which is never a dummy.
  capacity()   the worst-case file: jpeg_encode_oracle.capacity's header, blocks and EOI, the DRI, at most 7 pad bits per
               interval, every entropy byte stuffed, 2 marker bytes per interval but the first.

tests/golden/jpeg_restart.npz (oracle/gen_golden_jpeg_restart.py) pins it to Pillow's bytes.
"""
from oracle import jpeg_encode_oracle as E

MAX_INTERVAL = 65535                # the DRI field is 16 bits; jcmaster.c clamps restart_in_rows * MCUs_per_row to it


def check_restart(restart_blocks, restart_rows):
    """the library's refusals, in its wording"""
    if restart_blocks < 0 or restart_rows < 0:
        raise ValueError("restart_blocks and restart_rows must be >= 0")
    if restart_blocks and restart_rows:
        raise ValueError("restart_blocks and restart_rows cannot both be set")
    if restart_blocks > MAX_INTERVAL:
        raise ValueError("restart_blocks must be <= %d" % MAX_INTERVAL)


def interval(mode, height, width, restart_blocks=0, restart_rows=0):
    """jcmaster.c per_scan_setup: MCUs per restart interval of this image, 0 for none"""
    check_restart(restart_blocks, restart_rows)
    if restart_blocks:
        return restart_blocks
    if restart_rows:
        mx, _, _ = E.geometry(mode, height, width)
        return min(restart_rows * mx, MAX_INTERVAL)
    return 0


def intervals(mode, height, width, restart_blocks=0, restart_rows=0):
    """the number of restart intervals of the scan: ceil(MCUs / R), 1 without an interval"""
    R = interval(mode, height, width, restart_blocks, restart_rows)
    mx, my, _ = E.geometry(mode, height, width)
    return -(-(mx * my) // R) if R else 1


def header(mode, quality, height, width, R):
    """jpeg_encode_oracle.header with jcmarker.c emit_dri's segment before SOS when R > 0"""
    h = E.header(mode, quality, height, width)
    if not R:
        return h
    sos = h.rindex(b"\xff\xda")
    return h[:sos] + b"\xff\xdd\x00\x04" + R.to_bytes(2, "big") + h[sos:]


def entropy(coef, comp, bpm, R):
    """jchuff.c with restart_interval R: each interval's blocks coded with the predictors reset to 0 and padded to a byte
    (jpeg_encode_oracle.entropy of the interval's blocks), joined by RST0 .. RST7 in turn"""
    if not R:
        return E.entropy(coef, comp)
    step = R * bpm
    parts = [E.entropy(coef[s:s + step], comp[s:s + step]) for s in range(0, len(coef), step)]
    out = parts[0]
    for k, p in enumerate(parts[1:]):
        out += bytes([0xFF, 0xD0 + (k & 7)]) + p
    return out


def encode(img, mode="RGB", quality=95, restart_blocks=0, restart_rows=0):
    """uint8 [H, W] or [H, W, 1] ('L'), [H, W, 3] ('RGB') -> the JPEG file's bytes, equal to Pillow's save(quality=quality,
    restart_marker_blocks=restart_blocks) or save(quality=quality, restart_marker_rows=restart_rows)"""
    import numpy as np
    img = np.asarray(img, np.uint8)
    if mode == "L" and img.ndim == 3:
        img = img[..., 0]
    E.check_args(mode, quality, img.shape[0], img.shape[1])
    R = interval(mode, img.shape[0], img.shape[1], restart_blocks, restart_rows)
    coef, comp, _ = E.blocks(img, mode, quality)
    bpm = 6 if mode == "RGB" else 1
    return header(mode, quality, img.shape[0], img.shape[1], R) + entropy(coef, comp, bpm, R) + b"\xff\xd9"


def capacity(mode, height, width, restart_blocks=0, restart_rows=0):
    """the worst-case file size the library reserves per image.  Interval k of K carries b_k <= its blocks *
    MAX_BLOCK_BITS bits and is padded to ceil(b_k / 8) <= (b_k + 7) / 8 bytes, so the entropy-coded bytes before stuffing
    are at most floor((blocks * MAX_BLOCK_BITS + 7 K) / 8); every one may be stuffed; then 2 bytes per RST, the DRI's 6
    and EOI.  K = 1 and no DRI give jpeg_encode_oracle.capacity."""
    R = interval(mode, height, width, restart_blocks, restart_rows)
    K = intervals(mode, height, width, restart_blocks, restart_rows)
    raw = (E.blocks_per_image(mode, height, width) * E.MAX_BLOCK_BITS + 7 * K) // 8
    return E.header_bytes(mode) + (6 if R else 0) + 2 * raw + 2 * (K - 1) + 2
