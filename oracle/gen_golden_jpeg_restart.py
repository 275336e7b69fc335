"""Write tests/golden/jpeg_restart.npz: Pillow's JPEG bytes with restart intervals (Image.save(quality=q,
restart_marker_blocks=n) or restart_marker_rows=r over libjpeg-turbo) of every fixture of FIXTURES, after checking that
oracle/jpeg_restart_oracle.py writes the same bytes, that cv2.imencode with IMWRITE_JPEG_RST_INTERVAL = n does too for the
blocks form, and that the set covers what the rules have to get right: an RST directly after a stuffed FF 00, RST numbering
that wraps, intervals that divide the MCUs exactly, a DRI without any RST, a rows interval clamped to 65535 that cuts an MCU
row, and RGB intervals that start in an MCU with right-edge and with bottom-edge dummy blocks.

The inputs are not stored: jpeg_encode_oracle.fixture(kind, H, W, C, seed) regenerates them, and each fixture keeps the
CRC-32 of its input.  Per fixture NAME:
  jpg_NAME  uint8 [bytes]  the file
  crc_NAME  int64          zlib.crc32 of the input image
and `names`, `specs` (mode, kind, H, W, seed, quality, restart_blocks, restart_rows per row) index them.

    python -m oracle.gen_golden_jpeg_restart
"""
import io
import os
import zlib

import numpy as np

from oracle import jpeg_encode_oracle as E
from oracle import jpeg_restart_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg_restart.npz")

SMALL = [(1, 1), (8, 8), (17, 9), (37, 23), (23, 37)]          # (H, W)
LARGE = [(256, 340), (360, 480)]
KINDS = ["noise", "const128", "ramp"]                            # random, flat, smooth
QUALITIES = [1, 50, 95, 100]
OPTIONS = [(b, 0) for b in (1, 2, 3, 7, 8, 9, 22, 65535)] + [(0, r) for r in (1, 2, 3, 9)]


def fixtures():
    """(mode, kind, H, W, seed, quality, restart_blocks, restart_rows) of every fixture"""
    out = []
    for mode in ("L", "RGB"):
        for h, w in SMALL:
            for j, (rb, rr) in enumerate(OPTIONS):
                out.append((mode, KINDS[j % 3], h, w, h * 131 + w + j, QUALITIES[j % 4], rb, rr))
        for h, w in LARGE:
            for rb, rr in ((0, 1), (0, 2), (1, 0), (22, 0)):
                out.append((mode, "flow" if mode == "L" else "ramp", h, w, h + w + rb, 95, rb, rr))
            out.append((mode, "noise", h, w, 5, 50, 0, 1))
        out.append((mode, "noise", 32, 128, 11, 95, 8, 0))       # 'RGB': 16 MCUs in 2 intervals of 8
    out.append(("RGB", "noise", 32, 128, 12, 95, 1, 0))          # 16 intervals
    out.append(("L", "noise", 8, 64, 13, 95, 1, 0))              # 8 intervals: RST0 .. RST7, no wrap yet
    out.append(("L", "noise", 8, 72, 14, 95, 1, 0))              # 9 intervals: RST7 then RST0
    out.append(("L", "const128", 16, 65500, 0, 95, 0, 9))        # 9 rows clamp to 65535 >= 16376 MCUs: DRI, no RST
    out.append(("L", "ramp", 72, 65500, 0, 95, 0, 9))            # 65535 of 73692 MCUs: the interval ends inside row 8
    for s in range(8):                                           # random q100 at one MCU per interval: FF 00 FF Dn
        out.append(("L", "noise", 16, 64, 100 + s, 100, 1, 0))
    return out


def name(mode, kind, h, w, seed, q, rb, rr):
    return "%s_%dx%d_%s_s%d_q%d_%s" % (mode, h, w, kind, seed, q, "b%d" % rb if rb else "r%d" % rr)


def image(mode, kind, h, w, seed):
    return E.fixture(kind, h, w, E.MODES[mode], seed)


def pillow(img, mode, q, rb=0, rr=0):
    from PIL import Image
    f = io.BytesIO()
    kw = {"restart_marker_blocks": rb} if rb else {"restart_marker_rows": rr} if rr else {}
    Image.fromarray(img[..., 0] if mode == "L" else img, mode).save(f, format="JPEG", quality=q, **kw)
    return f.getvalue()


def dummy_starts(h, w, rb, rr):
    """for 'RGB': do intervals start in an MCU with right-edge dummies, and in one with bottom-edge dummies?"""
    mx, my, _ = E.geometry("RGB", h, w)
    Rv = R.interval("RGB", h, w, rb, rr)
    starts = range(0, mx * my, Rv) if Rv else [0]
    right = any(m % mx == mx - 1 and 0 < w % 16 <= 8 for m in starts)
    bottom = any(m // mx == my - 1 and 0 < h % 16 <= 8 for m in starts)
    return right, bottom


def main():
    import cv2
    out, names, specs = {}, [], []
    stuffed_before_rst, wraps, exact, dri_only, right, bottom = 0, False, False, False, False, False
    for mode, kind, h, w, seed, q, rb, rr in fixtures():
        img = image(mode, kind, h, w, seed)
        b = pillow(img, mode, q, rb, rr)
        n = name(mode, kind, h, w, seed, q, rb, rr)
        assert R.encode(img, mode, q, rb, rr) == b, ("oracle vs Pillow", n)
        if rb:
            ok, enc = cv2.imencode(".jpg", img[..., 0] if mode == "L" else img[..., ::-1],
                                   [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rb])
            assert ok and enc.tobytes() == b, ("cv2.imencode vs Pillow", n)
        K = R.intervals(mode, h, w, rb, rr)
        mx, my, _ = E.geometry(mode, h, w)
        stuffed_before_rst += sum(b.count(bytes([0xFF, 0, 0xFF, 0xD0 + k])) for k in range(8))
        wraps |= K > 8
        exact |= K > 1 and (mx * my) % R.interval(mode, h, w, rb, rr) == 0
        dri_only |= K == 1 and b"\xff\xdd" in b
        if mode == "RGB":
            r_, b_ = dummy_starts(h, w, rb, rr)
            right, bottom = right or r_, bottom or b_
        out["jpg_" + n] = np.frombuffer(b, np.uint8)
        out["crc_" + n] = np.int64(zlib.crc32(img.tobytes()))
        names.append(n)
        specs.append((mode, kind, h, w, seed, q, rb, rr))
    assert stuffed_before_rst > 0, "no RST directly after a stuffed FF 00"
    assert wraps and exact and dri_only and right and bottom, (wraps, exact, dri_only, right, bottom)
    out["names"] = np.array(names)
    out["specs"] = np.array([[str(v) for v in s] for s in specs])
    np.savez_compressed(OUT, **out)
    print("wrote %s: %d fixtures, %d JPEG bytes, %d RSTs after a stuffed FF 00, oracle and cv2.imencode identical"
          % (OUT, len(names), sum(out["jpg_" + n].size for n in names), stuffed_before_rst))


if __name__ == "__main__":
    main()
