"""Write tests/golden/frame_resize.npz: cv2.resize(img, (dst_w, dst_h), interpolation=cv2.INTER_LINEAR) of every fixture of
FIXTURES (cv2 4.13), after checking that oracle/frame_resize_oracle.py computes the same bytes.

Sources are the frame sizes of the data sets (THUMOS14's 320 x 240, ActivityNet's YouTube sizes), the identity, exact 2x
and 3x downscales and degenerate 1-pixel sides, each resized to DenseFlow's 340 x 256; a sweep of destination widths
1 .. 40 crosses every block boundary of OpenCV's vector passes.  Contents: noise, constant 0 and 255, a ramp and a 0 / 255
checkerboard (saturation).  The inputs are not stored: jpeg_encode_oracle.fixture(kind, H, W, 3, seed) regenerates them
without numpy's random generators, and each fixture keeps the CRC-32 of its input so a drift of the generator is caught.
Per fixture NAME:
  out_NAME   uint8 [dst_h, dst_w, 3]  cv2's output, kept for every fixture but the 340 x 256 noise ones other than
                                      THUMOS14's 320 x 240 and the 1280 x 720 source (noise does not compress: the ten
                                      others would add 2.3 MB)
  ocrc_NAME  int64                    zlib.crc32 of cv2's output, every fixture
  crc_NAME   int64                    zlib.crc32 of the input frame
and `names`, `specs` (kind, H, W, seed, dst_h, dst_w per row) index them.

    python -m oracle.gen_golden_frame_resize
"""
import os
import zlib

import numpy as np

from oracle import frame_resize_oracle as R
from oracle.jpeg_encode_oracle import fixture

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "frame_resize.npz")

# (H, W) of the sources resized to 340 x 256: 1 x 1, 1 x N, N x 1, upscales, the identity, downscales (exact 2x and 3x)
SOURCES = [(1, 1), (1, 300), (300, 1), (100, 77), (240, 320), (256, 340), (360, 480), (360, 640), (512, 680), (768, 1020),
           (480, 854), (720, 1280)]
KINDS = ["noise", "const0", "const255", "ramp", "checker"]
DST = (256, 340)
SWEEP_SOURCES = [(240, 320), (3, 5)]           # a downscale and an upscale for every destination width 1 .. 40
SWEEP_HEIGHT = 7
NOISE_KEPT = [(240, 320), (720, 1280)]        # the 340 x 256 noise fixtures whose outputs are stored in full


def fixtures():
    """(kind, H, W, seed, dst_h, dst_w) of every fixture"""
    out = []
    for h, w in SOURCES:
        for k, kind in enumerate(KINDS):
            out.append((kind, h, w, h * 131 + w + k, DST[0], DST[1]))
    for h, w in SWEEP_SOURCES:
        for dw in range(1, 41):
            out.append(("noise", h, w, 1000 + dw, SWEEP_HEIGHT, dw))
    return out


def name(kind, h, w, seed, dh, dw):
    return "%dx%d_%s_s%d_to_%dx%d" % (h, w, kind, seed, dh, dw)


def image(kind, h, w, seed):
    return fixture(kind, h, w, 3, seed)


def golden(cv2):
    """-> the arrays of the golden file, each fixture's cv2 output asserted equal to the oracle's"""
    out, names, specs = {}, [], []
    for spec in fixtures():
        kind, h, w, seed, dh, dw = spec
        img = image(kind, h, w, seed)
        ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        n = name(*spec)
        assert R.resize(img, dw, dh).tobytes() == ref.tobytes(), ("oracle vs cv2.resize", n)
        if kind != "noise" or (dh, dw) != DST or (h, w) in NOISE_KEPT:
            out["out_" + n] = ref
        out["ocrc_" + n] = np.int64(zlib.crc32(ref.tobytes()))
        out["crc_" + n] = np.int64(zlib.crc32(img.tobytes()))
        names.append(n)
        specs.append(spec)
    out["names"] = np.array(names)
    out["specs"] = np.array([[str(v) for v in s] for s in specs])
    return out


def main():
    import cv2
    out = golden(cv2)
    np.savez_compressed(OUT, **out)
    print("wrote %s: %d fixtures, cv2 %s, oracle identical" % (OUT, len(out["names"]), cv2.__version__))


if __name__ == "__main__":
    main()
