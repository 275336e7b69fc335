"""Write tests/golden/jpeg_encode.npz: Pillow's JPEG bytes (Image.save(quality=q) over libjpeg-turbo) of every fixture of
FIXTURES, after checking that oracle/jpeg_encode_oracle.py writes the same bytes and, where cv2 imports, that
cv2.imencode('.jpg', IMWRITE_JPEG_QUALITY=q) does too (DenseFlow writes its frames and flow planes with OpenCV).

The inputs are not stored: jpeg_encode_oracle.fixture(kind, H, W, C, seed) regenerates them without numpy's random
generators, and each fixture keeps the CRC-32 of its input so a drift of the generator is caught.  Per fixture NAME:
  jpg_NAME  uint8 [bytes]  the file
  crc_NAME  int64          zlib.crc32 of the input image
and `names`, `specs` (mode, kind, H, W, seed, quality per row) index them.

    python -m oracle.gen_golden_jpeg_encode
"""
import io
import os
import zlib

import numpy as np

from oracle import jpeg_encode_oracle as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg_encode.npz")

SMALL = [(1, 1), (1, 17), (7, 9), (8, 8), (9, 16), (15, 17), (16, 16), (17, 31)]
LARGE = [(256, 340), (256, 341), (340, 256), (360, 480)]
KINDS = ["const0", "const128", "const255", "ramp", "noise", "checker", "flow"]
QUALITIES = [1, 5, 25, 50, 75, 90, 95, 100]


def fixtures():
    """(mode, kind, H, W, seed, quality) of every fixture"""
    out = []
    for mode in ("L", "RGB"):
        for h, w in SMALL:
            for k in KINDS:
                out.append((mode, k, h, w, h * 131 + w, 95))
        for h, w in LARGE:
            for k in ("ramp", "flow", "checker"):
                out.append((mode, k, h, w, h + w, 95))
        out.append((mode, "noise", 256, 340, 7, 95))
        out.append((mode, "noise", 360, 480, 8, 90))
        out.append((mode, "noise", 1, 2000, 9, 95))
        out.append((mode, "flow", 1, 2000, 9, 95))
        for q in QUALITIES:
            out.append((mode, "noise", 17, 31, 100 + q, q))
            out.append((mode, "checker", 16, 16, 0, q))
            out.append((mode, "flow", 256, 341, 200 + q, q))
    return out


def name(mode, kind, h, w, seed, q):
    return "%s_%dx%d_%s_s%d_q%d" % (mode, h, w, kind, seed, q)


def image(mode, kind, h, w, seed):
    return E.fixture(kind, h, w, E.MODES[mode], seed)


def pillow(img, mode, q):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(img[..., 0] if mode == "L" else img, mode).save(f, format="JPEG", quality=q)
    return f.getvalue()


def main():
    try:
        import cv2
    except ImportError:
        cv2 = None
    out, names, specs = {}, [], []
    for mode, kind, h, w, seed, q in fixtures():
        img = image(mode, kind, h, w, seed)
        b = pillow(img, mode, q)
        n = name(mode, kind, h, w, seed, q)
        assert E.encode(img, mode, q) == b, ("oracle vs Pillow", n)
        if cv2 is not None:
            ok, enc = cv2.imencode(".jpg", img[..., 0] if mode == "L" else img[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, q])
            assert ok and enc.tobytes() == b, ("cv2.imencode vs Pillow", n)
        out["jpg_" + n] = np.frombuffer(b, np.uint8)
        out["crc_" + n] = np.int64(zlib.crc32(img.tobytes()))
        names.append(n)
        specs.append((mode, kind, h, w, seed, q))
    out["names"] = np.array(names)
    out["specs"] = np.array([[str(v) for v in s] for s in specs])
    np.savez_compressed(OUT, **out)
    print("wrote %s: %d fixtures, %d JPEG bytes%s" % (OUT, len(names), sum(out["jpg_" + n].size for n in names),
                                                      ", cv2.imencode identical" if cv2 is not None else ""))


if __name__ == "__main__":
    main()
