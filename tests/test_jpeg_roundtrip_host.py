"""The JPEG round trip without a GPU: an oracle composed from the encoder's and the decoder's numpy restatements
(oracle/jpeg_encode_oracle.py up to the quantised blocks, oracle/jpeg_oracle.py from them on), bitwise against Pillow's
save -> open -> convert on every size, content and quality of the grid; the library's refusals, which launch nothing; and
the header's declaration against the ctypes binding."""
import ctypes as C
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import jpeg_encode_oracle as E
from oracle import jpeg_oracle as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (height, width): 1 x 1 up to the frames of the extraction step, sides that are and are not multiples of 8 and 16
SIZES = [(1, 1), (9, 7), (8, 8), (17, 15), (16, 16), (15, 17), (256, 340), (256, 341), (360, 480)]
KINDS = ["ramp", "noise", "const128", "checker"]          # smooth, noise, constant, saturated (0 / 255)
QUALITIES = [1, 50, 75, 95, 100]


def roundtrip(img, mode="RGB", quality=95):
    """uint8 [H, W, C] -> the decoder's uint8 [H, W, C] for the encoder's file of img: the encoder's component planes (edge
    expansion, colour conversion, h2v2 downsampling), islow FDCT and quantisation, then the decoder's islow IDCT (with the
    dequantisation), fancy upsampling and colour conversion.  The Huffman coding in between is lossless and skipped."""
    img = np.asarray(img, np.uint8)
    if mode == "L" and img.ndim == 3:
        img = img[..., 0]
    H, W = img.shape[:2]
    E.check_args(mode, quality, H, W)
    q = E.quant_tables(quality)
    _, _, grid = E.geometry(mode, H, W)
    planes = []
    for c, (p, (bw, bh)) in enumerate(zip(E.component_planes(img, mode), grid)):
        blocks = p.reshape(bh, 8, bw, 8).swapaxes(1, 2).reshape(-1, 8, 8)
        coef = E.quantize(E.fdct_islow(blocks), q[min(c, 1)]).reshape(bh, bw, 64)
        planes.append(J.idct(coef, q[min(c, 1)]).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    comps = [(1, 1, 1)] if mode == "L" else [(1, 2, 2), (2, 1, 1), (3, 1, 1)]
    hdr = dict(width=W, height=H, comps=comps, colour="gray" if mode == "L" else "ycc")
    return J.colour(planes, hdr, mode)


def pillow_roundtrip(img, mode, quality):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(img[..., 0] if mode == "L" else img, mode).save(f, format="JPEG", quality=quality)
    f.seek(0)
    return np.asarray(Image.open(f).convert(mode)).reshape(img.shape)


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_oracle_equals_pillow(mode, size):
    h, w = size
    for k, kind in enumerate(KINDS):
        img = E.fixture(kind, h, w, E.MODES[mode], seed=h * 131 + w + k)
        for q in QUALITIES:
            got = roundtrip(img, mode, q)
            assert got.dtype == np.uint8 and got.shape == img.shape
            assert got.tobytes() == pillow_roundtrip(img, mode, q).tobytes(), (mode, kind, size, q)


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_oracle_equals_the_two_oracles_through_the_file(mode):
    for h, w in SIZES[:6] + [(33, 47)]:
        img = E.fixture("noise", h, w, E.MODES[mode], seed=h + w)
        for q in (5, 95):
            assert roundtrip(img, mode, q).tobytes() == J.decode(E.encode(img, mode, q), mode).tobytes(), (mode, h, w, q)


def _lib():
    from ssn_b200 import _lib
    return _lib


def test_refusals_return_before_any_launch():
    L = _lib()
    lib = L.lib
    n0 = lib.ssnb_global_launch_count()
    src, out = C.c_void_p(1 << 20), C.c_void_p(1 << 30)     # non-null pointers that are never dereferenced

    def call(mode=3, quality=95, sizes=((16, 24), (9, 7)), src_bytes=10 ** 6, out_bytes=10 ** 6, offset=None, ptrs=(src, out), n=None,
             images=True):
        arr = (L.JpegEncodeImage * max(len(sizes), 1))()
        off = 0
        for e, (h, w) in zip(arr, sizes):
            e.src_offset, e.height, e.width = off if offset is None else offset, h, w
            off += h * w * mode
        rc = lib.ssnb_jpeg_roundtrip(mode, quality, ptrs[0], src_bytes, arr if images else None, src, len(sizes) if n is None else n,
                                     ptrs[1], out_bytes, None)
        return rc, (lib.ssnb_last_error(None) or b"").decode()

    for kw, why in ((dict(mode=2), "mode"), (dict(mode=0), "mode"), (dict(quality=0), "quality"), (dict(quality=101), "quality"),
                    (dict(sizes=((0, 8),)), "height and width"), (dict(sizes=((8, 65501),)), "height and width"),
                    (dict(sizes=()), "no image"), (dict(n=0), "no image"), (dict(images=False), "NULL images"),
                    (dict(src_bytes=16 * 24 * 3), "outside src"), (dict(offset=-1), "outside src"),
                    (dict(out_bytes=16 * 24 * 3 + 9 * 7 * 3 - 1), "outside out"), (dict(ptrs=(None, out)), "NULL src"),
                    (dict(ptrs=(src, None)), "NULL src"), (dict(ptrs=(src, C.c_void_p((1 << 20) + 100))), "overlaps"),
                    (dict(ptrs=(src, C.c_void_p((1 << 20) - 10 ** 6 + 1))), "overlaps")):
        rc, msg = call(**kw)
        assert rc == 1, (kw, msg)
        assert msg.startswith("jpeg_roundtrip: ") and why in msg, (kw, msg)
    assert lib.ssnb_global_launch_count() == n0


def test_python_refusals():
    import torch
    from ops.jpeg import jpeg_roundtrip, JpegRoundtripPlan
    from ops.optical_flow import flow_images, frame_images
    with pytest.raises(RuntimeError):
        jpeg_roundtrip(torch.zeros(2, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        jpeg_roundtrip([torch.zeros(8, 8, 1, dtype=torch.uint8)], mode="L")
    with pytest.raises(RuntimeError):
        flow_images(torch.zeros(2, 8, 8, 1, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        frame_images(torch.zeros(2, 8, 8, 3, dtype=torch.uint8))
    assert jpeg_roundtrip([]) == []
    with pytest.raises(ValueError, match="mode"):
        JpegRoundtripPlan([(8, 8)], mode="CMYK")
    for q in (0, 101):
        with pytest.raises(ValueError, match="quality"):
            JpegRoundtripPlan([(8, 8)], quality=q)
    for hw in ((0, 8), (8, 65501)):
        with pytest.raises(ValueError, match="height and width"):
            JpegRoundtripPlan([hw], mode="L")
    with pytest.raises(ValueError, match="no image"):
        JpegRoundtripPlan([])


def _c_kind(decl):
    """a parameter's C declaration -> the ctypes class it must be bound with"""
    decl = decl.strip()
    if "*" in decl:
        return "pointer"
    return {"int": C.c_int, "int64_t": C.c_int64, "size_t": C.c_size_t}[decl.rsplit(None, 1)[0]]


def test_header_declaration_matches_the_binding(tmp_path):
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    decl = re.search(r"\bint ssnb_jpeg_roundtrip\(([^)]*)\);", hdr).group(1)
    params = [p for p in decl.split(",")]
    res, args = L.SIGNATURES["ssnb_jpeg_roundtrip"]
    assert res is C.c_int and len(params) == len(args) == 10
    for p, a in zip(params, args):
        k = _c_kind(p)
        if k == "pointer":
            assert a is C.c_void_p or a.__name__.startswith("LP_"), (p, a)
        else:
            assert a is k, (p, a)
    assert args[4]._type_ is L.JpegEncodeImage
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    # the prototype the binding assumes, checked against the header's by the C compiler
    src = tmp_path / "abi.c"
    src.write_text('#include <stddef.h>\n#include "ssnb.h"\n'
                   'int (*f)(int, int, const uint8_t*, int64_t, const ssnb_jpeg_encode_image*, const ssnb_jpeg_encode_image*, int, '
                   'uint8_t*, int64_t, void*) = ssnb_jpeg_roundtrip;\n'
                   'int main(void) { return f == 0; }\n')
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-c", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "abi.o")],
                   check=True)
