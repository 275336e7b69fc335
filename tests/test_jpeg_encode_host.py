"""JPEG encode without a GPU: the numpy oracle (oracle/jpeg_encode_oracle.py) against Pillow's bytes of every golden fixture
(tests/golden/jpeg_encode.npz, oracle/gen_golden_jpeg_encode.py), the library's refusals and capacities, the header's image
struct against the ctypes mirror, and write_frame_jpegs' layout from host frames."""
import ctypes as C
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from oracle import jpeg_encode_oracle as E
from oracle.gen_golden_jpeg_encode import image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode.npz"))
SPECS = [(m, k, int(h), int(w), int(s), int(q)) for m, k, h, w, s, q in GOLD["specs"]]


@pytest.mark.parametrize("i", range(len(SPECS)))
def test_oracle_equals_pillow_bytes(i):
    mode, kind, h, w, seed, q = SPECS[i]
    name = str(GOLD["names"][i])
    img = image(mode, kind, h, w, seed)
    assert zlib.crc32(img.tobytes()) == int(GOLD["crc_" + name]), "fixture generator drifted: " + name
    assert E.encode(img, mode, q) == GOLD["jpg_" + name].tobytes(), name


def test_fixtures_cover_the_sizes_contents_and_qualities():
    got = {(m, h, w) for m, _, h, w, _, _ in SPECS}
    for mode in ("L", "RGB"):
        for hw in [(1, 1), (1, 17), (7, 9), (8, 8), (9, 16), (15, 17), (16, 16), (17, 31), (256, 340), (256, 341), (340, 256),
                   (360, 480), (1, 2000)]:
            assert (mode,) + hw in got
    assert {k for _, k, *_ in SPECS} == {"const0", "const128", "const255", "ramp", "noise", "checker", "flow"}
    assert {q for *_, q in SPECS} == {1, 5, 25, 50, 75, 90, 95, 100}
    # noise fixtures stuff many 0xFF bytes; the checkerboard reaches the largest coefficients
    b = GOLD["jpg_" + str(GOLD["names"][SPECS.index(("RGB", "noise", 256, 340, 7, 95))])].tobytes()
    assert b.count(b"\xff\x00") > 200


def test_quant_tables_and_header():
    lum, chrom = E.quant_tables(50)
    assert (lum == E.STD_QUANT[0]).all() and (chrom == E.STD_QUANT[1]).all()
    assert (E.quant_tables(100)[0] == 1).all() and E.quant_tables(1)[0].max() == 255
    assert E.header_bytes("L") == 328 and E.header_bytes("RGB") == 623


def _lib():
    from ssn_b200 import _lib
    return _lib


@pytest.mark.parametrize("mode,code", [("L", 1), ("RGB", 3)])
def test_capacity_matches_the_oracle_and_bounds_the_golden_files(mode, code):
    lib = _lib().lib
    for i, (m, _, h, w, _, _) in enumerate(SPECS):
        if m == mode:
            cap = lib.ssnb_jpeg_encode_capacity(code, h, w)
            assert cap == E.capacity(mode, h, w)
            assert GOLD["jpg_" + str(GOLD["names"][i])].size <= cap
    assert lib.ssnb_jpeg_encode_capacity(code, 65500, 65500) == E.capacity(mode, 65500, 65500)
    for h, w in ((0, 8), (8, 0), (65501, 8), (8, 65501)):
        assert lib.ssnb_jpeg_encode_capacity(code, h, w) == 0
    assert lib.ssnb_jpeg_encode_capacity(2, 8, 8) == 0


def test_refusals_return_before_any_launch():
    L = _lib()
    lib = L.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(256)                    # a non-null, aligned pointer that is never dereferenced

    def table(*sizes, src=None):
        arr = (L.JpegEncodeImage * len(sizes))()
        off = 0
        for e, (h, w) in zip(arr, sizes):
            e.src_offset, e.height, e.width = off if src is None else src, h, w
            off += h * w * 3
        return arr

    def call(mode=3, quality=95, sizes=((16, 24), (9, 7)), src_bytes=10 ** 6, out_bytes=None, ws_bytes=None, src=None, ptr=one, n=None):
        imgs = table(*sizes, src=src)
        ws, ob = C.c_size_t(), C.c_int64()
        rc = lib.ssnb_jpeg_encode_sizes(mode, quality, imgs, len(sizes), C.byref(ws), C.byref(ob))
        if rc == 0:
            assert ob.value == sum(E.capacity("RGB" if mode == 3 else "L", h, w) for h, w in sizes)
        rc2 = lib.ssnb_jpeg_encode(mode, quality, ptr, src_bytes, imgs, one, len(sizes) if n is None else n, one,
                                   ob.value if out_bytes is None else out_bytes, one, one, ws.value if ws_bytes is None else ws_bytes, None)
        return rc, rc2, ws.value, ob.value

    rc, _, ws, ob = call(ptr=None)
    assert rc == 0 and ws > 0 and ob > 0
    for kw, why in ((dict(mode=2), "mode 2"), (dict(mode=0), "mode 0"), (dict(quality=0), "quality 0"), (dict(quality=101), "quality 101"),
                    (dict(sizes=((0, 8),)), "height 0"), (dict(sizes=((8, 65501),)), "width 65501"), (dict(sizes=()), "no image")):
        rc, rc2, _, _ = call(**kw)
        assert rc == 1 and rc2 == 1, why
        assert b"jpeg_encode" in lib.ssnb_last_error(None)
    assert call(src_bytes=16 * 24 * 3)[1] == 1                       # the second image lies outside src
    assert call(src=-1)[1] == 1
    assert call(out_bytes=ob - 1)[1] == 1
    assert call(ws_bytes=ws - 1)[1] == 1
    assert call(ptr=None)[1] == 1                                     # NULL src
    assert b"src" in lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0


def test_python_refusals():
    import torch
    from ops.jpeg import encode_jpeg, JpegEncodePlan
    with pytest.raises(RuntimeError):
        encode_jpeg(torch.zeros(2, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        encode_jpeg([torch.zeros(8, 8, 1, dtype=torch.uint8)], mode="L")
    with pytest.raises(ValueError):
        JpegEncodePlan([(8, 8)], mode="CMYK")
    with pytest.raises(ValueError, match="quality"):
        JpegEncodePlan([(8, 8)], quality=0)
    with pytest.raises(ValueError, match="height and width"):
        JpegEncodePlan([(8, 65501)], mode="L")
    for args in (("CMYK", 95, 8, 8), ("L", 101, 8, 8), ("RGB", 95, 0, 8), ("RGB", 95, 8, 65501)):
        with pytest.raises(ValueError):
            E.check_args(*args)


def test_write_frame_jpegs_layout(tmp_path):
    from PIL import Image
    from ops.optical_flow import write_frame_jpegs
    frames = E.fixture("noise", 12, 16, 3, 0)[None].repeat(5, 0)
    frames[:, 0, 0, 0] = np.arange(5, dtype=np.uint8) * 40
    paths = write_frame_jpegs(frames, [str(tmp_path / "a"), str(tmp_path / "b")], offsets=[0, 3, 5])
    assert [os.path.relpath(p, tmp_path) for p in paths] == ["a/img_00001.jpg", "a/img_00002.jpg", "a/img_00003.jpg", "b/img_00001.jpg",
                                                             "b/img_00002.jpg"]
    for i, p in enumerate(paths):
        assert open(p, "rb").read() == E.encode(frames[i], "RGB", 95)
    im = Image.open(paths[4])
    assert im.mode == "RGB" and im.size == (16, 12)
    one = write_frame_jpegs(frames[:2], str(tmp_path / "c"), prefix="rgb_", quality=50)
    assert [os.path.basename(p) for p in one] == ["rgb_00001.jpg", "rgb_00002.jpg"]
    assert open(one[1], "rb").read() == E.encode(frames[1], "RGB", 50)
    for bad in (dict(offsets=[0, 3, 5]), dict(offsets=[0, 2])):
        with pytest.raises(ValueError):
            write_frame_jpegs(frames, [str(tmp_path / "d")], **bad)
    with pytest.raises(ValueError):
        write_frame_jpegs(frames[..., :1], str(tmp_path / "e"))


def test_header_mirror_of_the_encode_image(tmp_path):
    L = _lib()
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct \{([^{}]*)\}\s*ssnb_jpeg_encode_image;", hdr).group(1), flags=re.S)
    names = []
    for d in body.split(";"):
        if d.strip():
            names += [n.strip() for n in d.split(None, 1)[1].split(",")]
    assert names == [n for n, _ in L.JpegEncodeImage._fields_]
    prints = ['printf("size %zu\\n", sizeof(ssnb_jpeg_encode_image));']
    prints += ['printf("%s %%zu\\n", offsetof(ssnb_jpeg_encode_image, %s));' % (n, n) for n in names]
    prints += ['printf("L %d\\n", SSNB_JPEG_ENC_L);', 'printf("RGB %d\\n", SSNB_JPEG_ENC_RGB);']
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "abi")], check=True)
    lay = dict(l.split() for l in subprocess.run([str(tmp_path / "abi")], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(lay["size"]) == C.sizeof(L.JpegEncodeImage)
    for n, _ in L.JpegEncodeImage._fields_:
        assert int(lay[n]) == getattr(L.JpegEncodeImage, n).offset
    assert (int(lay["L"]), int(lay["RGB"])) == (L.JPEG_ENC_L, L.JPEG_ENC_RGB)
    for name, n_args in (("ssnb_jpeg_encode", 13), ("ssnb_jpeg_encode_sizes", 6), ("ssnb_jpeg_encode_capacity", 3)):
        decl = re.search(r"\b%s\(([^)]*)\);" % name, hdr).group(1)
        assert len(decl.split(",")) == n_args == len(L.SIGNATURES[name][1]), name
