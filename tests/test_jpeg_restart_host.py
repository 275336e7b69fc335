"""JPEG encode with restart intervals, without a GPU: the numpy oracle (oracle/jpeg_restart_oracle.py) against Pillow's bytes of
every golden fixture (tests/golden/jpeg_restart.npz, oracle/gen_golden_jpeg_restart.py) and the generator re-run, the
restart-aware capacity against the oracle's bound and the golden files, the refusals, the new prototypes against their
ctypes rows, the decoded pixels with and without markers, and write_frame_jpegs / write_flow_jpegs' Pillow path with each
keyword."""
import ctypes as C
import io
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from oracle import jpeg_encode_oracle as E
from oracle import jpeg_restart_oracle as R
from oracle import gen_golden_jpeg_restart as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_restart.npz"))
SPECS = [(m, k, int(h), int(w), int(s), int(q), int(b), int(r)) for m, k, h, w, s, q, b, r in GOLD["specs"]]
CODE = {"L": 1, "RGB": 3}


def _gold(i):
    return GOLD["jpg_" + str(GOLD["names"][i])].tobytes()


@pytest.mark.parametrize("i", range(len(SPECS)))
def test_oracle_equals_pillow_bytes(i):
    mode, kind, h, w, seed, q, rb, rr = SPECS[i]
    name = str(GOLD["names"][i])
    img = G.image(mode, kind, h, w, seed)
    assert zlib.crc32(img.tobytes()) == int(GOLD["crc_" + name]), "fixture generator drifted: " + name
    assert R.encode(img, mode, q, rb, rr) == _gold(i), name


def test_generator_reproduces_the_golden_file(tmp_path, monkeypatch):
    pytest.importorskip("cv2")
    pytest.importorskip("PIL")
    out = tmp_path / "jpeg_restart.npz"
    monkeypatch.setattr(G, "OUT", str(out))
    G.main()
    new = np.load(out)
    assert sorted(new.files) == sorted(GOLD.files)
    for k in GOLD.files:
        assert np.array_equal(new[k], GOLD[k]), k


def test_fixtures_cover_the_rules():
    assert {(m, h, w) for m, _, h, w, *_ in SPECS} >= {(m, h, w) for m in ("L", "RGB") for h, w in G.SMALL + G.LARGE}
    assert ("L", 16, 65500) in {(m, h, w) for m, _, h, w, *_ in SPECS}
    assert {q for *_, q, _, _ in SPECS} == {1, 50, 95, 100}
    assert {b for *_, b, _ in SPECS} >= {1, 2, 3, 7, 8, 9, 22, 65535} and {r for *_, r in SPECS} >= {1, 2, 3, 9}
    assert {k for _, k, *_ in SPECS} >= {"noise", "const128", "ramp"}
    counts = {R.intervals(m, h, w, b, r) for m, _, h, w, _, _, b, r in SPECS}
    assert {1, 8, 9, 16} <= counts
    # the 72 x 65500 plane: rows 9 clamps to 65535 MCUs, which ends inside MCU row 8 of 8188 MCUs each
    assert R.interval("L", 72, 65500, 0, 9) == 65535 and 65535 % 8188 and R.intervals("L", 72, 65500, 0, 9) == 2
    stuffed = sum(_gold(i).count(bytes([0xFF, 0, 0xFF, 0xD0 + k])) for i in range(len(SPECS)) for k in range(8))
    assert stuffed > 0


def test_markers_and_dri_are_where_libjpeg_puts_them():
    for i, (mode, _, h, w, _, q, rb, rr) in enumerate(SPECS):
        b = _gold(i)
        Rv, K = R.interval(mode, h, w, rb, rr), R.intervals(mode, h, w, rb, rr)
        sos = b.rindex(b"\xff\xda")
        assert b[sos - 6:sos] == b"\xff\xdd\x00\x04" + Rv.to_bytes(2, "big")
        scan = b[sos + 2 + int.from_bytes(b[sos + 2:sos + 4], "big"):-2]
        rst = [m.group(0)[1] for m in re.finditer(rb"\xff[\xd0-\xd7]", scan)]
        assert rst == [0xD0 + (k & 7) for k in range(K - 1)]


def test_decoded_pixels_do_not_change():
    """the markers change only the entropy-coded layout: Pillow decodes every golden file to the pixels of the same image
    saved without markers, which is what jpeg_roundtrip, frame_images and flow_images compute"""
    from PIL import Image
    for i, (mode, kind, h, w, seed, q, rb, rr) in enumerate(SPECS):
        img = G.image(mode, kind, h, w, seed)
        plain = np.asarray(Image.open(io.BytesIO(G.pillow(img, mode, q))).convert(mode))
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(_gold(i))).convert(mode)), plain), str(GOLD["names"][i])


def _lib():
    from ssn_b200 import _lib
    return _lib


def test_capacity_matches_the_oracle_and_bounds_the_golden_files():
    lib = _lib().lib
    for i, (m, _, h, w, _, _, rb, rr) in enumerate(SPECS):
        cap = lib.ssnb_jpeg_encode_restart_capacity(CODE[m], h, w, rb, rr)
        assert cap == R.capacity(m, h, w, rb, rr)
        assert len(_gold(i)) <= cap
    for mode, code in CODE.items():
        for h, w in ((1, 1), (17, 9), (256, 340), (360, 480), (65500, 65500), (8, 65500), (65500, 8)):
            assert lib.ssnb_jpeg_encode_restart_capacity(code, h, w, 0, 0) == lib.ssnb_jpeg_encode_capacity(code, h, w) == E.capacity(mode, h, w)
            for rb, rr in ((1, 0), (7, 0), (65535, 0), (0, 1), (0, 3), (0, 1 << 30)):
                assert lib.ssnb_jpeg_encode_restart_capacity(code, h, w, rb, rr) == R.capacity(mode, h, w, rb, rr)
    # the worst case per interval: a pad byte that is stuffed and two marker bytes over the marker-free bound
    assert R.capacity("L", 8, 16, 1, 0) - E.capacity("L", 8, 16) == 6 + 2 * ((2 * E.MAX_BLOCK_BITS + 14) // 8 - (2 * E.MAX_BLOCK_BITS + 7) // 8) + 2
    for rb, rr in ((-1, 0), (0, -1), (1, 1), (65536, 0)):
        assert lib.ssnb_jpeg_encode_restart_capacity(1, 8, 8, rb, rr) == 0
    from ops.jpeg import jpeg_encode_capacity
    assert jpeg_encode_capacity("RGB", 256, 340, restart_marker_rows=1) == R.capacity("RGB", 256, 340, 0, 1)
    assert jpeg_encode_capacity("RGB", 256, 340) == E.capacity("RGB", 256, 340)


def test_refusals_return_before_any_launch():
    L = _lib()
    lib = L.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(256)                    # a non-null, aligned pointer that is never dereferenced
    imgs = (L.JpegEncodeImage * 2)()
    for e, (h, w), off in zip(imgs, ((16, 24), (9, 7)), (0, 16 * 24 * 3)):
        e.src_offset, e.height, e.width = off, h, w
    ws, ob = C.c_size_t(), C.c_int64()
    assert lib.ssnb_jpeg_encode_restart_sizes(3, 95, 0, 1, imgs, 2, C.byref(ws), C.byref(ob)) == 0
    assert ob.value == R.capacity("RGB", 16, 24, 0, 1) + R.capacity("RGB", 9, 7, 0, 1)
    for rb, rr, why in ((1, 1, b"both"), (-1, 0, b">= 0"), (0, -3, b">= 0"), (65536, 0, b"65535"), (70000, 0, b"65535")):
        assert lib.ssnb_jpeg_encode_restart_sizes(3, 95, rb, rr, imgs, 2, C.byref(ws), C.byref(ob)) == 1
        assert why in lib.ssnb_last_error(None)
        rc = lib.ssnb_jpeg_encode_restart(3, 95, rb, rr, one, 10 ** 6, imgs, one, 2, one, 10 ** 9, one, one, 10 ** 9, None)
        assert rc == 1 and b"jpeg_encode" in lib.ssnb_last_error(None)
    # a slot or workspace sized without the markers is too small for them
    assert lib.ssnb_jpeg_encode_restart_sizes(3, 95, 1, 0, imgs, 2, C.byref(ws), C.byref(ob)) == 0
    ws0, ob0 = C.c_size_t(), C.c_int64()
    assert lib.ssnb_jpeg_encode_sizes(3, 95, imgs, 2, C.byref(ws0), C.byref(ob0)) == 0
    assert ob.value > ob0.value and ws.value >= ws0.value
    assert lib.ssnb_jpeg_encode_restart(3, 95, 1, 0, one, 10 ** 6, imgs, one, 2, one, ob0.value, one, one, ws.value, None) == 1
    assert lib.ssnb_global_launch_count() == n0


def test_python_refusals():
    import torch
    from ops.jpeg import encode_jpeg, JpegEncodePlan
    x = torch.zeros(1, 8, 8, 3, dtype=torch.uint8)
    for kw in (dict(restart_marker_blocks=1, restart_marker_rows=1), dict(restart_marker_blocks=-1), dict(restart_marker_rows=-2),
               dict(restart_marker_blocks=65536)):
        with pytest.raises(ValueError, match="restart_marker"):
            encode_jpeg(x, **kw)
        with pytest.raises(ValueError, match="restart_marker"):
            JpegEncodePlan([(8, 8)], **kw)
    for args in ((1, 1), (-1, 0), (0, -1), (65536, 0)):
        with pytest.raises(ValueError):
            R.check_restart(*args)


@pytest.mark.parametrize("kw", [dict(restart_marker_blocks=1), dict(restart_marker_blocks=5), dict(restart_marker_rows=1),
                                dict(restart_marker_rows=2)])
def test_write_jpegs_pillow_path_with_markers(tmp_path, kw):
    from ops.optical_flow import write_flow_jpegs, write_frame_jpegs
    rb, rr = kw.get("restart_marker_blocks", 0), kw.get("restart_marker_rows", 0)
    frames = np.stack([E.fixture("noise" if s % 2 else "ramp", 40, 56, 3, s) for s in range(5)])
    planes = np.stack([E.fixture("flow", 40, 56, 1, s) for s in range(6)])
    fp = write_frame_jpegs(frames, [str(tmp_path / "a"), str(tmp_path / "b")], offsets=[0, 3, 5], **kw)
    pp = write_flow_jpegs(planes, [str(tmp_path / "a"), str(tmp_path / "b")], offsets=[0, 3, 5], **kw)
    assert len(fp) == 5 and len(pp) == 6
    for p, a in zip(fp, frames):
        assert open(p, "rb").read() == G.pillow(a, "RGB", 95, rb, rr) == R.encode(a, "RGB", 95, rb, rr)
    for p, a in zip(pp, planes):
        assert open(p, "rb").read() == G.pillow(a, "L", 95, rb, rr) == R.encode(a, "L", 95, rb, rr)


def test_write_jpegs_refuse_both_keywords(tmp_path):
    from ops.optical_flow import write_flow_jpegs, write_frame_jpegs
    with pytest.raises(ValueError, match="restart_marker"):
        write_frame_jpegs(np.zeros((1, 8, 8, 3), np.uint8), str(tmp_path / "f"), restart_marker_blocks=1, restart_marker_rows=1)
    with pytest.raises(ValueError, match="restart_marker"):
        write_flow_jpegs(np.zeros((2, 8, 8, 1), np.uint8), str(tmp_path / "g"), restart_marker_blocks=-1)
    assert not os.path.exists(tmp_path / "f") and not os.path.exists(tmp_path / "g")


_CTYPE = {C.c_int: "int", C.c_int64: "int64_t", C.c_size_t: "size_t", C.c_void_p: "void*"}


def _c_type(t, L):
    if t in _CTYPE:
        return _CTYPE[t]
    if t is C.POINTER(L.JpegEncodeImage):
        return "const ssnb_jpeg_encode_image*"
    return _CTYPE[t._type_] + "*"


def test_header_prototypes_against_the_binding(tmp_path):
    """gcc compiles a call of each new entry with the argument and result types of its ctypes row, warnings as errors"""
    L = _lib()
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    body = []
    for name, n_args in (("ssnb_jpeg_encode_restart", 15), ("ssnb_jpeg_encode_restart_sizes", 8),
                         ("ssnb_jpeg_encode_restart_capacity", 5)):
        decl = re.search(r"\b%s\(([^)]*)\);" % name, hdr).group(1)
        res, args = L.SIGNATURES[name]
        assert len(decl.split(",")) == n_args == len(args), name
        body.append("%s r_%s = %s(%s);" % (_c_type(res, L), name, name, ", ".join("(%s)0" % _c_type(a, L) for a in args)))
        body.append("(void)r_%s;" % name)
    # the existing entries keep their prototypes
    for name, n_args in (("ssnb_jpeg_encode", 13), ("ssnb_jpeg_encode_sizes", 6), ("ssnb_jpeg_encode_capacity", 3)):
        assert len(re.search(r"\b%s\(([^)]*)\);" % name, hdr).group(1).split(",")) == n_args == len(L.SIGNATURES[name][1])
    src = tmp_path / "abi.c"
    src.write_text('#include <stddef.h>\n#include <stdint.h>\n#include "ssnb.h"\nvoid f(void) { %s }\n' % " ".join(body))
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Wconversion", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src),
                    "-o", str(tmp_path / "abi.o")], check=True)
