"""Frame resize without a GPU: the numpy restatement of cv2.resize(INTER_LINEAR) (oracle/frame_resize_oracle.py) against
every cv2 output of tests/golden/frame_resize.npz, OpenCV's copy and 2 x 2 area paths against the linear rule the kernel
computes, the generator against the golden file where cv2 imports; the library's refusals, which launch nothing; and the
header's declaration against the ctypes binding."""
import ctypes as C
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from oracle import frame_resize_oracle as R
from oracle import gen_golden_frame_resize as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "frame_resize.npz")


def _golden():
    return np.load(GOLDEN)


def test_golden_index_matches_the_generator():
    g = _golden()
    assert list(g["names"]) == [G.name(*s) for s in G.fixtures()]
    assert len(g["names"]) == len(G.SOURCES) * len(G.KINDS) + 40 * len(G.SWEEP_SOURCES)


def test_oracle_equals_every_golden_fixture():
    g = _golden()
    stored = 0
    for spec in G.fixtures():
        kind, h, w, seed, dh, dw = spec
        n = G.name(*spec)
        img = G.image(kind, h, w, seed)
        assert zlib.crc32(img.tobytes()) == int(g["crc_" + n]), ("input drifted", n)
        got = R.resize(img, dw, dh)
        assert got.shape == (dh, dw, 3) and got.dtype == np.uint8
        assert zlib.crc32(got.tobytes()) == int(g["ocrc_" + n]), n
        if "out_" + n in g.files:
            assert got.tobytes() == g["out_" + n].tobytes(), n
            stored += 1
    assert stored == len(G.fixtures()) - (len(G.SOURCES) - len(G.NOISE_KEPT))


def test_linear_equals_special_paths():
    """cv::resize's copy (dsize == ssize) and hal::resize's area fast path (exact 2 x 2) give what the linear rule gives,
    which is why the kernel has no separate path for them"""
    for kind in G.KINDS:
        for (h, w), (dh, dw) in (((256, 340), (256, 340)), ((512, 680), (256, 340)), ((2, 2), (1, 1)), ((14, 6), (7, 3)),
                                 ((1, 1), (1, 1)), ((7, 5), (7, 5))):
            img = G.image(kind, h, w, h + w)
            assert R.is_area_fast_2x(h, w, dh, dw) or (h, w) == (dh, dw)
            assert R.resize(img, dw, dh).tobytes() == R.linear(img, dw, dh).tobytes(), (kind, h, w, dh, dw)
    # not the area path: 3x, 2x along one axis only, 2x of an odd side
    assert not R.is_area_fast_2x(768, 1020, 256, 340)
    assert not R.is_area_fast_2x(256, 680, 256, 340)
    assert not R.is_area_fast_2x(15, 14, 7, 7)


def test_oracle_over_frames_equals_each_frame():
    rng = np.random.default_rng(3)
    for n, h, w in ((3, 240, 320), (2, 512, 680), (4, 1, 5), (2, 256, 340)):
        v = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
        assert R.resize(v, 340, 256).tobytes() == np.stack([R.resize(f, 340, 256) for f in v]).tobytes()


def test_generator_reproduces_the_golden_file():
    cv2 = pytest.importorskip("cv2")
    g, new = _golden(), G.golden(cv2)
    assert sorted(g.files) == sorted(new)
    for k in g.files:
        assert g[k].dtype == new[k].dtype and g[k].tobytes() == new[k].tobytes(), k


def test_oracle_equals_cv2_on_random_sizes():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    for _ in range(150):
        h, w = int(rng.integers(1, 1081)), int(rng.integers(1, 1921))
        if rng.random() < 0.3:
            h, w = int(rng.integers(1, 24)), int(rng.integers(1, 24))
        dh, dw = int(rng.integers(1, 400)), int(rng.integers(1, 400))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert R.resize(img, dw, dh).tobytes() == ref.tobytes(), (h, w, dh, dw)


def _lib():
    from ssn_b200 import _lib
    return _lib


def test_refusals_return_before_any_launch():
    L = _lib()
    lib = L.lib
    n0 = lib.ssnb_global_launch_count()
    src, dst = C.c_void_p(1 << 20), C.c_void_p(1 << 30)     # non-null pointers that are never dereferenced

    def call(videos=((2, 16, 24), (1, 9, 7)), dst_hw=(8, 10), src_bytes=10 ** 6, dst_bytes=10 ** 6, first=None, offset=None,
             ptrs=(src, src, dst), n=None, table=True):
        arr = (L.ResizeVideo * max(len(videos), 1))()
        off, fr = 0, 0
        for i, (e, (f, h, w)) in enumerate(zip(arr, videos)):
            e.src_offset, e.first_frame, e.height, e.width, e.frames = off if offset is None else offset, fr if first is None else first[i], h, w, f
            off += f * h * w * 3
            fr += f
        rc = lib.ssnb_frame_resize(ptrs[0], src_bytes, arr if table else None, ptrs[1], len(videos) if n is None else n, dst_hw[0],
                                   dst_hw[1], ptrs[2], dst_bytes, None)
        return rc, (lib.ssnb_last_error(None) or b"").decode()

    need = 3 * 8 * 10 * 3
    for kw, why in ((dict(videos=()), "no video"), (dict(n=0), "no video"), (dict(table=False), "NULL videos"),
                    (dict(dst_hw=(0, 10)), "destination height and width"), (dict(dst_hw=(8, 65501)), "destination height and width"),
                    (dict(videos=((1, 0, 8),)), "height and width"), (dict(videos=((1, 8, 65501),)), "height and width"),
                    (dict(videos=((0, 8, 8),)), "frames must be"), (dict(first=(0, 1)), "first_frame"), (dict(first=(1, 3)), "first_frame"),
                    (dict(src_bytes=2 * 16 * 24 * 3), "outside src"), (dict(offset=-1), "outside src"),
                    (dict(dst_bytes=need - 1), "fewer than"), (dict(ptrs=(None, src, dst)), "NULL src"),
                    (dict(ptrs=(src, None, dst)), "NULL src"), (dict(ptrs=(src, src, None)), "NULL src"),
                    (dict(ptrs=(src, src, C.c_void_p((1 << 20) + 100))), "overlaps"),
                    (dict(ptrs=(src, src, C.c_void_p((1 << 20) - need + 1))), "overlaps")):
        rc, msg = call(**kw)
        assert rc == 1, (kw, msg)
        assert msg.startswith("frame_resize: ") and why in msg, (kw, msg)
    assert lib.ssnb_global_launch_count() == n0


def test_python_refusals():
    import torch
    from ops.optical_flow import resize_frames, ResizePlan
    with pytest.raises(RuntimeError, match="no CPU path"):
        resize_frames([torch.zeros(2, 8, 8, 3, dtype=torch.uint8)])
    with pytest.raises(RuntimeError, match="no CPU path"):
        resize_frames(torch.zeros(2, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="at least one video"):
        resize_frames([])
    with pytest.raises(ValueError, match="at least one video"):
        ResizePlan([])
    with pytest.raises(ValueError, match="at least one frame"):
        ResizePlan([(2, 8, 8), (0, 8, 8)])
    for hw in ((0, 8), (8, 65501)):
        with pytest.raises(ValueError, match="frame height and width"):
            ResizePlan([(1,) + hw])
        with pytest.raises(ValueError, match="destination height and width"):
            ResizePlan([(1, 8, 8)], width=hw[1], height=hw[0])


def test_header_declaration_matches_the_binding(tmp_path):
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    decl = re.search(r"\bint ssnb_frame_resize\(([^)]*)\);", hdr).group(1)
    res, args = L.SIGNATURES["ssnb_frame_resize"]
    assert res is C.c_int and len(decl.split(",")) == len(args) == 10
    kinds = {"int": C.c_int, "int64_t": C.c_int64}
    for p, a in zip(decl.split(","), args):
        if "*" in p:
            assert a is C.c_void_p or a.__name__.startswith("LP_"), (p, a)
        else:
            assert a is kinds[p.strip().rsplit(None, 1)[0]], (p, a)
    assert args[2]._type_ is L.ResizeVideo
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    names = [n for n, _ in L.ResizeVideo._fields_]
    prints = ['printf("size %zu\\n", sizeof(ssnb_resize_video));']
    prints += ['printf("%s %%zu\\n", offsetof(ssnb_resize_video, %s));' % (n, n) for n in names]
    inc = os.path.join(ROOT, "include")
    # the prototype the binding assumes, checked against the header's by the C compiler
    proto = tmp_path / "proto.c"
    proto.write_text('#include <stddef.h>\n#include "ssnb.h"\n'
                     'int (*f)(const uint8_t*, int64_t, const ssnb_resize_video*, const ssnb_resize_video*, int, int, int, uint8_t*, '
                     'int64_t, void*) = ssnb_frame_resize;\n')
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-c", "-I", inc, str(proto), "-o", str(tmp_path / "proto.o")], check=True)
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(tmp_path / "abi")], check=True)
    run = subprocess.run([str(tmp_path / "abi")], check=True, capture_output=True, text=True)
    lay = dict(l.split() for l in run.stdout.splitlines())
    assert int(lay["size"]) == C.sizeof(L.ResizeVideo)
    for n in names:
        assert int(lay[n]) == getattr(L.ResizeVideo, n).offset, n
