"""TV-L1 optical flow without a GPU: the float64 oracle (oracle/tvl1_oracle.py) against what OpenCV computed
(tests/golden/optical_flow.npz, oracle/gen_golden_flow.py) and on known motions, DenseFlow's quantisation at its edges, the
library's argument checks, and the header's parameter struct against the ctypes mirror."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import tvl1_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "optical_flow.npz"))


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


def test_oracle_grey_and_pyramid_against_opencv_golden():
    assert (O.grey(GOLD["grey_rgb"]) == GOLD["grey_cv2"]).all()
    sizes = [tuple(s) for s in GOLD["pyr_sizes"]]
    assert sizes == O.level_sizes(*sizes[0])
    for l in range(1, len(sizes)):
        assert _rel(O.resize(GOLD["pyr_%d" % (l - 1)], *sizes[l]), GOLD["pyr_%d" % l]) <= 1e-6
    assert _rel(O.resize(GOLD["up_src"], 49, 65), GOLD["up_cv2"]) <= 1e-6


def test_level_sizes_round_half_even_and_stop_under_16():
    assert O.level_sizes(256, 340) == [(256, 340), (205, 272), (164, 218), (131, 174), (105, 139)]
    assert O.level_sizes(40, 56) == [(40, 56), (32, 45), (26, 36), (21, 29), (17, 23)]
    assert O.level_sizes(25, 200) == [(25, 200), (20, 160), (16, 128)]
    assert O.level_sizes(15, 15) == [(15, 15)]
    assert O.level_sizes(256, 340, nscales=2) == [(256, 340), (205, 272)]


def test_library_level_count_equals_oracle_for_every_size():
    """ssnb_tvl1_levels against len(O.level_sizes(...)) for every h, w in 1 .. 600 at scale_step 0.8, 0.75 and 0.5 (odd sizes
    at 0.5 are exact half ties of R2's round half to even).  The oracle's count at nscales 32 is the shorter of the two axes'
    chains (R2 stops at the first axis under 16), checked against O.level_sizes itself on every seventh size; nscales 1 .. 32
    on every seventh h and w."""
    from ssn_b200._lib import lib
    assert O.level_sizes(33, 33, 5, 0.5) == [(33, 33), (16, 16)]           # 16.5 -> 16 (even), still a level
    assert O.level_sizes(35, 31, 5, 0.5) == [(35, 31), (18, 16)]           # 17.5 -> 18, 15.5 -> 16
    assert O.level_sizes(34, 600, 5, 0.5) == [(34, 600), (17, 300)]
    sizes = range(1, 601)
    for step in (0.8, 0.75, 0.5):
        axis = {n: len(O.level_sizes(n, 1 << 40, 32, step)) for n in sizes}
        want = lambda h, w, ns=32: min(ns, axis[h], axis[w])
        for h in sizes[::7]:
            for w in sizes[::7]:
                assert len(O.level_sizes(h, w, 32, step)) == want(h, w), (h, w, step)
        prm = _params(scale_step=step, nscales=32)
        bad = [(h, w) for h in sizes for w in sizes if lib.ssnb_tvl1_levels(prm, h, w) != want(h, w)]
        assert not bad, (step, bad[:10])
        for ns in range(1, 33):
            prm = _params(scale_step=step, nscales=ns)
            bad = [(h, w) for h in sizes[::7] for w in sizes[::7] if lib.ssnb_tvl1_levels(prm, h, w) != want(h, w, ns)]
            assert not bad, (step, ns, bad[:10])
            assert lib.ssnb_tvl1_levels(prm, 33, 33) == min(ns, 2 if step == 0.5 else 3 if step == 0.75 else 4)


def test_oracle_trace_brackets_its_own_stopping_rule():
    """trace= records R8's error per iteration: where the oracle's own rule stops a warp early, the last traced error is
    <= epsilon^2 h_l w_l of that level and every earlier one above it; a warp that runs out of iterations never went under.
    Replaying the counts traces the same errors."""
    I0, I1, _ = O.moving_pair(40, 56, ("shift", 0.8, -0.45), seed=4)
    tr = {}
    _, its = O.tvl1(np.rint(I0), np.rint(I1), iterations=40, trace=tr)
    sizes = O.level_sizes(40, 56)
    assert sorted(tr) == [(l, w) for l in range(len(sizes)) for w in range(5)]
    early = 0
    for (l, w), errs in tr.items():
        thr = 0.01 ** 2 * sizes[l][0] * sizes[l][1]
        assert len(errs) == its[l, w]
        assert all(e > thr for e in errs[:-1]), (l, w)
        if its[l, w] < 40:
            assert errs[-1] <= thr, (l, w)
            early += 1
        else:
            assert errs[-1] > thr, (l, w)
    assert early >= 10 and (its == 40).any()
    tr2 = {}
    O.tvl1(np.rint(I0), np.rint(I1), counts=its, trace=tr2)
    assert tr2 == tr


def test_single_frame_videos_in_offsets(tmp_path):
    """videos of one frame (no pair) at the start, in the middle, back to back and at the end: pair_offsets gives them empty
    ranges, and write_flow_jpegs (host planes) makes their directories and writes nothing in them"""
    from ops.optical_flow import pair_offsets, write_flow_jpegs
    off = [0, 1, 4, 5, 6, 9, 10]                           # 1, 3, 1, 1, 3, 1 frames
    assert pair_offsets(off).tolist() == [0, 0, 2, 2, 2, 4, 4]
    planes = np.arange(8, dtype=np.uint8).reshape(8, 1, 1, 1).repeat(8, 1).repeat(8, 2) * 30
    dirs = [str(tmp_path / ("v%d" % v)) for v in range(6)]
    paths = write_flow_jpegs(planes, dirs, offsets=off)
    assert [os.path.relpath(p, tmp_path) for p in paths] == ["v1/flow_x_00001.jpg", "v1/flow_y_00001.jpg", "v1/flow_x_00002.jpg",
                                                             "v1/flow_y_00002.jpg", "v4/flow_x_00001.jpg", "v4/flow_y_00001.jpg",
                                                             "v4/flow_x_00002.jpg", "v4/flow_y_00002.jpg"]
    assert all(os.path.isdir(d) for d in dirs) and not os.listdir(dirs[0]) and not os.listdir(dirs[5])
    from PIL import Image
    assert [int(np.asarray(Image.open(p)).mean().round()) for p in paths] == [0, 30, 60, 90, 120, 150, 180, 210]
    with pytest.raises(ValueError):
        write_flow_jpegs(planes, dirs, offsets=[0, 1, 4, 5, 6, 9, 11])


@pytest.mark.parametrize("motion", [("shift", 0.37, -0.61), ("shift", 1.6, 0.85), ("shift", -2.3, 0.2), ("rotate", 2.0)])
def test_oracle_recovers_known_motion(motion):
    """a seeded texture moved by a sub-pixel / two-pixel translation or a 2 degree rotation about the centre, rounded to
    uint8 grey: interior (8 px border) end-point error mean <= 0.05 px and max <= 0.25 px (measured 0.010 .. 0.018 and
    0.03 .. 0.08), with the stopping rule ending every warp early"""
    I0, I1, u = O.moving_pair(48, 64, motion, seed=1)
    flow, its = O.tvl1(np.rint(I0), np.rint(I1))
    mean, mx = O.epe(flow, u)
    assert mean <= 0.05 and mx <= 0.25, (mean, mx)
    assert its.shape == (5, 5) and its.max() < 300 and its.min() >= 1


def test_replayed_counts_reproduce_the_run():
    I0, I1, _ = O.moving_pair(32, 40, ("shift", 0.5, 0.25), seed=2)
    f, its = O.tvl1(I0, I1, iterations=20)
    g, its2 = O.tvl1(I0, I1, counts=its)
    assert (its == its2).all() and np.array_equal(f, g)
    h, its3 = O.tvl1(I0, I1, iterations=20, fixed_iterations=True)
    assert (its3 == 20).all()


def test_quantisation_edges():
    b = 20.0
    step = 40.0 / 255.0
    v = np.array([-b, b, np.nextafter(np.float32(-b), np.float32(-30)), np.nextafter(np.float32(b), np.float32(30)), -1e30, 1e30,
                  np.nan, 0.0, -step * 0.5 + 1e-6], np.float32)
    q = O.planes(v, b)
    assert q.tolist()[:7] == [0, 255, 0, 255, 0, 255, 0]
    assert q[7] == 128                      # 127.5 -> 128 (half to even)
    # exact halfway ties in double: 255 (v + 20) / 40 = k + 0.5 at v = (k + 0.5) * 40 / 255 - 20; fp32 values that land there
    ties = []
    for k in range(255):
        x = np.float32((k + 0.5) * 40.0 / 255.0 - 20.0)
        if 255.0 * (float(x) + 20.0) / 40.0 == k + 0.5:
            ties.append((x, k))
    for x, k in ties:
        assert O.planes(np.array([x]), b)[0] == (k if k % 2 == 0 else k + 1)
    assert ties                             # 0.0 is one (k = 127)
    assert O.planes(np.array([np.float32(-20.0 + 40.0 / 255.0 * 0.49)]), b)[0] == 0
    assert O.planes(np.array([np.float32(-20.0 + 40.0 / 255.0 * 0.51)]), b)[0] == 1


def _params(**kw):
    from ops.optical_flow import tvl1_params
    return tvl1_params(**kw)


def test_rejected_arguments_return_before_any_launch():
    from ssn_b200 import _lib
    lib = _lib.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(8)                                   # a non-null pointer that is never dereferenced
    off = np.array([0, 3, 5], np.int64)
    po = lambda a: np.ascontiguousarray(a, np.int64).ctypes.data_as(C.POINTER(C.c_int64))
    keep = []

    def call(prm=None, offsets=off, V=2, h=24, w=32, frames=one, flow=one, ws_bytes=None, **kw):
        prm = prm or _params(**kw)
        o = np.ascontiguousarray(offsets, np.int64)
        keep.append(o)
        need = lib.ssnb_tvl1_workspace_bytes(prm, po(o), V, h, w)
        rc = lib.ssnb_tvl1_flow(prm, frames, po(o), one, V, h, w, flow, None, one, need if ws_bytes is None else ws_bytes, None)
        return rc, need
    ws = lib.ssnb_tvl1_workspace_bytes(_params(), po(off), 2, 24, 32)
    assert ws > 0 and lib.ssnb_tvl1_workspace_bytes(_params(), po([0, 3, 9]), 2, 24, 32) > ws + 4 * 24 * 32 * 4 * 10
    for kw, why in ((dict(tau=0), "tau 0"), (dict(theta=-1), "negative theta"), (dict(lambda_=float("nan")), "NaN lambda"),
                    (dict(epsilon=-1), "negative epsilon"), (dict(scale_step=1.0), "scale_step 1"), (dict(scale_step=0), "scale_step 0"),
                    (dict(gamma=0.1), "gamma"), (dict(nscales=0), "no level"), (dict(warps=0), "no warp"), (dict(iterations=0), "no iteration"),
                    (dict(h=0), "height 0"), (dict(w=8193), "width 8193"), (dict(V=0), "no video"),
                    (dict(offsets=[1, 3, 5]), "offsets[0] != 0"), (dict(offsets=[0, 3, 3]), "a video without frames"),
                    (dict(offsets=[0, 1, 2]), "no pair"), (dict(offsets=[0, 32769], V=1), "32768 pairs")):
        rc, need = call(**kw)
        assert rc == 1 and need == 0, why
    assert call(frames=None)[0] == 1 and call(flow=None)[0] == 1
    assert call(ws_bytes=ws - 1)[0] == 1
    assert b"tvl1_flow" in lib.ssnb_last_error(None)
    ins, outs = (C.c_void_p * 6)(*[8] * 6), (C.c_void_p * 4)(*[8] * 4)
    for stage, n, h, w, oh, ow in ((6, 1, 8, 8, 0, 0), (-1, 1, 8, 8, 0, 0), (0, 0, 8, 8, 0, 0), (0, 65536, 8, 8, 0, 0), (1, 1, 8, 8, 0, 4),
                                   (3, 1, 0, 8, 0, 0)):
        assert lib.ssnb_tvl1_stage(stage, _params(), n, h, w, oh, ow, 1.0, ins, outs, None) == 1
    assert lib.ssnb_tvl1_stage(0, _params(), 1, 8, 8, 0, 0, 1.0, None, outs, None) == 1
    assert lib.ssnb_tvl1_stage(4, _params(gamma=1.0), 1, 8, 8, 0, 0, 1.0, ins, outs, None) == 1
    assert lib.ssnb_flow_planes(one, 1, 8, 8, 0.0, one, None) == 1
    assert lib.ssnb_flow_planes(one, 0, 8, 8, 20.0, one, None) == 1
    assert lib.ssnb_flow_planes(None, 1, 8, 8, 20.0, one, None) == 1
    assert lib.ssnb_tvl1_levels(_params(), 256, 340) == 5 and lib.ssnb_tvl1_levels(_params(nscales=0), 256, 340) == 0
    assert lib.ssnb_global_launch_count() == n0


def test_python_refusals():
    import torch
    from ops import optical_flow as F
    with pytest.raises(RuntimeError):
        F.tvl1_flow(torch.zeros(2, 16, 16, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        F.flow_planes(torch.zeros(1, 2, 4, 4))
    with pytest.raises(TypeError):
        F.tvl1_params(iteration=3)
    assert F.tvl1_params(**{"lambda": 0.2}).__getattribute__("lambda") == 0.2
    assert F.pair_offsets([0, 6, 9]).tolist() == [0, 5, 7]


def test_write_flow_jpegs_layout(tmp_path):
    from PIL import Image
    from ops.optical_flow import write_flow_jpegs
    rng = np.random.default_rng(0)
    planes = rng.integers(0, 256, (6, 12, 16, 1), dtype=np.uint8)
    paths = write_flow_jpegs(planes, [str(tmp_path / "a"), str(tmp_path / "b")], offsets=[0, 3, 5])
    names = [os.path.relpath(p, tmp_path) for p in paths]
    assert names == ["a/flow_x_00001.jpg", "a/flow_y_00001.jpg", "a/flow_x_00002.jpg", "a/flow_y_00002.jpg", "b/flow_x_00001.jpg",
                     "b/flow_y_00001.jpg"]
    im = Image.open(paths[4])
    assert im.mode == "L" and im.size == (16, 12)
    with pytest.raises(ValueError):
        write_flow_jpegs(planes, [str(tmp_path / "c")], offsets=[0, 3, 5])


def test_header_mirror_of_tvl1_params(tmp_path):
    from ssn_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct \{([^{}]*)\}\s*ssnb_tvl1_params;", hdr).group(1), flags=re.S)
    names = []
    for d in body.split(";"):
        if d.strip():
            names += [n.strip() for n in d.split(None, 1)[1].split(",")]
    assert names == [n for n, _ in _lib.TVL1Params._fields_]
    prints = ['printf("size %zu\\n", sizeof(ssnb_tvl1_params));'] + ['printf("%s %%zu\\n", offsetof(ssnb_tvl1_params, %s));' % (n, n) for n in names]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "abi")], check=True)
    lay = dict(l.split() for l in subprocess.run([str(tmp_path / "abi")], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(lay["size"]) == C.sizeof(_lib.TVL1Params)
    for n, _ in _lib.TVL1Params._fields_:
        assert int(lay[n]) == getattr(_lib.TVL1Params, n).offset
    for name, n_args in (("ssnb_tvl1_flow", 12), ("ssnb_tvl1_workspace_bytes", 5), ("ssnb_tvl1_stage", 11), ("ssnb_flow_planes", 7),
                         ("ssnb_tvl1_levels", 3)):
        decl = re.search(r"\b%s\(([^)]*)\);" % name, hdr).group(1)
        assert len(decl.split(",")) == n_args == len(_lib.SIGNATURES[name][1]), name
