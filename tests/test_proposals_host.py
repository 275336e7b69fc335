"""TAG bottom-up proposals without a GPU: the numpy oracle against the reference's own outputs
(tests/golden/proposals.npz, oracle/gen_golden_proposals.py) bit for bit, its Gaussian against scipy, and the library's
argument checks, workspace formula and compiled kernels."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import proposal_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = ("ss", "smoothed", "labels", "raw_start", "raw_end", "raw_score", "nms_start", "nms_end", "nms_score", "pr_box")


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "proposals.npz"), allow_pickle=False)


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _tags():
    return [str(t) for t in np.load(os.path.join(ROOT, "tests", "golden", "proposals.npz"))["tags"]]


@pytest.mark.parametrize("tag", _tags())
def test_oracle_matches_reference(golden_dir, tag):
    z, p = _golden(golden_dir), tag + "_"
    bw = float(z[p + "bw"])
    r = P.gen_prop(z[p + "f_score"], float(z[p + "duration"]), bw=None if bw < 0 else bw, thresholds=z[p + "thresholds"].tolist(),
                   tolerances=z[p + "tolerances"].tolist(), nms_threshold=float(z[p + "nms_thresh"]),
                   minimum_len=float(z[p + "minimum_len"]))
    for k in STAGES:
        assert _same_bits(r[k], z[p + k]), k
    if tag == "minlen":
        assert len(r["pr_box"]) < len(r["nms_start"])
        # the reference pairs the filtered boxes with ALL survivors' scores; the oracle keeps each box's own score
        assert len(z[p + "pr_score_ref"]) == len(r["nms_score"]) != len(r["pr_score"])
    else:
        assert _same_bits(r["pr_score"], z[p + "pr_score_ref"])


def test_fixture_coverage(golden_dir):
    z = _golden(golden_dir)
    assert len(z["noisy_raw_start"]) >= 20000 and len(z["noisy_f_score"]) == 12000
    assert z["all_fg_labels"].all() and not z["all_bg_labels"].any() and len(z["all_bg_raw_start"]) == 0
    assert z["edges_labels"][:, 0].any() and z["edges_labels"][:, -1].any() and not z["edges_labels"][:, 200].any()
    assert float(z["alt_bw"]) < 0 and (z["alt_labels"][:, 1:] != z["alt_labels"][:, :-1]).mean() > 0.5
    assert {len(z[t + "_f_score"]) for t in ("t1", "t2", "t5", "t13", "t700", "t3000")} == {1, 2, 5, 13, 700, 3000}
    assert (z["t5_raw_end"] == 6).any()                 # a box ending after the video (T + 1)


def test_merge_matches_reference(golden_dir):
    z = _golden(golden_dir)
    streams = [z["merge_stream%d" % i] for i in range(3)]
    assert streams[1].shape[0] < streams[0].shape[0] < streams[2].shape[0]
    assert _same_bits(P.merge_scores(streams, z["merge_weights"].tolist()), z["merge_f_score"])


@pytest.mark.parametrize("T", [1, 2, 5, 12, 13, 26, 100, 701])
@pytest.mark.parametrize("sigma", [0.1, 1, 2.5, 3])
def test_numpy_gaussian_equals_scipy(T, sigma):
    from scipy.ndimage import gaussian_filter
    x = np.random.RandomState(T).rand(T).astype(np.float32)
    assert _same_bits(P.gaussian_filter1d(x, sigma), gaussian_filter(x, sigma))


def _layout_bytes(V, N, n_thr, n_tol):
    a = lambda b: (b + 255) // 256 * 256
    S = N + V
    slots, edges = n_thr * n_tol * S, n_thr * S
    return (a(40 * V) + 3 * a(4 * N) + a(4 * V * n_thr) + 2 * a(4 * V) + 4 * a(4 * edges) + a(32 * edges)
            + 2 * a(4 * slots) + 2 * a(8 * slots) + a(slots) + 256)


def test_workspace_formula():
    from ssn_b200._lib import lib
    for V, N, n_thr, n_tol in ((1, 1, 12, 9), (1, 100, 12, 9), (3, 17, 1, 1), (200, 2_400_000, 12, 9), (5, 999, 32, 32)):
        assert lib.ssnb_tag_proposals_workspace_bytes(V, N, n_thr, n_tol) == _layout_bytes(V, N, n_thr, n_tol)
    assert lib.ssnb_tag_proposals_workspace_bytes(0, 0, 12, 9) == _layout_bytes(0, 0, 12, 9)
    for bad in ((1, 1, 0, 9), (1, 1, 33, 9), (1, 1, 12, 0), (-1, 1, 12, 9), (1, 30_000_000, 12, 9)):
        assert lib.ssnb_tag_proposals_workspace_bytes(*bad) == 0


def _call(offsets=(0, 5, 9), offs_dev=256, K=2, cls=0, thr=(0.5,), tol=(0.2,), sigma=3.0, nms=0.9, min_len=0.0, out=256, ws_bytes=1 << 40):
    from ssn_b200._lib import lib, TagProposalsCfg
    thr_c, tol_c = (C.c_double * len(thr))(*thr), (C.c_double * len(tol))(*tol)
    cfg = TagProposalsCfg(cls, len(thr), len(tol), 0, sigma, nms, min_len, thr_c, tol_c)
    V = len(offsets) - 1
    offs = (C.c_int64 * len(offsets))(*offsets)
    p = 256                                                           # never dereferenced: validation fails first
    return lib.ssnb_tag_proposals(C.byref(cfg), p, K, offs, offs_dev, V, p, out, p, p, p, None, None, None, None, None, p, ws_bytes, None)


def test_arguments_are_validated():
    from ssn_b200._lib import lib
    assert _call(offsets=(0, 5, 5)) == 1                               # an empty video
    assert b"offsets" in lib.ssnb_last_error(None)
    assert _call(offsets=(0, 5, 3)) == 1                               # not monotone
    assert _call(offsets=(1, 5, 9)) == 1
    assert _call(K=1) == 1 and b"cls + 1" in lib.ssnb_last_error(None)
    assert _call(K=2, cls=1) == 1
    assert _call(nms=1.0) == 1 and b"nms_thresh" in lib.ssnb_last_error(None)
    assert _call(nms=-0.1) == 1 and _call(nms=float("nan")) == 1
    assert _call(thr=()) == 1 and _call(thr=(0.5,) * 33) == 1 and _call(tol=()) == 1
    assert _call(thr=(float("nan"),)) == 1 and _call(tol=(float("inf"),)) == 1
    assert _call(sigma=-1.0) == 1 and _call(sigma=16.0) == 1 and _call(sigma=float("nan")) == 1
    assert _call(min_len=float("nan")) == 1
    assert _call(out=None) == 1 and b"NULL" in lib.ssnb_last_error(None)
    assert _call(offs_dev=None) == 1 and b"device offsets" in lib.ssnb_last_error(None)
    assert _call(ws_bytes=100) == 1 and b"workspace" in lib.ssnb_last_error(None)
    assert _call(offsets=(0,)) == 0                                    # no videos: nothing to do


def test_wrapper_rejects_bad_input():
    from ops.proposals import bottom_up_proposals, bottom_up_proposals_packed
    with pytest.raises(RuntimeError):                                   # no CPU fallback
        bottom_up_proposals([torch.zeros(10, 2)], [1.0])
    with pytest.raises(RuntimeError):
        bottom_up_proposals_packed(torch.zeros(10, 2), [0, 10], [1.0])


def test_kernels_compile_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "action-detection_b200", "csrc", "proposals.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                          "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "proposals.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", out.stderr)
    assert sum("proposals_cu" in k for k in kernels) == 7
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", out.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills)
