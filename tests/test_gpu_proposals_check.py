"""TAG bottom-up proposals on the GPU (csrc/proposals.cu through ops/proposals.bottom_up_proposals_packed(trace=True)),
every video checked stage by stage by oracle/proposal_check.py on random ragged batches: block-size boundaries of every
kernel (T around 256 / 512 / 1024, run counts around the search tree's powers of two, more than 128 videos per call), score
families with exact ties, NaN of either sign and inf, and the parameter edges (K = 2 / 3 / 21 and cls, Gaussian radius 0 to
63, 32 thresholds and tolerances with duplicates, nms_thresh 0 to 0.999, minimum_len -inf to 1e9).  Properties of the call
itself: per-video calls, a repeat, trace=False and pre-filled memory give the same bits.  Run on an H100: pytest -m gpu."""
import ctypes as Cc

import numpy as np
import pytest
import torch

from oracle import proposal_check as C
from oracle import proposal_oracle as P

pytestmark = pytest.mark.gpu

FAMILIES = ("smooth", "sinus", "quant", "zero_fg", "nan", "nan_bg", "inf", "neginf_row", "runs", "runs_regular")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _videos(Ts, seed, K=2, cls=0, families=FAMILIES, end_fg=False):
    g = np.random.RandomState(seed)
    out = []
    for i, T in enumerate(Ts):
        kind = families[i % len(families)]
        out.append((C.make_scores(kind, int(T), g, K=K, cls=cls, end_fg=end_fg), T / g.uniform(2.0, 8.0)))
    return out


def _call(dev, f, offsets, durs, trace=True, **kw):
    from ops.proposals import bottom_up_proposals_packed
    return bottom_up_proposals_packed(torch.from_numpy(f).to(dev), offsets, durs, trace=trace, **kw)


def _checked(dev, videos, name, **kw):
    f, offsets, durs = C.pack(videos)
    r = _call(dev, f, offsets, durs, **kw)
    chk = C.check(r, f, offsets, durs, **kw)
    print("%s: %s" % (name, chk.report()))
    chk.assert_ok()
    return r, chk, (f, offsets, durs)


def _slices(r, v, keys=("frames", "scores", "seconds"), count="counts"):
    a, n = int(r["slot0"][v]), int(r[count][v])
    return [r[k][a:a + n].cpu().numpy().view(np.uint8).tobytes() for k in keys]


def _same_video(a, b, va, vb, trace=True):
    assert int(a["counts"][va]) == int(b["counts"][vb])
    assert _slices(a, va) == _slices(b, vb)
    if trace:
        assert int(a["raw_counts"][va]) == int(b["raw_counts"][vb])
        assert _slices(a, va, ("raw_frames", "raw_scores"), "raw_counts") == _slices(b, vb, ("raw_frames", "raw_scores"), "raw_counts")


def _prefilled_call(dev, f, offsets, durs, thresholds=P.THRESHOLDS, tolerances=P.TOLERANCES, **kw):
    """the C ABI with every output and the workspace filled with 0xFF bytes first"""
    from ssn_b200._lib import lib, check, TagProposalsCfg
    V, N, n_thr, n_tol = len(offsets) - 1, offsets[-1], len(thresholds), len(tolerances)
    slots = n_thr * n_tol * (N + V)

    def buf(n, dtype):
        size = torch.tensor([], dtype=dtype).element_size()
        return torch.full((n * size,), 0xFF, dtype=torch.uint8, device=dev).view(dtype)
    out = {"frames": buf(2 * slots, torch.int32).view(-1, 2), "scores": buf(slots, torch.float32),
           "seconds": buf(2 * slots, torch.float64).view(-1, 2), "counts": buf(V, torch.int32), "smoothed": buf(N, torch.float32),
           "labels": buf(N, torch.int32), "raw_frames": buf(2 * slots, torch.int32).view(-1, 2), "raw_scores": buf(slots, torch.float32),
           "raw_counts": buf(V, torch.int32)}
    ws_bytes = lib.ssnb_tag_proposals_workspace_bytes(V, N, n_thr, n_tol)
    ws = buf(ws_bytes, torch.uint8)
    bw = kw.get("bw", 3)
    cfg = TagProposalsCfg(int(kw.get("cls", 0)), n_thr, n_tol, 0, 0.0 if bw is None else float(bw), float(kw.get("nms_threshold", 0.9)),
                          float(kw.get("minimum_len", 0.0)), (Cc.c_double * n_thr)(*thresholds), (Cc.c_double * n_tol)(*tolerances))
    fd = torch.from_numpy(f).to(dev)
    offs_dev = torch.tensor(offsets, dtype=torch.int64, device=dev)
    durs_dev = torch.tensor(durs, dtype=torch.float64, device=dev)
    p = {k: v.data_ptr() for k, v in out.items()}
    check(lib.ssnb_tag_proposals(Cc.byref(cfg), fd.data_ptr(), fd.shape[1], (Cc.c_int64 * (V + 1))(*offsets), offs_dev.data_ptr(), V,
                                 durs_dev.data_ptr(), p["frames"], p["scores"], p["seconds"], p["counts"], p["smoothed"], p["labels"],
                                 p["raw_frames"], p["raw_scores"], p["raw_counts"], ws.data_ptr(), ws_bytes,
                                 Cc.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "tag_proposals")
    torch.cuda.synchronize()
    out["slot0"] = torch.tensor([n_thr * n_tol * (offsets[v] + v) for v in range(V)], dtype=torch.int64)
    return out


def test_ragged_batch_of_300_videos_and_call_properties():
    """one call of 300 videos (more than 128: desc_kernel's block), T from 1 to 3000, every score family, gen_prop's
    defaults; then a sample of the videos one at a time, a repeat, trace=False and pre-filled memory give the same bits"""
    dev = _cuda()
    g = np.random.RandomState(300)
    Ts = np.minimum(3000, np.exp(g.uniform(0, np.log(3000), 300)).astype(int) + 1)
    fams = FAMILIES * 3 + ("noisy",)
    r, chk, (f, offsets, durs) = _checked(dev, _videos(Ts, 1, families=fams), "300 videos")
    assert chk.stats["nan_boxes"] > 0 and chk.stats["tied_boxes"] > 0
    b = _call(dev, f, offsets, durs)
    nt = _call(dev, f, offsets, durs, trace=False)
    for k in ("counts", "raw_counts", "labels"):
        assert torch.equal(r[k], b[k]), k
    assert torch.equal(r["smoothed"].view(torch.int32), b["smoothed"].view(torch.int32))
    assert torch.equal(r["counts"], nt["counts"])
    for v in range(300):
        _same_video(r, b, v, v)
        _same_video(r, nt, v, v, trace=False)
    for v in (0, 1, 97, 128, 129, 299):
        lo, hi = offsets[v], offsets[v + 1]
        one = _call(dev, np.ascontiguousarray(f[lo:hi]), [0, hi - lo], [durs[v]])
        _same_video(r, one, v, 0)
        assert torch.equal(r["labels"][lo:hi], one["labels"][:hi - lo])
        assert torch.equal(r["smoothed"][lo:hi].view(torch.int32), one["smoothed"][:hi - lo].view(torch.int32))
    ff = _prefilled_call(dev, f, offsets, durs)
    for k in ("counts", "raw_counts", "labels"):
        assert torch.equal(r[k], ff[k]), k
    assert torch.equal(r["smoothed"].view(torch.int32), ff["smoothed"].view(torch.int32))
    for v in range(300):
        _same_video(r, ff, v, v)


def test_block_boundary_lengths():
    """T at the edges of kEdgeThreads / kSearchThreads (256), the 4 x 128 score split and kNmsThreads (512): runs that end
    on the last tick (the final falling edge) with bw None, then smooth / quantised scores with bw 3 and a 12000-tick noisy
    video"""
    dev = _cuda()
    Ts = (1, 2, 12, 13, 255, 256, 257, 511, 512, 513, 1024, 1025)
    _checked(dev, _videos(Ts, 2, families=("runs_regular", "runs"), end_fg=True), "runs ending on the last tick", bw=None)
    vids = _videos(Ts, 3, families=("quant", "smooth", "zero_fg"))
    g = np.random.RandomState(4)
    vids.append((C.make_scores("noisy", 12000, g), 1200.0))
    _checked(dev, vids, "boundary lengths + noisy 12000")


@pytest.mark.parametrize("regular", [False, True])
def test_exact_run_counts(regular):
    """exactly U foreground runs at threshold 0.5 (bw None), U around the search tree's sizes and the 256-thread loop,
    32 tolerances (0 / 0.5 / 1 / 1.3 / -0.2 among them; regular runs tie every signal at 0.5)"""
    dev = _cuda()
    g = np.random.RandomState(5 + regular)
    vids = []
    for U in (1, 2, 3, 255, 256, 257, 511, 512, 513):
        T = 4 * U + int(g.randint(0, 9)) if not regular else 4 * U
        vids.append((C.make_scores("runs_regular" if regular else "runs", T, g, U=U, end_fg=bool(U % 2)), T / 5.0))
    r, chk, (f, offsets, durs) = _checked(dev, vids, "run counts (regular %s)" % regular, bw=None, thresholds=(0.5,),
                                          tolerances=C.TOL32)
    lab = r["labels"].cpu().numpy().view(np.uint32) & 1
    for v, U in enumerate((1, 2, 3, 255, 256, 257, 511, 512, 513)):
        x = lab[offsets[v]:offsets[v + 1]].astype(int)
        assert int((np.diff(np.concatenate([[0], x])) == 1).sum()) == U


PARAMS = [  # K, cls, bw, thresholds, tolerances, nms_threshold, minimum_len
    (3, 1, None, C.THR32, C.TOL32, 0.5, 0.0),
    (21, 19, 15.7, P.THRESHOLDS, P.TOLERANCES, 0.999, float("-inf")),
    (21, 0, 1e-16, (0.3, 0.5, 0.5, 0.7, 0.3), C.TOL32, 0.0, 4.0),
    (3, 0, 0.3, C.THR32, P.TOLERANCES, 0.9, 1e9),
    (2, 0, 3, P.THRESHOLDS, P.TOLERANCES, 0.0, 0.0),
    (21, 1, 3, C.THR32, C.TOL32, 0.9, 0.0),
    (3, 1, 15.7, (0.5, 0.5, 0.5), (0.5, 1.0, 0.5), 0.5, 4.0),
]


@pytest.mark.parametrize("K, cls, bw, thr, tol, nms, min_len", PARAMS)
def test_parameters(K, cls, bw, thr, tol, nms, min_len):
    dev = _cuda()
    g = np.random.RandomState(K * 100 + cls)
    Ts = [1, 2, 40, 62] + [int(x) for x in g.randint(63, 400 if len(thr) * len(tol) > 200 else 900, 8)]
    _checked(dev, _videos(Ts, K + cls, K=K, cls=cls), "K %d cls %d bw %s %dx%d nms %g min_len %g" % (K, cls, bw, len(thr), len(tol), nms, min_len),
             cls=cls, bw=bw, thresholds=thr, tolerances=tol, nms_threshold=nms, minimum_len=min_len)
