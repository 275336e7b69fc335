"""TAG bottom-up proposals on the GPU (csrc/proposals.cu, ops/proposals.py) against the reference's own outputs
(tests/golden/proposals.npz, oracle/gen_golden_proposals.py): labels, raw boxes and their order, box scores, NMS
survivors and pr_box exactly; smoothed values and the score merge to 1e-6; one batched call against per-video calls and
against a repeat; an adversarial alternating-label video.  Run on an H100: pytest -m gpu."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "proposals.npz"), allow_pickle=False)


def _kwargs(z, tag, minimum_len=None):
    p = tag + "_"
    bw = float(z[p + "bw"])
    return dict(bw=None if bw < 0 else bw, thresholds=z[p + "thresholds"].tolist(), tolerances=z[p + "tolerances"].tolist(),
                nms_threshold=float(z[p + "nms_thresh"]), minimum_len=float(z[p + "minimum_len"]) if minimum_len is None else minimum_len)


def _video(r, v, key, count_key):
    a, n = int(r["slot0"][v]), int(r[count_key][v])
    return r[key][a:a + n].cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def test_matches_reference_per_fixture(golden_dir):
    dev = _cuda()
    from ops.proposals import bottom_up_proposals_packed
    z = _golden(golden_dir)
    for tag in z["tags"]:
        p = tag + "_"
        f = torch.tensor(z[p + "f_score"], device=dev)
        T = f.shape[0]
        dur = [float(z[p + "duration"])]
        # every NMS survivor (no length filter), with the intermediate stages
        r = bottom_up_proposals_packed(f, [0, T], dur, trace=True, **_kwargs(z, tag, minimum_len=float("-inf")))
        sm = r["smoothed"][:T].cpu().numpy()
        assert np.abs(sm.astype(np.float64) - z[p + "smoothed"]).max() <= 1e-6, tag
        lab = r["labels"][:T].cpu().numpy().astype(np.int64)
        n_thr = len(z[p + "thresholds"])
        got_labels = np.stack([(lab >> k) & 1 for k in range(n_thr)]).astype(bool)
        np.testing.assert_array_equal(got_labels, z[p + "labels"], err_msg=tag)
        raw = _video(r, 0, "raw_frames", "raw_counts")
        np.testing.assert_array_equal(raw[:, 0], z[p + "raw_start"], err_msg=tag)
        np.testing.assert_array_equal(raw[:, 1], z[p + "raw_end"], err_msg=tag)
        np.testing.assert_array_equal(_bits(_video(r, 0, "raw_scores", "raw_counts")), _bits(z[p + "raw_score"]), err_msg=tag)
        kept = _video(r, 0, "frames", "counts")
        np.testing.assert_array_equal(kept[:, 0], z[p + "nms_start"], err_msg=tag)
        np.testing.assert_array_equal(kept[:, 1], z[p + "nms_end"], err_msg=tag)
        np.testing.assert_array_equal(_bits(_video(r, 0, "scores", "counts")), _bits(z[p + "nms_score"]), err_msg=tag)
        # gen_prop's pr_box, with the fixture's minimum_len; each box keeps its own score
        r = bottom_up_proposals_packed(f, [0, T], dur, **_kwargs(z, tag))
        np.testing.assert_array_equal(_bits(_video(r, 0, "seconds", "counts")), _bits(z[p + "pr_box"]), err_msg=tag)
        ok = (z[p + "nms_end"] / float(T) * dur[0] - z[p + "nms_start"] / float(T) * dur[0]) > float(z[p + "minimum_len"])
        np.testing.assert_array_equal(_bits(_video(r, 0, "scores", "counts")), _bits(z[p + "nms_score"][ok]), err_msg=tag)
    assert int(z["minlen_pr_box"].shape[0]) < int(z["minlen_nms_start"].shape[0])     # the filter is exercised


def test_list_interface_and_merge(golden_dir):
    dev = _cuda()
    from ops.proposals import bottom_up_proposals, merge_scores
    z = _golden(golden_dir)
    streams = [torch.tensor(z["merge_stream%d" % i], device=dev) for i in range(3)]
    merged = merge_scores(streams, z["merge_weights"].tolist())
    assert merged.shape == z["merge_f_score"].shape
    assert (merged.double().cpu() - torch.tensor(z["merge_f_score"]).double()).abs().max().item() <= 1e-6
    gold = torch.tensor(z["merge_f_score"], device=dev)
    props = bottom_up_proposals([gold, torch.tensor(z["t3000_f_score"], device=dev)],
                                [float(z["merge_duration"]), float(z["t3000_duration"])])
    prop = props[0]
    # the results are compact: they hold the kept boxes only, not the call's 12 * 9 * (T + 1) slots per video
    kept = sum(len(p.scores) for p in props)
    assert kept == len(z["merge_nms_score"]) + len(z["t3000_nms_score"])
    for p in props:
        assert p.pr_box.untyped_storage().nbytes() == kept * 16
        assert p.scores.untyped_storage().nbytes() == kept * 4 and p.frames.untyped_storage().nbytes() == kept * 8
    np.testing.assert_array_equal(_bits(prop.pr_box.cpu().numpy()), _bits(z["merge_pr_box"]))
    np.testing.assert_array_equal(prop.frames.cpu().numpy(), np.stack([z["merge_nms_start"], z["merge_nms_end"]], axis=1))
    np.testing.assert_array_equal(_bits(prop.scores.cpu().numpy()), _bits(z["merge_nms_score"]))


def test_batched_call_equals_single_calls_and_repeats(golden_dir):
    """all fixtures with the default parameters in ONE call (a K=2 score gets a -inf third column, which changes no softmax
    value and no box score, so the K=3 fixture can share the call) equal the videos called one at a time, bitwise; a repeat
    of the batched call is bitwise identical"""
    dev = _cuda()
    from ops.proposals import bottom_up_proposals_packed
    z = _golden(golden_dir)
    tags = [t for t in z["tags"] if float(z[t + "_bw"]) == 3 and len(z[t + "_thresholds"]) == 12 and len(z[t + "_tolerances"]) == 9]
    assert len(tags) >= 10
    fs, offsets, durs = [], [0], []
    for t in tags:
        f = torch.tensor(z[t + "_f_score"])
        if f.shape[1] == 2:
            f = torch.cat([f, torch.full((f.shape[0], 1), float("-inf"))], dim=1)
        fs.append(f)
        offsets.append(offsets[-1] + f.shape[0])
        durs.append(float(z[t + "_duration"]))
    packed = torch.cat(fs).to(dev)
    kw = dict(minimum_len=1.0)
    a = bottom_up_proposals_packed(packed, offsets, durs, trace=True, **kw)
    b = bottom_up_proposals_packed(packed, offsets, durs, trace=True, **kw)
    for k in ("counts", "raw_counts", "smoothed", "labels"):
        assert torch.equal(a[k], b[k]), k
    for v, t in enumerate(tags):
        one = bottom_up_proposals_packed(torch.tensor(z[t + "_f_score"], device=dev), [0, offsets[v + 1] - offsets[v]], [durs[v]],
                                         trace=True, **kw)
        for key, cnt in (("frames", "counts"), ("scores", "counts"), ("seconds", "counts"), ("raw_frames", "raw_counts"),
                         ("raw_scores", "raw_counts")):
            g, h, o = _video(a, v, key, cnt), _video(b, v, key, cnt), _video(one, 0, key, cnt)
            assert g.shape == o.shape, (t, key)
            np.testing.assert_array_equal(g.view(np.uint8), o.view(np.uint8), err_msg="%s %s" % (t, key))
            np.testing.assert_array_equal(g.view(np.uint8), h.view(np.uint8), err_msg="%s %s repeat" % (t, key))
        lo, hi = offsets[v], offsets[v + 1]
        assert torch.equal(a["labels"][lo:hi], one["labels"][:hi - lo]), t
        assert torch.equal(a["smoothed"][lo:hi], one["smoothed"][:hi - lo]), t


def test_adversarial_alternating_labels():
    """bw=None and labels alternating at every tick of T = 20000: ~1.1 M boxes before NMS, inside the workspace bound; every
    kept pair has IoU <= thresh and the kept scores do not increase"""
    dev = _cuda()
    from ops.proposals import bottom_up_proposals_packed
    T, thresh = 20000, 0.9
    f = torch.zeros(T, 2)
    f[:, 1] = torch.where(torch.arange(T) % 2 == 0, 8.0, -8.0)
    f[:, 1] += torch.linspace(-0.5, 0.5, T)
    f = f.to(dev)
    r = bottom_up_proposals_packed(f, [0, T], [600.0], bw=None, nms_threshold=thresh, trace=True)
    n_raw = int(r["raw_counts"][0])
    assert 12 * 9 * T // 2 <= n_raw <= 12 * 9 * (T + 1)
    n = int(r["counts"][0])
    assert n > 0
    fr = r["frames"][:n].long()
    sc = r["scores"][:n]
    assert bool((sc[1:] <= sc[:-1]).all())
    s, e = fr[:, 0], fr[:, 1]
    d = e - s + 1
    for lo in range(0, n, 2048):
        si, ei, di = s[lo:lo + 2048, None], e[lo:lo + 2048, None], d[lo:lo + 2048, None]
        inter = torch.minimum(ei, e[None]) - torch.maximum(si, s[None]) + 1
        iou = inter.double() / (di + d[None] - inter).double()
        idx = torch.arange(lo, min(lo + 2048, n), device=dev)[:, None]
        iou[idx == torch.arange(n, device=dev)[None]] = 0
        assert float(iou.max()) <= thresh


def test_call_captures_in_a_cuda_graph(golden_dir):
    """ssnb_tag_proposals only enqueues kernels (descriptors come from device offsets / durations): it captures in a CUDA
    graph, and a replay on new scores equals an eager call on them, bitwise"""
    dev = _cuda()
    import ctypes as C
    from ssn_b200._lib import lib, check, TagProposalsCfg
    from ops.proposals import THRESHOLDS, TOLERANCES, bottom_up_proposals_packed
    z = _golden(golden_dir)
    a, b = torch.tensor(z["t700_f_score"][:, :2]), torch.tensor(z["minlen_f_score"][:700])
    T, n_thr, n_tol = 700, len(THRESHOLDS), len(TOLERANCES)
    slots = n_thr * n_tol * (T + 1)
    f = a.clone().to(dev)
    offs = (C.c_int64 * 2)(0, T)
    offs_dev = torch.tensor([0, T], dtype=torch.int64, device=dev)
    durs_dev = torch.tensor([70.0], dtype=torch.float64, device=dev)
    thr_c = (C.c_double * n_thr)(*THRESHOLDS)
    tol_c = (C.c_double * n_tol)(*TOLERANCES)
    cfg = TagProposalsCfg(0, n_thr, n_tol, 0, 3.0, 0.9, 0.0, thr_c, tol_c)
    frames = torch.empty(slots, 2, dtype=torch.int32, device=dev)
    scores = torch.empty(slots, dtype=torch.float32, device=dev)
    seconds = torch.empty(slots, 2, dtype=torch.float64, device=dev)
    counts = torch.zeros(1, dtype=torch.int32, device=dev)
    ws_bytes = lib.ssnb_tag_proposals_workspace_bytes(1, T, n_thr, n_tol)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    def call():
        check(lib.ssnb_tag_proposals(C.byref(cfg), f.data_ptr(), 2, offs, offs_dev.data_ptr(), 1, durs_dev.data_ptr(),
                                     frames.data_ptr(), scores.data_ptr(), seconds.data_ptr(), counts.data_ptr(), None, None,
                                     None, None, None, ws.data_ptr(), ws_bytes,
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)), None, "tag_proposals")
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    f.copy_(b.to(dev))
    g.replay()
    torch.cuda.synchronize()
    n = int(counts[0])
    ref = bottom_up_proposals_packed(b.to(dev), [0, T], [70.0])
    assert n == int(ref["counts"][0]) > 0
    assert torch.equal(frames[:n], ref["frames"][:n]) and torch.equal(scores[:n], ref["scores"][:n])
    assert torch.equal(seconds[:n], ref["seconds"][:n])
