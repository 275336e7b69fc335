"""The proposal-labelling oracle (oracle/proplist_oracle.py) against tests/golden/proplist.npz, which holds what the real
reference computed (oracle/gen_golden_proplist.py): everything bitwise, the list text character by character.  No GPU."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import proplist_oracle as P

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proplist.npz"))


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def split(flat, counts):
    return np.split(flat, np.cumsum(counts)[:-1])


def ragged():
    b, g, l = (split(GOLD[k], GOLD[c]) for k, c in (("rag_boxes", "rag_count"), ("rag_gt", "rag_gt_count"), ("rag_gt_label", "rag_gt_count")))
    return b, g, l, GOLD["rag_duration"], GOLD["rag_frame_cnt"]


def test_name_proposals_and_recall():
    boxes, gt, lab, _, _ = ragged()
    named = [P.name_proposals(g, l, b) for g, l, b in zip(gt, lab, boxes)]
    for i, k in enumerate(("rag_label", "rag_max_overlap", "rag_overlap_self")):
        assert same(np.concatenate([n[i] for n in named]), GOLD[k]), k
    # two ground truths at the same tIoU: the first is named (video 3, proposal 1)
    assert named[3][0][1] == 3 and named[3][1][1] == 5.0 / 7.0
    best = [P.gt_best_iou(g, b) for g, b in zip(gt, boxes)]
    hits, pv, pi = P.proposal_recall(best, GOLD["rag_thresholds"])
    assert same(hits, GOLD["rag_hits"])
    assert same(np.stack([pv, pi], 1), GOLD["rag_recall"])


def test_sliding_windows():
    for c, (ts, ml, ov) in enumerate(GOLD["sw_configs"]):
        got = [P.sliding_windows(d, int(ts), int(ml), float(ov)) for d in GOLD["sw_durations"]]
        assert same(np.array([len(x) for x in got], np.int32), GOLD["sw%d_count" % c])
        assert same(np.concatenate(got), GOLD["sw%d_boxes" % c])


def oracle_list_text():
    boxes, gt, lab, dur, fc = ragged()
    text = ""
    for v in range(len(boxes)):
        label, mo, ms = P.name_proposals(gt[v], lab[v], boxes[v])
        text += "# {}\n".format(v + 1) + P.format_window_list("frames/video_%04d" % v, int(fc[v]), lab[v] + 1, P.seconds_to_frames(gt[v], dur[v], fc[v]),
                                                              label, mo, ms, P.seconds_to_frames(boxes[v], dur[v], fc[v]))
    return text


def records(text, frame_cnts=None, normalised=False):
    """parsed list -> the kept rows per video, as proposal_targets / test_proposals take them"""
    vids = []
    for i, (_, n_frame, gt, pr) in enumerate(P.parse_proposal_list(text)):
        fc = n_frame if frame_cnts is None else int(frame_cnts[i])
        conv = (lambda b: P.normalised_to_frames(b, fc)) if normalised else (lambda b: np.array([[int(x) for x in r] for r in b], np.int64).reshape(-1, 2))
        pk, pv, pc = P.record_rows(conv([r[3:5] for r in pr]), fc)
        gk, gv, _ = P.record_rows(conv([r[1:3] for r in gt]), fc)
        col = lambda j, dt: np.array([dt(r[j]) for r in pr], np.float64 if dt is float else np.int32)[pk]
        vids.append(dict(frame_cnt=fc, frames=pv[pk], coverage=pc[pk], best_iou=col(1, float), overlap_self=col(2, float), label=col(0, int),
                         gt_frames=gv[gk], gt_label=np.array([int(r[0]) for r in gt], np.int32)[gk]))
    return vids


def check_dataset(vids, prefix):
    g = lambda k: GOLD[prefix + "ds_" + k]
    assert same(np.array([len(v["frames"]) for v in vids], np.int32), g("count"))
    assert same(np.array([len(v["gt_frames"]) for v in vids], np.int32), g("gt_count"))
    assert same(np.array([v["frame_cnt"] for v in vids], np.int32), g("frame_cnt"))
    for k in ("frames", "coverage", "best_iou", "overlap_self", "label", "gt_frames", "gt_label"):
        assert same(np.concatenate([v[k] for v in vids]), g(k)), k
    out, stats, totals = P.proposal_targets(vids)
    assert same(np.concatenate([o["tags"] for o in out]), g("tags"))
    assert same(np.concatenate([o["reg"] for o in out]), g("reg"))            # size_reg too: math.log on both sides
    assert same(np.array([o["pools"][:3] for o in out], np.int32), g("pools"))
    assert same(stats, g("stats"))
    # the data set's pools: fg with the ground truth added (gt_as_fg), incomplete, background, videos
    assert [totals[0] + totals[3], totals[1], totals[2], totals[4]] == g("pool_totals").tolist()
    t = [P.test_proposals(v["frames"], v["frame_cnt"]) for v in vids]
    assert same(np.array([x[0] for x in t], np.int32), g("num_ticks"))
    for i, k in ((1, "rel_prop"), (2, "ticks"), (3, "scaling")):
        assert same(np.concatenate([x[i] for x in t]), g(k)), k


def test_list_text_and_what_the_dataset_reads_from_it():
    text = oracle_list_text()
    assert text == str(GOLD["rag_text"])
    vids = records(text)
    assert len(vids[1]["frames"]) == 0 and len(vids[0]["gt_frames"]) == 0 and len(vids[5]["gt_frames"]) < GOLD["rag_gt_count"][5]
    check_dataset(vids, "rag_")


def test_normalised_list():
    vids = records(str(GOLD["norm_text"]), GOLD["norm_frame_cnt"], normalised=True)
    check_dataset(vids, "norm_")
    # process_proposal_list's text: unfiltered rows of the normalised list, converted
    blocks = []
    for i, ((vid, _, gt, pr), fc) in enumerate(zip(P.parse_proposal_list(str(GOLD["norm_text"])), GOLD["norm_frame_cnt"])):
        gf, pf = P.normalised_to_frames([r[1:3] for r in gt], int(fc)), P.normalised_to_frames([r[3:5] for r in pr], int(fc))
        gts = "".join("{} {:d} {:d}\n".format(int(r[0]), int(f[0]), int(f[1])) for r, f in zip(gt, gf))
        prs = "".join("{} {:.04f} {:.04f} {:d} {:d}\n".format(int(r[0]), float(r[1]), float(r[2]), int(f[0]), int(f[1])) for r, f in zip(pr, pf))
        blocks.append("# {}\nframes/{}\n{}\n1\n{}\n{}{}\n{}".format(i, vid, int(fc), len(gt), gts, len(pr), prs))
    assert "".join(blocks) == str(GOLD["norm_processed_text"])


def test_frame_conversion_lands_on_integers():
    # 0.29 * 100.0 = 28.999999999999996 -> 28 and 0.57 * 100.0 = 56.99999999999999 -> 56: one rounded multiply, then truncation
    assert P.seconds_to_frames([(0.29, 0.57), (0.1, 0.7)], 3.0, 300).tolist() == [[28, 56], [10, 70]]
    assert P.normalised_to_frames([("0.29", "0.57")], 100).tolist() == [[28, 56]]


def test_rejected_arguments_return_before_any_launch():
    """argument validation needs no device: the library returns SSNB_EINVAL (1) and launches nothing"""
    from ssn_b200 import _lib
    lib = _lib.lib
    n0 = lib.ssnb_global_launch_count()
    one = C.c_void_p(8)                                   # a non-null pointer that is never dereferenced
    off = (C.c_int64 * 3)(0, 2, 1)                        # not ascending
    ok = (C.c_int64 * 3)(0, 1, 2)
    thr = (C.c_double * 1)(0.5)
    assert lib.ssnb_name_proposals(one, one, one, -1, 0, one, one, ok, one, 0.0, one, one, one, one, None) == 1
    assert lib.ssnb_name_proposals(one, one, one, 2, 0, one, one, off, one, 0.0, one, one, one, one, None) == 1
    assert lib.ssnb_name_proposals(one, one, one, 2, 0, one, one, ok, one, 0.0, None, one, one, one, None) == 1
    assert lib.ssnb_name_proposals(one, one, one, 2, 0, one, one, ok, one, float("nan"), one, one, one, one, None) == 1
    assert lib.ssnb_proposal_recall(one, off, one, 2, thr, 1, one, one, None) == 1
    assert lib.ssnb_proposal_recall(one, ok, one, 2, thr, 33, one, one, None) == 1
    assert lib.ssnb_proposal_recall(one, ok, one, 2, thr, 1, None, one, None) == 1
    sp, bad = (C.c_double * 1)(1.0), (C.c_double * 1)(0.0)
    assert lib.ssnb_sliding_windows(one, 1, sp, bad, 1, 1, 1, one, one, one, one, one, None) == 1
    assert lib.ssnb_sliding_windows(one, 1, sp, sp, 1, 1, -1, one, one, one, one, one, None) == 1
    assert lib.ssnb_sliding_windows(one, 1, sp, sp, 1, 1, 1, None, one, one, one, one, None) == 1
    assert lib.ssnb_proposal_frames(one, one, one, 1, 0, None, one, _lib.PROPFRAMES_SECONDS, one, None, None, None, None) == 1
    assert lib.ssnb_proposal_frames(one, one, one, 1, 0, one, one, 7, one, None, None, None, None) == 1
    assert lib.ssnb_proposal_frames(one, one, one, 1, 0, one, one, 0, None, None, None, None, None) == 1
    cfg = _lib.ProposalTargetsCfg(0.7, 0.3, 0.01, 0.02, 0.7, 1, 0)
    args = [one] * 6 + [2, one, off, one] + [one] * 5 + [one, 1 << 20, None]
    assert lib.ssnb_proposal_targets(C.byref(cfg), *args) == 1
    args[8] = ok
    args[16] = 8                                          # workspace too small
    assert lib.ssnb_proposal_targets(C.byref(cfg), *args) == 1
    assert lib.ssnb_proposal_targets_workspace_bytes(-1) == 0 and lib.ssnb_proposal_targets_workspace_bytes(3) == 120
    assert lib.ssnb_test_proposals(one, one, one, one, 1, 0, one, 0, 6, one, one, one, one, None, None, None) == 1
    assert lib.ssnb_test_proposals(one, one, one, one, 1, 0, one, 1, 6, one, None, one, one, None, None, None) == 1
    assert lib.ssnb_test_proposals(one, one, one, one, -1, 0, one, 1, 6, one, one, one, one, None, None, None) == 1
    assert b"test_proposals" in lib.ssnb_last_error(None)
    assert lib.ssnb_global_launch_count() == n0
    # the ctypes mirror of the new struct: five doubles and two int32
    assert C.sizeof(_lib.ProposalTargetsCfg) == 48 and _lib.ProposalTargetsCfg.exclude_empty.offset == 40


def test_cpu_tensors_are_refused():
    import torch
    from ops import proposal_lists as L
    z = torch.zeros(1, 2, dtype=torch.float64)
    with pytest.raises(RuntimeError):
        L.name_proposals_packed(z, torch.zeros(1, dtype=torch.int64), torch.ones(1, dtype=torch.int32), z, [0], [0, 1])
    with pytest.raises(RuntimeError):
        L.proposal_frames(z, torch.zeros(1, dtype=torch.int64), torch.ones(1, dtype=torch.int32), [10], [1.0])
    with pytest.raises(RuntimeError):
        L.test_proposals(z.long(), [1], [10])
    with pytest.raises(RuntimeError):
        L.load_proposal_list(os.devnull, device="cpu")
