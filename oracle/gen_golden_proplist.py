"""tests/golden/proplist.npz from the REAL reference (python -m oracle.gen_golden_proplist, where a checkout of the reference
exists: $SSN_REFERENCE_DIR or a directory `reference` next to this repository).

Imported unedited from the checkout: ops.detection_metrics (name_proposal, temporal_recall, get_temporal_proposal_recall),
ops.sequence_funcs.gen_exponential_sw_proposal, ops.io (dump_window_list with a stub video object and a temporary directory
of empty img_*.jpg files for its glob, load_proposal_file, process_proposal_list) and ssn_dataset (SSNVideoRecord, SSNDataSet.
_parse_prop_file / get_test_data on an instance made without __init__'s file handling).  Patches from outside only:
np.int = int (ssn_dataset.py:397) and a stand-in `transforms` module supplying the names ssn_dataset star-imports (np, math,
torch), so that PIL / torchvision are not needed.  Nothing of the reference is written to the repository except the data
slice of one shipped list.  Only data is stored."""
import contextlib
import io
import math
import os
import sys
import tempfile
import types

import numpy as np

from oracle import ref_harness

REF = ref_harness.DEFAULT_SRC
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden", "proplist.npz")
RECALL_THRESHOLDS = np.arange(0.5, 1, 0.2)              # gen_bottom_up_proposals.py:170
SW_CONFIGS = ((1, 8, 0.7), (2, 6, 0.4), (1, 8, 0.4))    # (time_step, max_level, overlap): the script's defaults first
SW_DURATIONS = (0.5, 1.0, 1.5, 7.0, 33.37, 128.0, 211.96, 755.2)
SLICE_FILE, SLICE_VIDEOS, SLICE_PROPS = "thumos14_tag_val_normalized_proposal_list.txt", 3, 40
SLICE_FRAME_CNTS = (5632, 4469, 10383)


def ragged_set(seed=7):
    """-> list of dicts(duration, frame_cnt, boxes [n, 2], gt [g, 2], gt_label [g]); the special cases come first"""
    g = np.random.RandomState(seed)
    vids = []

    def add(duration, frame_cnt, boxes, gt, labels):
        vids.append(dict(duration=float(duration), frame_cnt=int(frame_cnt), boxes=np.array(boxes, np.float64).reshape(-1, 2),
                         gt=np.array(gt, np.float64).reshape(-1, 2), gt_label=np.array(labels, np.int32).reshape(-1)))
    add(30.0, 750, [(1.0, 5.0), (7.5, 9.0)], [], [])                                         # no ground truth
    add(42.5, 1063, [], [(3.0, 9.5)], [4])                                                   # no proposals
    add(20.0, 500, [(4.0, 4.0), (9.0, 3.0), (2.0, 6.0), (25.0, 31.0), (19.5, 26.0)],         # zero-length, reversed, past the end
        [(2.0, 6.0), (18.0, 20.0)], [1, 0])                                                  # and one identical to a ground truth
    add(16.0, 480, [(4.0, 8.0), (3.0, 9.0)], [(2.0, 8.0), (4.0, 10.0), (4.5, 7.5)], [2, 5, 7])   # two ground truths at equal tIoU
    add(10.0, 300, [(1.0, 2.0), (0.1, 0.7), (3.3, 9.9), (9.9, 10.0)], [(1.0, 2.0), (3.0, 9.0)], [0, 3])  # x * 30.0 on integers
    add(7.3, 219, [(0.3, 2.9), (2.1, 7.0)], [(0.0, 0.02), (7.29, 7.4), (2.0, 7.0)], [1, 1, 2])   # ground truth that the record drops
    for _ in range(10):
        duration = float(np.round(g.uniform(20, 240), 2))
        frame_cnt = int(duration * g.choice([25.0, 29.97, 30.0]))
        ng, n = int(g.randint(1, 9)), int(g.randint(5, 120))
        c, d = g.uniform(0, duration, ng), g.uniform(1, duration / 4, ng)
        gt = np.stack([np.clip(c - d / 2, 0, duration), np.clip(c + d / 2, 0, duration)], 1)
        pc, pd = g.uniform(0, duration, n), g.uniform(0.5, duration / 3, n)
        boxes = np.stack([np.clip(pc - pd / 2, 0, None), pc + pd / 2], 1)
        k = min(n, ng)                                                                        # jittered copies of the ground truth: fg rows
        boxes[:k] = gt[:k] + g.uniform(-0.05, 0.05, (k, 2)) * (gt[:k, 1:] - gt[:k, :1])
        add(duration, frame_cnt, boxes, gt, g.randint(0, 20, ng))
    return vids


def import_reference():
    np.int = int
    stub = types.ModuleType("transforms")
    import torch
    stub.np, stub.math, stub.torch = np, math, torch
    sys.modules["transforms"] = stub
    sys.path.insert(0, REF)
    import ops.detection_metrics as DM
    import ops.io as IO
    import ops.sequence_funcs as SF
    import ssn_dataset as SD
    return DM, IO, SF, SD


class _Instance:
    def __init__(self, label, span):
        self.num_label, self.time_span = label, span


class _Video:
    def __init__(self, name, v):
        self.path, self.id, self.duration = "videos/%s.mp4" % name, name, v["duration"]
        self.instance = [_Instance(int(l), (float(a), float(b))) for l, (a, b) in zip(v["gt_label"], v["gt"])]


def dataset_outputs(SD, list_path, out, prefix):
    """the real SSNDataSet on a written list -> per-row arrays in list order (kept rows only)"""
    ds = SD.SSNDataSet.__new__(SD.SSNDataSet)
    ds.prop_file, ds.verbose, ds.exclude_empty, ds.gt_as_fg = list_path, False, True, True
    ds.fg_iou_thresh, ds.incomplete_iou_thresh, ds.bg_iou_thresh = 0.7, 0.3, 0.01
    ds.bg_coverage_thresh, ds.incomplete_overlap_thresh = 0.02, 0.7
    ds.new_length, ds.starting_ratio, ds.ending_ratio = 1, 0.5, 0.5
    with contextlib.redirect_stdout(io.StringIO()):
        ds._parse_prop_file(stats=None)
    used = {v.id for v in ds.video_list}
    records = [SD.SSNVideoRecord(p) for p in SD.load_proposal_file(list_path)]
    by_id = {v.id: v for v in ds.video_list}
    rows = {k: [] for k in ("frames", "best_iou", "overlap_self", "coverage", "label", "tags", "reg", "gt_frames", "gt_label", "rel_prop",
                            "ticks", "scaling")}
    count, gt_count, n_ticks, pools = [], [], [], []
    for rec in records:
        v = by_id.get(rec.id, rec)
        fg = {id(p) for p in v.get_fg(0.7, False)} if rec.id in used else set()
        inc, bg = v.get_negatives(0.3, 0.01, 0.02, 0.7) if rec.id in used else ([], [])
        inc, bg = {id(p) for p in inc}, {id(p) for p in bg}
        for p in v.proposals:
            rows["frames"].append((p.start_frame, p.end_frame))
            rows["best_iou"].append(p.best_iou)
            rows["overlap_self"].append(p.overlap_self)
            rows["coverage"].append(p.coverage)
            rows["label"].append(p.label)
            rows["tags"].append((1 if id(p) in fg else 0) | (2 if id(p) in inc else 0) | (4 if id(p) in bg else 0))
            rows["reg"].append(p.regression_targets if id(p) in fg else [0, 0])
        for q in v.gt:
            rows["gt_frames"].append((q.start_frame, q.end_frame))
            rows["gt_label"].append(q.label)
        count.append(len(v.proposals))
        gt_count.append(len(v.gt))
        pools.append((len(fg), len(inc), len(bg)))
        _, nt, rel, ticks, scaling = ds.get_test_data(SD.SSNVideoRecord(rec._data), 6)      # a fresh record: the call may append to it
        n_ticks.append(nt)
        rows["rel_prop"] += rel.numpy().reshape(-1, 2).tolist()
        rows["ticks"] += ticks.numpy().reshape(-1, 4).tolist()
        rows["scaling"] += scaling.numpy().reshape(-1, 2).tolist()
    shapes = dict(frames=(np.int64, 2), best_iou=(np.float64, 0), overlap_self=(np.float64, 0), coverage=(np.float64, 0), label=(np.int32, 0),
                  tags=(np.uint8, 0), reg=(np.float64, 2), gt_frames=(np.int64, 2), gt_label=(np.int32, 0), rel_prop=(np.float64, 2),
                  ticks=(np.int64, 4), scaling=(np.float64, 2))
    for k, (dt, w) in shapes.items():
        out[prefix + "ds_" + k] = np.array(rows[k], dt).reshape((-1, w) if w else (-1,))
    out[prefix + "ds_count"] = np.array(count, np.int32)
    out[prefix + "ds_gt_count"] = np.array(gt_count, np.int32)
    out[prefix + "ds_frame_cnt"] = np.array([r.num_frames for r in records], np.int32)
    out[prefix + "ds_num_ticks"] = np.array(n_ticks, np.int32)
    out[prefix + "ds_pools"] = np.array(pools, np.int32).reshape(-1, 3)
    out[prefix + "ds_stats"] = np.asarray(ds.stats, np.float64)
    out[prefix + "ds_pool_totals"] = np.array([len(ds.fg_pool), len(ds.incomp_pool), len(ds.bg_pool), len(ds.video_list)], np.int64)


def main():
    DM, IO, SF, SD = import_reference()
    out = {}
    # ---- seconds boxes -> named proposals, recall, the written list, the data set's view of it
    vids = ragged_set()
    names = ["video_%04d" % i for i in range(len(vids))]
    out["rag_duration"] = np.array([v["duration"] for v in vids])
    out["rag_frame_cnt"] = np.array([v["frame_cnt"] for v in vids], np.int32)
    out["rag_count"] = np.array([len(v["boxes"]) for v in vids], np.int32)
    out["rag_gt_count"] = np.array([len(v["gt"]) for v in vids], np.int32)
    out["rag_boxes"] = np.concatenate([v["boxes"] for v in vids])
    out["rag_gt"] = np.concatenate([v["gt"] for v in vids])
    out["rag_gt_label"] = np.concatenate([v["gt_label"] for v in vids])
    pr_list = [[tuple(map(float, b)) for b in v["boxes"]] for v in vids]
    gt_full = [[(int(l), tuple(map(float, s))) for l, s in zip(v["gt_label"], v["gt"])] for v in vids]
    gt_spans = [[x[1] for x in g] for g in gt_full]
    named = [DM.name_proposal(g, p) for g, p in zip(gt_full, pr_list)]
    flat = [r for n in named for r in n]
    out["rag_label"] = np.array([r[0] for r in flat], np.int32)
    out["rag_max_overlap"] = np.array([r[1] for r in flat], np.float64)
    out["rag_overlap_self"] = np.array([r[2] for r in flat], np.float64)
    out["rag_thresholds"] = RECALL_THRESHOLDS
    out["rag_hits"] = np.array([[DM.temporal_recall(g, p, thresh=th)[0] for th in RECALL_THRESHOLDS] for g, p in zip(gt_spans, pr_list)], np.int64)
    rec = [DM.get_temporal_proposal_recall(pr_list, gt_spans, th) for th in RECALL_THRESHOLDS]
    out["rag_recall"] = np.array(rec, np.float64)            # [n_thr, (per video, per instance)]
    with tempfile.TemporaryDirectory() as tmp:
        for name, v in zip(names, vids):
            os.makedirs(os.path.join(tmp, name))
            for i in range(v["frame_cnt"]):
                open(os.path.join(tmp, name, "img_%05d.jpg" % (i + 1)), "w").close()
        text = ""
        for i, (name, v, prs) in enumerate(zip(names, vids, named)):
            text += "# {}\n".format(i + 1) + IO.dump_window_list(_Video(name, v), prs, tmp, "img_*.jpg")
        out["rag_text"] = np.array(text.replace(tmp, "frames"))
        path = os.path.join(tmp, "list.txt")
        open(path, "w").write(text)
        dataset_outputs(SD, path, out, "rag_")
        # ---- a slice of a shipped normalised list through process_proposal_list
        groups = [g for g in IO.load_proposal_file(os.path.join(REF, "data", SLICE_FILE)) if len(g[2]) > 0][:SLICE_VIDEOS]
        norm = ""
        for i, (vid, _, gt, pr) in enumerate(groups):
            pr = pr[:SLICE_PROPS]
            norm += "# %d\n%s\n1\n1\n%d\n%s%d\n%s" % (i + 1, vid, len(gt), "".join(" ".join(x) + "\n" for x in gt), len(pr),
                                                     "".join(" ".join(x) + "\n" for x in pr))
        out["norm_text"] = np.array(norm)
        out["norm_frame_cnt"] = np.array(SLICE_FRAME_CNTS, np.int32)
        npath, ppath = os.path.join(tmp, "norm.txt"), os.path.join(tmp, "processed.txt")
        open(npath, "w").write(norm)
        frame_dict = {g[0]: ("frames/" + g[0], fc, fc) for g, fc in zip(groups, SLICE_FRAME_CNTS)}
        IO.process_proposal_list(npath, ppath, frame_dict)
        out["norm_processed_text"] = np.array(open(ppath).read())
        dataset_outputs(SD, ppath, out, "norm_")
    # ---- sliding windows
    out["sw_durations"] = np.array(SW_DURATIONS)
    out["sw_configs"] = np.array(SW_CONFIGS, np.float64)
    for c, (ts, ml, ov) in enumerate(SW_CONFIGS):
        boxes = [SF.gen_exponential_sw_proposal(types.SimpleNamespace(duration=d), time_step=ts, max_level=ml, overlap=ov) for d in SW_DURATIONS]
        out["sw%d_count" % c] = np.array([len(b) for b in boxes], np.int32)
        out["sw%d_boxes" % c] = np.array([x for b in boxes for x in b], np.float64).reshape(-1, 2)
    np.savez_compressed(GOLD, **out)
    print("wrote", GOLD, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
