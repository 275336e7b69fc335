"""CPU checks of detection evaluation: the numpy oracle (oracle/eval_oracle.py) against tests/golden/eval.npz, produced
from the REAL reference's eval_detection_results.py functions and the ActivityNet toolkit's AP (oracle/gen_golden_eval.py);
the staged checker (oracle/eval_check.py) catching a planted error at every stage; the ctypes mirror of
ssnb_detect_batch_cfg; argument rejection of the workspace queries."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import eval_oracle as D
from oracle import eval_check as E
from oracle import gen_golden_eval as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "eval.npz"))


def fixture_inputs(fx):
    """the generator's inputs of one fixture, merged as the script merges them (fp32 under Python float weights)"""
    srcs, cls_scores, gt = G.synth(fx, int(GOLD[fx[0] + "_seed"]))
    n_src, weights = fx[10], fx[11]
    w = [1.0 / n_src] * n_src if weights is None else [float(x) / sum(weights) for x in weights]
    merged = {}
    for vid in srcs[0]:
        parts = [None if srcs[0][vid][i] is None else np.sum([s[vid][i] * wi for s, wi in zip(srcs, w)], axis=0) for i in (1, 2, 3)]
        merged[vid] = (srcs[0][vid][0],) + tuple(parts)
    return srcs, merged, cls_scores, gt


def oracle_run(fx, merged, cls_scores, gt):
    name, K, V, _, mode, top_k, cls_top_k, sbf, nms, thr_kind, _, _, regress, _ = fx
    dets = {}
    by_name = {os.path.splitext(os.path.basename(k))[0]: v for k, v in cls_scores.items()}
    vids = list(merged)
    for vi, vid in enumerate(vids):
        rel, act, comp, reg = merged[vid]
        classes = D.class_topk(by_name[vid], cls_top_k) if mode == "cls" else None
        out = D.video_detections_branch(rel, act, comp, reg, nms, mode, top_k, classes, sbf, regress)
        for c, rows in out.items():
            dets.setdefault(c, []).append((vi, rows))
    gt_idx = [(vids.index(v) if v in vids else -1, c, a, b) for v, c, a, b in gt]
    return dets, D.ap_table(dets, gt_idx, K, G.thresholds(thr_kind))


@pytest.mark.parametrize("fx", G.FIXTURES, ids=[f[0] for f in G.FIXTURES])
def test_oracle_reproduces_reference_detections_and_ap(fx):
    _, merged, cls_scores, gt = fixture_inputs(fx)
    dets, ap = oracle_run(fx, merged, cls_scores, gt)
    name, K = fx[0], fx[1]
    for c in range(K):
        rows = dets.get(c, [])
        got = np.concatenate([r for _, r in rows]).astype(np.float64) if rows else np.zeros((0, 5))
        vid = np.concatenate([np.full(len(r), v) for v, r in rows]) if rows else np.zeros(0, np.int64)
        assert np.array_equal(got, GOLD["%s_det_%d" % (name, c)]), (name, c)
        assert np.array_equal(vid, GOLD["%s_det_video_%d" % (name, c)]), (name, c)
        assert np.array_equal(got[:, :3], GOLD["%s_pred_%d" % (name, c)]), (name, c)
    ref = GOLD[name + "_ap"]
    assert np.array_equal(np.isnan(ap), np.isnan(ref)), name
    assert np.nanmax(np.abs(ap - ref)) <= 1e-12, name


def test_golden_covers_the_edges():
    """the fixtures reach what they were built for: NaN AP (a class without ground truth), 0 AP (a class without
    detections), zero-length boxes regressed onto [0, 0] / [1, 1] and matched to zero-length ground truth"""
    ap = GOLD["thumos_ap"]
    assert np.isnan(ap[0]).all() and (ap[19] == 0).all()
    zero = [GOLD["thumos_det_%d" % c] for c in range(20)]
    z = np.concatenate([d[(d[:, 0] == d[:, 1]) & ((d[:, 0] == 0) | (d[:, 0] == 1))] for d in zero])
    assert len(z) > 0
    # with only NaN-tIoU matches the zero-length boxes are true positives: drop them and the AP falls
    fx = G.FIXTURES[0]
    _, merged, cls_scores, gt = fixture_inputs(fx)
    dets, ap_all = oracle_run(fx, merged, cls_scores, gt)
    gt_nz = [g for g in gt if g[2] != g[3]]
    vids = list(merged)
    ap_nz = D.ap_table(dets, [(vids.index(v) if v in vids else -1, c, a, b) for v, c, a, b in gt_nz], 20, G.thresholds("thumos"))
    assert not np.allclose(np.nan_to_num(ap_all), np.nan_to_num(ap_nz))


def _planted_case(mode):
    g = np.random.RandomState(5)
    offsets = [0, 7, 7, 19, 30]
    N, K = offsets[-1], 4
    c = g.rand(N)
    d = 0.05 + 0.3 * g.rand(N)
    props = np.stack([np.clip(c - d / 2, 0, 1), np.clip(c + d / 2, 0, 1)], 1).astype(np.float32)
    act = (g.randn(N, K + 1) * 2).astype(np.float32)
    comp = g.randn(N, K).astype(np.float32)
    reg = (g.randn(N, K, 2) * 0.3).astype(np.float32)
    gt_rows = []
    for v in range(4):
        for _ in range(3):
            a = g.rand() * 0.7
            gt_rows.append((v, int(g.randint(0, K)), a, a + 0.05 + 0.2 * g.rand()))
    offs, cls, seg = [0], [], []
    for v in range(4):
        rows = [r for r in gt_rows if r[0] == v]
        offs.append(offs[-1] + len(rows))
        cls += [r[1] for r in rows]
        seg += [(r[2], r[3]) for r in rows]
    gt = {"offsets": offs, "cls": np.array(cls, np.int32), "seg": np.array(seg, np.float64)}
    kw = dict(mode=mode, nms_threshold=0.4, top_k=9 if mode == "top_k" else None,
              cls_sel=np.array([[1, 3], [0, 2], [2, 3], [0, 1]]) if mode == "cls" else None, regress=True)
    return props, act, comp, reg, offsets, gt, np.arange(0.1, 1.0, 0.1), kw


@pytest.mark.parametrize("mode", ["all", "top_k", "cls"])
def test_stage_checker_passes_the_oracle_and_names_each_planted_error(mode):
    props, act, comp, reg, offsets, gt, thr, kw = _planted_case(mode)
    args = (props, act, comp, reg, offsets)

    def run(plant=None):
        res, ap = E.standin(*args, kw["mode"], kw["nms_threshold"], gt, thr, top_k=kw["top_k"], cls_sel=kw["cls_sel"], plant=plant)
        return E.check(res, ap, *args, kw["mode"], kw["nms_threshold"], gt, thr, top_k=kw["top_k"], cls_sel=kw["cls_sel"])
    clean = run()
    clean.assert_ok()
    assert clean.stats["kept"] > 0

    def plant_at(stage):
        def f(s, x):
            if s != stage:
                return x
            if s == "combined":
                x = x.copy(); x[3, 1] *= 1.01
            elif s == "sel":
                x = x.copy(); x[[0, 1]] = x[[1, 0]]
            elif s == "dets":
                d, cnt = x
                cnt = cnt.copy(); d = d.copy()
                v, c = np.argwhere(cnt > 0)[0]
                cnt[v, c] -= 1                            # one survivor lost
                return d, cnt
            elif s == "boxes":
                x = x.copy(); x[0, 0] += 1e-3
            elif s == "rank":
                x = x.copy(); i = np.nonzero(x >= 0)[0][:2]; x[i] = x[i[::-1]]
            elif s == "tp":
                x = x.copy(); i = np.nonzero(x[0] != 255)[0][0]; x[0, i] ^= 1
            elif s == "ap":
                x = x.copy(); x[np.isfinite(x)] += 1e-9
            return x
        return f
    for stage, expect in (("combined", "combined"), ("sel", "select"), ("dets", "nms"), ("boxes", "boxes"), ("rank", "rank"),
                          ("tp", "tp"), ("ap", "ap")):
        failed = run(plant_at(stage)).failed()
        assert expect in failed, (stage, failed)
        first = min(E.STAGES.index(s) for s in failed)
        assert E.STAGES[first] == expect, (stage, failed)


def test_header_mirror_of_detect_batch_cfg(tmp_path):
    """ssnb_detect_batch_cfg compiles as C99 and the ctypes mirror has its size and field offsets"""
    from ssn_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\}\s*ssnb_detect_batch_cfg;", hdr).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [d.strip().split(None, 1)[1].strip() for d in body.split(";") if d.strip()]
    prints = ['printf("size %zu\\n", sizeof(ssnb_detect_batch_cfg));']
    prints += ['printf("%s %%zu\\n", offsetof(ssnb_detect_batch_cfg, %s));' % (n, n) for n in names]
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssnb.h"\nint main(void) { %s return 0; }\n' % " ".join(prints))
    exe = tmp_path / "abi"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    lay = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    M = _lib.DetectBatchCfg
    assert int(lay["size"]) == C.sizeof(M)
    assert [n for n, _ in M._fields_] == names
    for n in names:
        assert getattr(M, n).offset == int(lay[n]), n


def test_workspace_queries_reject_bad_arguments():
    from ssn_b200._lib import lib, DetectBatchCfg, DET_ALL, DET_TOPK, DET_CLS
    offs = (C.c_int64 * 3)(0, 5, 9)
    bad = [(DetectBatchCfg(DET_TOPK, 0, 0, 0, 1, 0, 0.5), 4, offs, 2),      # top_k < 1
           (DetectBatchCfg(DET_CLS, 0, 5, 0, 1, 0, 0.5), 4, offs, 2),       # n_sel > K
           (DetectBatchCfg(7, 1, 1, 0, 1, 0, 0.5), 4, offs, 2),             # unknown mode
           (DetectBatchCfg(DET_ALL, 0, 0, 0, 1, 0, float("nan")), 4, offs, 2),
           (DetectBatchCfg(DET_ALL, 0, 0, 0, 1, 0, 0.5), 0, offs, 2),       # K = 0
           (DetectBatchCfg(DET_ALL, 0, 0, 0, 1, 0, 0.5), 4, (C.c_int64 * 3)(0, 5, 3), 2)]   # decreasing offsets
    for cfg, K, o, V in bad:
        assert lib.ssnb_detect_batch_workspace_bytes(C.byref(cfg), K, o, V) == 0
    for args in ((0, 4, 10, 5, 9), (2, 0, 10, 5, 9), (2, 2000, 10, 5, 9), (2, 4, -1, 5, 9), (2, 4, 10, 5, 0), (2, 4, 10, 5, 65)):
        assert lib.ssnb_detection_ap_workspace_bytes(*args) == 0
