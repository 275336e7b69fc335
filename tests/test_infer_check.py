"""oracle/infer_check.py on the CPU: the float64 restatement of the test-time tail against numpy, the fp32 oracle and the
golden fixtures, and the comparator against planted errors -- each reported at its own op and quantity, and only there."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle import detect_oracle as D
from oracle import infer_check as IC
from oracle import ssn_oracle as O

CPU_BAR = 1e-5           # fp32 stand-ins against float64 (fp32 sums of up to a few hundred rows)
NPOT_CFG = ((1, 3), (1, 2, 3, 5), (1, 6))


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name), allow_pickle=False)


# ---- reorg_ticks: numpy's arange fill rule ---------------------------------------------------------------------------------
def _naive_ticks(left, right, n_part):
    step = (right - left) / n_part
    return [int(left + q * step) for q in range(n_part + 1)]


def test_reorg_ticks_equal_numpy_arange():
    """left 0..599, span 1..199, n_part 3, 5, 6, 7: reorg_ticks is np.arange's boundaries (ops/ssn_ops.py:144-147), and
    left + q * step -- what the re-organised STPP kernels used to compute -- is not, at 164 397 of the 2 985 000"""
    bad = 0
    for n_part in (3, 5, 6, 7):
        for left in range(600):
            for span in range(1, 200):
                right = left + span
                want = [int(v) for v in np.arange(left, right + 1e-5, (right - left) / n_part)[:n_part + 1]]
                assert IC.reorg_ticks(left, right, n_part) == want, (left, right, n_part)
                bad += sum(a != b for a, b in zip(_naive_ticks(left, right, n_part), want))
    assert bad == 164397
    # numpy ends the last of three parts of [1, 2) at 1 (1.9999999999999998): every part is empty
    assert IC.reorg_ticks(1, 2, 3) == [1, 1, 1, 1] and _naive_ticks(1, 2, 3) == [1, 1, 1, 2]


def test_reorg_ticks_powers_of_two_are_exact():
    for n_part in (1, 2, 4, 8):
        for left in range(0, 700, 7):
            for span in range(1, 260):
                assert IC.reorg_ticks(left, left + span, n_part) == _naive_ticks(left, left + span, n_part)


# ---- reorg64 against the fp32 oracle and the golden fixture -----------------------------------------------------------------
@pytest.mark.parametrize("cfg", [(1, (1, 2), 1), NPOT_CFG])
def test_reorg64_matches_fp32_oracle(cfg):
    g = torch.Generator().manual_seed(41)
    K, T, N = 3, 90, 120
    mult = sum(sum(O.parse_stage_config(c)[0]) for c in cfg)
    scores = torch.randn(T, (K + 1) + mult * 3 * K, generator=g)
    ticks = torch.sort(torch.randint(-3, T + 3, (N, 4), generator=g), dim=1)[0]
    sc = torch.rand(N, 2, generator=g)
    ref = IC.reorg64(scores, ticks, sc, K + 1, K, 2 * K, cfg)
    assert any(torch.isnan(r).any() for r in ref)          # ticks beyond T give empty activity slices
    chk = IC.Checker()
    IC.check_reorg(chk, "reorg", scores, ticks, sc, K + 1, K, 2 * K, cfg,
                   O.stpp_reorganized(scores, ticks, sc, K + 1, K, 2 * K, cfg), bar=CPU_BAR, ref=ref)
    chk.assert_ok()


@pytest.mark.parametrize("tag,cfg", [("flat", (1, 1, 1)), ("pyr", (1, (1, 2), 1))])
def test_reorg64_matches_golden(golden_dir, tag, cfg):
    z = _golden(golden_dir, "test_path.npz")
    K = 3
    chk = IC.Checker()
    IC.check_reorg(chk, "reorg " + tag, torch.tensor(z[tag + "_scores"]), torch.tensor(z[tag + "_ticks"]),
                   torch.tensor(z[tag + "_sc"]), K + 1, K, 2 * K, cfg,
                   tuple(torch.tensor(z[tag + k]) for k in ("_act", "_comp", "_reg")), bar=CPU_BAR)
    chk.assert_ok()


def test_dataset_ticks():
    """ssn_dataset.py:406-428 on proposals touching 0 and 1: the augmented span clipped to the video, its scaling below 1"""
    ticks, sc = IC.dataset_ticks([[0.0, 0.2], [0.4, 0.6], [0.9, 1.0]], 100)
    assert ticks.tolist() == [[0, 0, 20, 30], [30, 40, 60, 70], [85, 90, 100, 100]]
    np.testing.assert_allclose(sc.numpy(), [[0.0, 1.0], [1.0, 1.0], [1.0, 0.0]], atol=1e-12)


# ---- detection ---------------------------------------------------------------------------------------------------------------
def test_nms64_regress64_reproduce_detect_golden(golden_dir):
    """detect.npz (the reference's own temporal_nms / perform_regression): survivors and order exactly, the regressed boxes
    to fp32 rounding"""
    z = _golden(golden_dir, "detect.npz")
    for tag in "abcd":
        props, comb, reg, thr = z[tag + "_props"], z[tag + "_combined"], z[tag + "_reg"], float(z[tag + "_thr"])
        for c in range(comb.shape[1]):
            k = IC.nms64(props, comb[:, c], thr)
            rows = np.concatenate((props[k], comb[k, c][:, None], reg[k, c]), 1)
            np.testing.assert_array_equal(rows, z["%s_nms_%d" % (tag, c)])
            det = z["%s_det_%d" % (tag, c)]
            box = IC.regress64(props[k], reg[k, c, 0], reg[k, c, 1]).numpy()
            assert np.abs(det[:, :2] - box).max() <= 2e-7, (tag, c)


def test_nms_order():
    """NaN first like argsort()[::-1]; ties larger index first like argsort(kind="stable")[::-1]"""
    g = np.random.default_rng(5)
    fixtures = [np.array([0.5, np.nan, 0.2], np.float32)]
    for n in (2, 7, 33, 300):
        s = g.permutation(n).astype(np.float32) / n - 0.5
        s[g.integers(n)] = np.nan
        fixtures.append(s)
    for s in fixtures:
        np.testing.assert_array_equal(IC.nms_order(s), s.argsort()[::-1])
    assert IC.nms_order(fixtures[0]).tolist() == [1, 0, 2]
    ties = g.integers(0, 4, 500).astype(np.float32)
    ties[g.integers(0, 500, 20)] = np.nan
    ties[g.integers(0, 500, 20)] = -np.inf
    pad = np.full(40, -np.inf, np.float32)
    pad[3] = np.nan
    pad[10:20] = 1.0
    for s in (ties, pad, np.zeros(64, np.float32), np.array([0.0, -0.0, 0.0], np.float32)):
        np.testing.assert_array_equal(IC.nms_order(s), s.argsort(kind="stable")[::-1])


def test_nms64_threshold_is_inclusive():
    """IoU exactly at the threshold (dyadic boxes): kept; zero-duration boxes give 0 / 0 and are dropped like numpy's"""
    props = np.array([[0, 0.5], [0, 0.25], [0.25, 0.75], [0.5, 0.5], [0.5, 0.5]], np.float32)
    assert IC.nms64(props, [0.9, 0.8, 0.7, 0.6, 0.5], 0.5).tolist() == [0, 1, 2, 3]
    assert IC.nms64(props, [0.9, 0.8, 0.7, 0.6, 0.5], 0.4).tolist() == [0, 2, 3]


# ---- planted errors ---------------------------------------------------------------------------------------------------------
def _nms_idx(det, thr, strict=False, nan_last=False):
    """ops/utils.py:56-82 (oracle/detect_oracle.temporal_nms) returning the kept indices, with two planted variants"""
    t1, t2, scores = det[:, 0], det[:, 1], det[:, 2]
    durations = t2 - t1
    order = scores.argsort()[::-1]
    if nan_last:
        order = np.concatenate((order[~np.isnan(scores[order])], order[np.isnan(scores[order])]))
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        tt1 = np.maximum(t1[i], t1[order[1:]])
        tt2 = np.minimum(t2[i], t2[order[1:]])
        inter = tt2 - tt1
        iou = inter / (durations[i] + durations[order[1:]] - inter).astype(float)
        order = order[np.where(iou < thr if strict else iou <= thr)[0] + 1]
    return np.array(keep, dtype=np.int64)


@functools.lru_cache(maxsize=None)
def _fixture():
    g = torch.Generator().manual_seed(77)
    f = {}
    # crop mean: 4 crops x 6 ticks, 50 -> 9
    f["feat"], f["w"], f["b"] = torch.randn(24, 50, generator=g), torch.randn(9, 50, generator=g), torch.randn(9, generator=g)
    # re-organised STPP with non-power-of-two part counts over spans 1..60
    K, T = 2, 120
    mult = sum(sum(O.parse_stage_config(c)[0]) for c in NPOT_CFG)
    f["scores"] = torch.randn(T, (K + 1) + mult * 3 * K, generator=g) + 0.5
    rows = [(l - 2, l, l + s, l + s + 3) for s in range(1, 61) for l in (1, 37)]
    f["ticks"] = torch.tensor(rows)
    f["sc"] = torch.rand(len(rows), 2, generator=g)
    # a long video: T = 20000, scores offset by +30, short parts late in the video
    TL = 20000
    f["long_scores"] = torch.randn(TL, 2 + 5 * 3, generator=g) + 30
    lt = torch.sort(torch.randint(TL - 400, TL, (30, 4), generator=g), dim=1)[0]
    f["long_ticks"], f["long_sc"] = lt, torch.rand(30, 2, generator=g)
    # detection: dyadic boxes (exact IoU ties with the threshold), a NaN act row, regressions beyond [0, 1]
    N, Kd = 48, 3
    st = torch.randint(0, 48, (N,), generator=g).float() / 64
    f["props"] = torch.stack([st, st + torch.randint(1, 17, (N,), generator=g).float() / 64], 1).numpy()
    f["props"][:4] = [[0, 0.5], [0, 0.25], [0.25, 0.75], [0.5, 0.5]]
    act = torch.randn(N, Kd + 1, generator=g)
    act[0] += 3
    act[5] = float("nan")
    f["act"], f["comp"] = act.numpy(), (torch.randn(N, Kd, generator=g) * 0.5).numpy()
    f["reg"] = (torch.randn(N, Kd, 2, generator=g) * 0.6).numpy()
    f["thr"] = 0.5
    ref = {"reorg": IC.reorg64(f["scores"], f["ticks"], f["sc"], K + 1, K, 2 * K, NPOT_CFG),
           "long": IC.reorg64(f["long_scores"], f["long_ticks"], f["long_sc"], 2, 1, 2, (1, (1, 2), 1))}
    return f, ref


def _fp32_prefix_mean(src, pl, pr):
    """the column prefix of the re-organised STPP kept in fp32: (P[b] - P[a]) / (b - a)"""
    a, b, _ = slice(pl, pr).indices(src.shape[0])
    if b <= a:
        return np.full(src.shape[1], np.nan)
    P = np.concatenate([np.zeros((1, src.shape[1]), np.float32), np.cumsum(src.astype(np.float32), 0, dtype=np.float32)])
    return ((P[b] - P[a]) / np.float32(b - a)).astype(np.float64)


PLANTED = {
    "none": set(),
    "ticks_left_plus_q_step": {("reorg", "comp"), ("reorg", "reg")},
    "crop_mean_over_crops_minus_1": {("cropmean", "y")},
    "nms_strict_less": {("detect", "order")},
    "nan_ranked_last": {("detect", "order")},
    "activity_mean_inclusive": {("reorg", "act")},
    "regression_unclipped": {("detect", "boxes")},
    "fp32_column_prefix": {("reorg T=20000", "act"), ("reorg T=20000", "comp"), ("reorg T=20000", "reg")},
}


@pytest.mark.parametrize("plant", sorted(PLANTED))
def test_planted_error_reported_at_its_op(plant, monkeypatch):
    """stand-ins built from the fp32 oracle (ssn_oracle.stpp_reorganized, detect_oracle, an fp32 crop mean) pass every check
    at CPU_BAR; with one error planted, exactly the checks of that op and quantity fail"""
    f, ref = _fixture()
    chk = IC.Checker()
    # crop mean
    x = f["feat"].view(4, 6, -1)
    xm = x[:3].mean(0) if plant == "crop_mean_over_crops_minus_1" else x.mean(0)
    IC.check_cropmean(chk, "cropmean", f["feat"], f["w"], f["b"], 4, xm @ f["w"].T + f["b"], bar=CPU_BAR)
    # re-organised STPP
    args = (f["scores"], f["ticks"], f["sc"], 3, 2, 4, NPOT_CFG)
    if plant == "ticks_left_plus_q_step":
        with monkeypatch.context() as m:
            m.setattr(IC, "reorg_ticks", _naive_ticks)
            outs = tuple(t.float() for t in IC.reorg64(*args))
    else:
        outs = O.stpp_reorganized(*args)
    if plant == "activity_mean_inclusive":
        outs = (torch.stack([f["scores"][t1:max(t1 + 1, t2) + 1, :3].mean(0) for t1, t2 in f["ticks"][:, 1:3].tolist()]),) + outs[1:]
    IC.check_reorg(chk, "reorg", *args, outs, bar=CPU_BAR, ref=ref["reorg"])
    largs = (f["long_scores"], f["long_ticks"], f["long_sc"], 2, 1, 2, (1, (1, 2), 1))
    if plant == "fp32_column_prefix":
        with monkeypatch.context() as m:
            m.setattr(IC, "_mean_rows", _fp32_prefix_mean)
            outs = tuple(t.float() for t in IC.reorg64(*largs))
    else:
        outs = O.stpp_reorganized(*largs)
    IC.check_reorg(chk, "reorg T=20000", *largs, outs, bar=CPU_BAR, ref=ref["long"])
    # detection
    props, act, comp, reg, thr = f["props"], f["act"], f["comp"], f["reg"], f["thr"]
    combined = D.softmax(act)[:, 1:] * np.exp(comp)
    kept, dets = [], []
    for c in range(comp.shape[1]):
        det = np.concatenate((props, combined[:, c][:, None], reg[:, c]), 1)
        k = _nms_idx(det, thr, strict=plant == "nms_strict_less", nan_last=plant == "nan_ranked_last")
        if plant == "none":
            np.testing.assert_array_equal(det[k], D.temporal_nms(det, thr))
        rows = det[k]
        if plant == "regression_unclipped":
            ctr, dur = (rows[:, 0] + rows[:, 1]) / 2, rows[:, 1] - rows[:, 0]
            nc, nd = ctr + dur * rows[:, 3], dur * np.exp(rows[:, 4])
            rows = np.concatenate(((nc - nd / 2)[:, None], (nc + nd / 2)[:, None], rows[:, 2:]), 1)
        else:
            rows = D.perform_regression(rows)
        kept.append(k)
        dets.append(rows)
    IC.check_detect(chk, "detect", props, combined, thr, kept, dets, reg, act, comp, bar=CPU_BAR, combined_bar=CPU_BAR)
    assert chk.failed() == PLANTED[plant], chk.report()
