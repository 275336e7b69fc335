"""CPU checks of the float64 restatements in oracle/train_loop_oracle.py that tests/test_gpu_update_block.py holds the
device kernels to: top-1 and the meters against the torch-based accuracy() and the reference's own numbers
(tests/golden/train_loop.npz), hand-worked ties, NaN and signed zeros, the odd-row rule, the micro-batch schedule, and the
norm / clip / SGD rules against the reference's update blocks."""
import os

import numpy as np
import pytest
import torch

from oracle import train_loop_oracle as TL


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "train_loop.npz"))


def _ulps(got, want):
    """distance in fp32 units in the last place, elementwise"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return np.abs(got.astype(np.float64) - want.astype(np.float64)) / np.spacing(np.abs(want)).astype(np.float64)


def test_top1_matches_torch_accuracy_on_tie_free_scores():
    g = torch.Generator().manual_seed(0)
    for rows, cols in ((1, 1), (7, 2), (64, 21), (300, 201), (33, 1000)):
        s = torch.randn(rows, cols, generator=g)
        assert np.array_equal(TL.top1(s.numpy()), s.topk(1, 1)[1].view(-1).numpy())
        t = torch.randint(0, cols, (rows,), generator=g)
        t[::2] = s[::2].argmax(1)
        buf = TL.meters_update(np.zeros((3, 2)), s.numpy(), t.numpy(), None, [], 1.0)
        assert np.float32(buf[0, 0] / buf[0, 1]) == TL.accuracy(s, t).numpy()


def test_top1_hand_worked():
    nan, inf = np.float32("nan"), np.float32("inf")
    s = np.array([[1, 3, 3, 2],              # equal maxima: the lower index
                  [nan, 5, nan, 1],          # NaN above every number, NaN against NaN: the lower index
                  [1, 2, 3, nan],
                  [-0.0, 0.0, -1, -2],       # -0 == +0
                  [0.0, -0.0, -1, -2],
                  [-inf, -inf, -inf, -inf],  # all equal
                  [1, inf, inf, -inf]], np.float32)
    assert TL.top1(s).tolist() == [1, 0, 3, 0, 0, 0, 1]
    # maxima tied across the kernel's lanes: column c, c + 32 and c + 64 of a 96-column row
    row = np.zeros((1, 96), np.float32)
    row[0, [70, 38, 6]] = 4.0
    assert TL.top1(row).tolist() == [6]


def test_meters_hand_worked_and_odd_rows():
    # 8 rows, every score equal: class 0 everywhere; targets make 4 of 8 correct, 3 of the 4 fg and 1 of the 4 bg
    buf = TL.meters_update(np.zeros((4, 2)), np.zeros((8, 2), np.float32), np.array([0, 1, 0, 1, 1, 0, 0, 1]), None,
                           [0.5], 4.0)
    assert buf.tolist() == [[2.0, 4.0], [400.0, 8.0], [300.0, 4.0], [100.0, 4.0]]
    # prop_type: only types 0 and 2 count, in order; 5 of them is odd: the fifth counts in act_acc only
    pt = np.array([0, 1, 2, 1, 1, 0, 2, 1, 0])
    tg = np.array([0, 9, 0, 9, 9, 1, 1, 9, 0])
    buf = TL.meters_update(np.zeros((3, 2)), np.zeros((9, 2), np.float32), tg, pt, [], 1.0)
    # activity rows: targets 0 0 1 1 0 -> correct 1 1 0 0 1; pairs (1, 1), (0, 0); the unpaired last row is correct
    assert buf[0].tolist() == [float(np.float32(3) * np.float32(100.0 / 5)) * 5, 5.0]
    assert buf[1].tolist() == [100.0, 2.0] and buf[2].tolist() == [100.0, 2.0]
    # one activity row: no pair, fg and bg untouched
    buf = TL.meters_update(np.zeros((3, 2)), np.zeros((1, 3), np.float32), np.array([0]), None, [], 1.0)
    assert buf.tolist() == [[100.0, 1.0], [0.0, 0.0], [0.0, 0.0]]
    # the reference itself refuses an odd count
    with pytest.raises(RuntimeError):
        TL._update_acc(TL.new_meters(("act_acc", "fg_acc", "bg_acc")), torch.zeros(3, 2), torch.zeros(3, dtype=torch.long))


@pytest.mark.parametrize("tag", ["ssn", "binary"])
def test_meters_match_reference_golden(gold, tag):
    buf = np.zeros((3, 2))
    for step in range(3):
        p = "%s_acc%d_" % (tag, step)
        before = buf.copy()
        TL.meters_update(buf, gold[p + "scores"], gold[p + "target"], None, [], 1.0)
        n = buf[:, 1] - before[:, 1]
        vals = np.array([(buf[k, 0] - before[k, 0]) / n[k] for k in range(3)], np.float32)
        assert vals.tobytes() == gold[p + "vals"].tobytes()
    assert buf.tobytes() == gold[tag + "_meters"].tobytes()


def test_schedule():
    assert TL.step_schedule(3, 1) == [True, True, True]
    assert TL.step_schedule(7, 3) == [True, False, False, True, False, False, True]
    assert [i for i, s in enumerate(TL.step_schedule(10, 4)) if s] == [0, 4, 8]


def test_clip_rule():
    assert TL.clip_coef(2.0, 1.0) == 1.0 / (2.0 + 1e-6)
    assert TL.clip_coef(1.0, 1.0) == 1.0 / (1.0 + 1e-6)          # norm == max_norm still clips, by 1e-6
    assert TL.clip_coef(0.5, 1.0) is None
    assert TL.clip_coef(3.0, 0.0) == 0.0 and TL.clip_coef(0.0, 0.0) == 0.0
    assert TL.clip_coef(float("nan"), 1.0) is None
    assert TL.clip_coef(float("inf"), 1.0) == 0.0
    assert TL.clip_coef(1e30, float("inf")) is None
    g = np.array([1.0, -3.0, 0.1], np.float32)
    c = TL.clip_coef(7.0, 2.0)
    assert TL.clipped_grad(g, 1.0, c).tobytes() == (g * np.float32(np.float32(1.0) * np.float32(c))).tobytes()
    assert TL.clipped_grad(g, 1 / 3, None).tobytes() == (g * np.float32(1 / 3)).tobytes()


def test_grad_norm64():
    g = np.array([3.0, 4.0], np.float32)
    assert TL.grad_norm64(g, 1.0) == 5.0
    assert TL.grad_norm64(g * 2, 0.5, [np.array([12.0], np.float32)]) == 13.0
    assert TL.grad_norm64(np.full(4, 3e38, np.float32), 1.0) > float(np.finfo(np.float32).max)
    assert np.isnan(TL.grad_norm64(np.array([1.0, np.nan], np.float32), 1.0))
    assert TL.grad_norm64(np.zeros(0, np.float32), 1.0, [np.zeros(0, np.float32)]) == 0.0


@pytest.mark.parametrize("tag", ["ssn", "binary"])
@pytest.mark.parametrize("case", range(5))
def test_update_block_rules_match_reference(gold, tag, case):
    """the reference divides by iter_size and then multiplies by c; the rules above multiply once by fl(fl(1/iter_size) *
    fl(c)): with the reference's c the gradients it sees within 2 ulp; its norm and parameters within 1e-6.  The device
    forms c from its fp32 norm: that c is within 1 ulp of the reference's (so the gradients the device sees are within
    3 ulp of the reference's: tests/test_gpu_update_block.py holds them bitwise to clipped_grad at the device's norm)"""
    p = "%s_upd%d_" % (tag, case)
    iter_size, clip = gold[p + "cfg"]
    clip = None if np.isnan(clip) else float(clip)
    grads = [gold[p + "grad%d" % j].reshape(-1) for j in range(3)]
    params = [gold[p + "param%d" % j].reshape(-1) for j in range(3)]
    extra = gold[p + "grad3"].reshape(-1)
    sizes = [len(g) for g in grads]
    flat_g, flat_p = np.concatenate(grads), np.concatenate(params)
    gm = 1.0 / iter_size
    c = None
    if clip is not None:
        norm = TL.grad_norm64(flat_g, gm, [extra])
        assert abs(norm - gold[p + "total_norm"]) <= 1e-6 * gold[p + "total_norm"]
        c = TL.clip_coef(gold[p + "total_norm"], clip)
        c32 = TL.clip_coef(np.float32(norm), clip)
        assert (c is None) == (c32 is None)
        if c is not None:
            assert _ulps(c32, c) <= 1
    seen = TL.clipped_grad(flat_g, gm, c)
    want_seen = np.concatenate([gold[p + "seen%d" % j].reshape(-1) for j in range(3)])
    assert _ulps(seen, want_seen).max() <= 2
    assert _ulps(TL.clipped_grad(extra, 1.0, c), gold[p + "extra_after"]).max() <= 2
    ends = np.cumsum(sizes)
    new_p, _b, _ps, _bs = TL.sgd64(flat_p, flat_g, np.zeros_like(flat_p), ends, [0.1, 0.1, 0.2], [5e-4, 5e-4, 0.0], 0.9, gm, c)
    want_p = np.concatenate([gold[p + "param_after%d" % j].reshape(-1) for j in range(3)])
    assert np.abs(new_p - want_p).max() <= 1e-6 * np.abs(want_p).max()
