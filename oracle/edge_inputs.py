"""Inputs the continuous synthetic data never produce, and the comparisons that go with them, shared by the pooling / glue
edge tests of both backbones (tests/test_gpu_glue_edges.py, tests/test_gpu_inception_v3_edges.py).  TEST INFRASTRUCTURE ONLY.

`edge_input` builds a pool op's input of dyadic values (exact in fp16, so every window is full of exact ties, +-0 among
them) with one edge case per channel in the first and the last frame: NaN at each tap of a window, NaN beside +-inf, windows
of -inf only, poison in the partial last row and column.  It needs at least 21 channels and an 8 x 8 image.
"""
import math

import torch

NAN, INF = math.nan, math.inf
DYADIC = torch.tensor([-2.0, -1.0, -0.5, -0.0, 0.0, 0.5, 1.0, 2.0])       # exact in fp16: windows full of exact ties


def edge_input(frames, c, h, w, stride, pad, gen):
    """dyadic values; per channel one edge case, in the first and the last frame (the others: plain dyadic values)"""
    x = DYADIC[torch.randint(0, len(DYADIC), (frames, c, h, w), generator=gen)]
    x[:, 0::16] = 0.5                                                      # constant: every window tied
    x[:, 1::16] = torch.where(torch.rand(x[:, 1::16].shape, generator=gen) < 0.5, -0.0, 0.0)    # +-0 only
    y0 = x0 = stride - pad                    # the window of output (1, 1): tap t reads input (y0 + t // 3, x0 + t % 3)
    for f in sorted({0, frames - 1}):
        for t in range(9):
            x[f, 2 + t, y0 + t // 3, x0 + t % 3] = NAN                   # one NaN at each of the 9 taps
        x[f, 11, y0, x0] = x[f, 11, y0 + 2, x0 + 1] = NAN                # two NaNs in one window
        x[f, 12, y0, x0 + 1], x[f, 12, y0 + 1, x0 + 2] = INF, NAN        # NaN after +inf
        x[f, 13, y0, x0], x[f, 13, y0 + 2, x0 + 2] = NAN, -INF           # NaN before -inf
        x[f, 14, y0 + 1, x0 + 1], x[f, 14, y0 + 2, x0] = INF, -INF       # +inf and -inf (average: NaN)
        x[f, 15, :5, :5] = -INF                                           # windows of -inf only, padding around some
        x[f, 15, h // 2:h // 2 + 5, w // 2:w // 2 + 5] = -INF
        x[f, 17, -1, -1], x[f, 17, -1, 0], x[f, 17, 0, -1] = NAN, INF, -INF      # poison in the last row and column
        x[f, 17, -1, w // 2], x[f, 17, h // 2, -1] = NAN, INF
        x[f, 18, -2:, -2:] = -INF                                         # (part of) the partial last window
        x[f, 19, -1, -3:] = NAN                                           # NaNs side by side in the last row
        x[f, 20, 2:7, 2:7] = INF                                          # tied +inf
    return x


def same(got, ref):
    """equal values, NaN where the other is NaN (+0 == -0)"""
    return (got == ref) | (got.isnan() & ref.isnan())


def same_bits(got, ref):
    """`same`, and the sign of every zero as well: what a bitwise copy of the selected tap gives"""
    return same(got, ref) & ((got != 0) | (torch.signbit(got) == torch.signbit(ref)))


def nonfinite_masks_equal(got, ref):
    """[NaN, +inf, -inf] masks of got equal those of ref"""
    return [bool((t(got) == t(ref)).all()) for t in (torch.isnan, torch.isposinf, torch.isneginf)]
