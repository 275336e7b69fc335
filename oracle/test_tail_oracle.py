"""Numpy restatement of the packed test-time tail (ssnb_stpp_reorg_batch, ops.ssn_ops.reorg_packed).  TEST INFRASTRUCTURE ONLY.

ssn_test.py:87-92 per video: STPPReorgainzed.forward on the video's [T_v, D] tick scores (reorg64 of oracle/infer_check.py,
float64), then the regression de-normalisation by the checkpoint's reg_stats, which torch runs as two fp32 ops per column,
each rounded on its own: fp32(fp32(x * (float)std) + (float)mean), column 0 of a class pair location, column 1 size."""
import numpy as np
import torch

from .infer_check import reorg64


def reorg_packed64(scores, tick_offsets, ticks, scaling, offsets, act_len, comp_len, reg_len, stpp_cfg):
    """every video of a packed batch through reorg64 -> (act, comp, reg) float64 [sum N, .] in the packed row order"""
    scores = torch.as_tensor(scores)
    ticks, scaling = torch.as_tensor(ticks).reshape(-1, 4), torch.as_tensor(scaling).reshape(-1, 2)
    outs = [[], [], []]
    for v in range(len(offsets) - 1):
        t0, t1, r0, r1 = int(tick_offsets[v]), int(tick_offsets[v + 1]), int(offsets[v]), int(offsets[v + 1])
        if r1 == r0:
            continue
        for o, r in zip(outs, reorg64(scores[t0:t1], ticks[r0:r1], scaling[r0:r1], act_len, comp_len, reg_len, stpp_cfg)):
            o.append(r)
    return tuple(torch.cat(o) if o else torch.zeros(0, L, dtype=torch.float64)
                 for o, L in zip(outs, (act_len, comp_len, reg_len)))


def denorm32(reg, reg_stats):
    """reg [n, 2K] or [n, K, 2] (fp32 values), reg_stats [2, 2] (means, then stds) -> [n, K, 2] float32 as ssn_test.py:90-92"""
    r = np.array(reg, dtype=np.float32).reshape(len(reg), -1, 2)
    st = np.asarray(reg_stats, dtype=np.float64)
    for c in (0, 1):
        r[:, :, c] = (r[:, :, c] * np.float32(st[1, c])) + np.float32(st[0, c])
    return r
