"""tests/golden/test_tail.npz from the REAL reference (build container only: python -m oracle.gen_golden_test_tail).

The reference's STPPReorgainzed (ops/ssn_ops.py) is imported through oracle/ref_harness.py (vendored from a checkout of the
reference, patches 1-4; patch 4 lets its hard-coded .cuda() run on the CPU).  ssn_test.py is a script that does not import
on Python 3.12, so lines 87-92 of its worker loop -- the forward call and the two de-normalisation lines -- are compiled from
the script's own source text with ast, the reference's code unedited, and run in a namespace holding the loop's locals
(reorg_stpp, output, prop_ticks, prop_scaling, num_class, stats).

Each fixture set is one batch (one K and one stpp_cfg); together they hold ten ragged videos: T = 1, a video with only the
fallback proposal (0, frame_cnt - 1), ssn_dataset.py ticks touching 0 and T, negative ticks, K = 20 and K = 200, the configs
(1,(1,2),1) and ((1,3),(1,2,3,5),(1,6)), and a reg_stats with non-dyadic values.  The block runs twice: with torch's
default dtype float64 (the pooling in float64, against which the oracle is held to 1e-12) and as the script runs, in fp32
(the de-normalisation, held bitwise; the forward's raw fp32 reg is recorded before the two lines modify it in place)."""
import ast
import os

import numpy as np
import torch

from . import ref_harness
from .infer_check import dataset_ticks

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
NPOT_CFG = ((1, 3), (1, 2, 3, 5), (1, 6))
REG_STATS = np.array([[0.0123, -0.0457], [0.1789, 0.2345]])

# set name -> (K, stpp_cfg, [(T, kind, n)]): kind 'dataset' = ssn_dataset.py ticks of n proposals, some touching 0 and 1;
# 'fallback' = the single fallback proposal; 'raw' = n sorted tick rows drawn from [-3, T + 3]
SETS = {
    "a": (20, (1, (1, 2), 1), [(1, "dataset", 3), (90, "fallback", 1), (60, "dataset", 40), (120, "raw", 50)]),
    "b": (200, (1, (1, 2), 1), [(12, "dataset", 10), (1, "raw", 2), (16, "dataset", 12)]),
    "c": (20, NPOT_CFG, [(80, "dataset", 50), (7, "raw", 12), (1, "fallback", 1)]),
}


def _lens(K):
    return K + 1, K, 2 * K


def _D(K, cfg):
    from .ssn_oracle import parse_stage_config
    return K + 1 + sum(sum(parse_stage_config(c)[0]) for c in cfg) * 3 * K


def _video(T, kind, n, g):
    """-> ticks int64 [n, 4], scaling float64 [n, 2]"""
    if kind == "fallback":                             # ssn_dataset.py:398-401: (0, frame_cnt - 1) of a video without proposals
        frame_cnt = T * 6 + 1
        return dataset_ticks(np.array([[0.0, (frame_cnt - 1) / frame_cnt]]), T)
    if kind == "raw":
        return torch.sort(torch.from_numpy(g.randint(-3, T + 4, (n, 4))), 1)[0], torch.from_numpy(g.rand(n, 2))
    st = g.rand(n) * 0.9
    ed = np.minimum(st + g.rand(n) * 0.5 + 0.01, 1.0)
    st[:3], ed[3:6] = 0.0, 1.0
    return dataset_ticks(np.stack([st, ed], 1), T)


def tail_block():
    """ssn_test.py:87-92 (the forward call and the de-normalisation) compiled from the script's source text"""
    src = open(os.path.join(ref_harness.DEFAULT_SRC, "ssn_test.py")).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "runner_func"][0]
    loop = [n for n in fn.body if isinstance(n, ast.While)][0]
    first = [i for i, n in enumerate(loop.body) if isinstance(n, ast.Assign) and "reorg_stpp.forward" in ast.unparse(n.value)][0]
    body = loop.body[first:first + 2]                  # the assignment and `if reg_scores is not None:` with its three lines
    assert isinstance(body[1], ast.If) and len(body[1].body) == 3, ast.unparse(ast.Module(body=body, type_ignores=[]))
    return compile(ast.Module(body=body, type_ignores=[]), "ssn_test.py", "exec")


class _Recording:
    """the reference's STPPReorgainzed, keeping a copy of what forward returned before the caller edits it in place"""

    def __init__(self, inner):
        self.inner, self.raw = inner, None

    def forward(self, *a):
        out = self.inner.forward(*a)
        self.raw = [x.clone() for x in out]
        return out


def main():
    if not ref_harness.vendor():
        raise SystemExit("no checkout of the reference at %s (set SSN_REFERENCE_DIR)" % ref_harness.DEFAULT_SRC)
    _, R = ref_harness.import_reference()
    code = tail_block()
    g = np.random.RandomState(2026)
    out = {"reg_stats": REG_STATS}
    for name, (K, cfg, videos) in SETS.items():
        D = _D(K, cfg)
        toff, off, scores, ticks, scaling = [0], [0], [], [], []
        per = {"act64": [], "comp64": [], "reg64": [], "reg_raw32": [], "reg32": []}
        for T, kind, n in videos:
            tk, sc = _video(T, kind, n, g)
            s = (np.round(g.randn(T, D) * 1024) / 1024 + 0.5).astype(np.float32)    # multiples of 2^-10: a small file
            for dtype in (torch.float64, torch.float32):
                torch.set_default_dtype(dtype)
                try:
                    reorg = _Recording(R.STPPReorgainzed(D, K + 1, K, 2 * K, True, stpp_cfg=cfg))
                    ns = {"reorg_stpp": reorg, "output": torch.from_numpy(s).to(dtype), "prop_ticks": tk.clone(),
                          "prop_scaling": sc.clone(), "num_class": K, "stats": REG_STATS}
                    exec(code, ns)
                finally:
                    torch.set_default_dtype(torch.float32)
                if dtype == torch.float64:
                    for k, x in zip(("act64", "comp64", "reg64"), reorg.raw):
                        per[k].append(x.numpy())
                else:
                    per["reg_raw32"].append(reorg.raw[2].numpy())
                    per["reg32"].append(ns["reg_scores"].numpy())
            toff.append(toff[-1] + T)
            off.append(off[-1] + len(tk))
            scores.append(s)
            ticks.append(tk.numpy())
            scaling.append(sc.numpy())
        out[name + "_K"] = np.int64(K)
        out[name + "_cfg"] = np.array(repr(cfg))
        out[name + "_tick_offsets"] = np.array(toff, np.int64)
        out[name + "_offsets"] = np.array(off, np.int64)
        out[name + "_scores"] = np.concatenate(scores)
        out[name + "_ticks"] = np.concatenate(ticks).astype(np.int64)
        out[name + "_scaling"] = np.concatenate(scaling)
        for k, v in per.items():
            out[name + "_" + k] = np.concatenate(v).astype(np.float64 if k.endswith("64") else np.float32)
        assert out[name + "_reg32"].shape == (off[-1], K, 2)
    np.savez_compressed(os.path.join(GOLD, "test_tail.npz"), **out)
    print("wrote test_tail.npz:", len(out), "arrays,", sum(len(v[2]) for v in SETS.values()), "videos")


if __name__ == "__main__":
    main()
