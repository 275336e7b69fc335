"""2-GPU gradient norm after the data-parallel exchange (needs >= 2 CUDA devices: `python -m pytest tests/test_dp_train_loop.py
-m gpu`; skipped on a 1-GPU box): after GradSync.finish() both ranks' clip norms are bitwise equal, and equal to the norm of
the single-GPU step on the global batch."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_clip_norm_identical_on_both_ranks():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29733", os.path.join(ROOT, "tests", "dp_train_loop_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1200)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("DP_TRAIN_LOOP_RESULT ")]
    assert line, out.stdout[-2000:]
    r = json.loads(line[-1][len("DP_TRAIN_LOOP_RESULT "):])
    print("DP clip norm:", r)
    assert r["rank_norms_bitwise_equal"], r
    assert r["rel_vs_global"] < 1e-6, r
