"""umma_conv.cu compiles for sm_90a without register spills and without serialised wgmma sequences.

Each consumer thread of the ping-pong kernel holds up to 128 fp32 accumulators next to the epilogue code, so a spill or an
accumulator moved to local memory is the likely silent regression; ptxas then also serialises the wgmmas (C7520).
"""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_conv_kernel_compiles_without_spills_or_serialized_wgmma(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "action-detection_b200", "csrc", "umma_conv.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                          "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "umma_conv.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", out.stderr)
    assert sum("umma_conv_kernel" in k for k in kernels) == 8          # block_n = 16, 32, ..., 128
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out.stderr)
    assert len(props) == len(kernels) and all(p == ("0", "0", "0") for p in props), out.stderr[-4000:]
    assert "wgmma.mma_async instructions are serialized" not in out.stderr, out.stderr[-4000:]
