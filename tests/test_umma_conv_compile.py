"""umma_conv.cu and glue_vec.cu compile for sm_90a without register spills, and umma_conv.cu without serialised wgmma sequences.

Each consumer thread of the ping-pong kernel holds up to 128 fp32 accumulators next to the epilogue code, so a spill or an
accumulator moved to local memory is the likely silent regression; ptxas then also serialises the wgmmas (C7520).  The glue
kernels keep many 16-byte loads in flight per thread; a stack frame there means an unrolled array went to local memory.
"""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compile(name, tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "action-detection_b200", "csrc", name + ".cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                          "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (name + ".o"))], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", out.stderr)
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out.stderr)
    assert len(props) == len(kernels) and all(p == ("0", "0", "0") for p in props), out.stderr[-4000:]
    return kernels, out.stderr


def test_conv_kernel_compiles_without_spills_or_serialized_wgmma(tmp_path):
    kernels, log = _compile("umma_conv", tmp_path)
    assert sum("umma_conv_kernel" in k for k in kernels) == 8          # block_n = 16, 32, ..., 128
    assert "wgmma.mma_async instructions are serialized" not in log, log[-4000:]


def test_glue_kernels_compile_without_spills(tmp_path):
    kernels, _ = _compile("glue_vec", tmp_path)
    # five kernel families, each for fp32 (EXACT_TC, "If") and fp16 (FAST, "I6__half") storage
    for fam in ("maxpool_fwd_vec", "maxpool_bwd_vec", "avgpool3_pair_vec", "13mask_bias_vec", "pool_mask_bias2x2_vec"):
        for t in ("IfE", "I6__halfE"):
            assert sum(fam + t in k for k in kernels) == 1, (fam, t, kernels)
    assert len(kernels) == 10, kernels
