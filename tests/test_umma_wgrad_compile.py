"""umma_wgrad.cu compiles for sm_90a without register spills or serialised wgmma sequences, in every instantiation.

A consumer thread holds up to 128 fp32 accumulators plus the bias column sums, and the TMA producer runs on the 40 registers
setmaxnreg leaves it; a spill in either, or ptxas serialising the wgmmas (C7520), is the likely silent regression.
"""
from test_umma_conv_compile import _compile


def test_wgrad_kernel_compiles_without_spills_or_serialized_wgmma(tmp_path):
    kernels, log = _compile("umma_wgrad", tmp_path)
    # 1-4 accumulator blocks, each for FAST (one plane per stage) and EXACT_TC (four planes per stage)
    assert sum("umma_wgrad_kernel" in k for k in kernels) == 8, kernels
    assert "wgmma.mma_async instructions are serialized" not in log, log[-4000:]
