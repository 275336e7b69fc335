"""Test infrastructure (never imported by the product): CPU emulation of the EXACT_TC arithmetic of csrc/umma_conv.cu.

A product a.b of two fp32 numbers is formed on the tensor cores from fp16 planes hi = fp16(x), lo = fp16(x - hi) as
a_lo.b_hi + a_hi.b_lo + a_hi.b_hi (fp32 accumulate); weight planes are scaled by a power of two so that the layer's
largest weight lies in [4096, 8192) -- without it `lo` of a ~1e-3 weight is a subnormal fp16 number with 2-3
significant bits (DESIGN.md section 2, "Why split operands").  This module restates that arithmetic with torch CPU
ops so the error model can be checked without a GPU; the reference computes the same products in fp32
(model_zoo/bninception/layer_factory.py:25-39: nn.Conv2d, no AMP).

Gradients are split the same way: the backward reads the planes of dz * grad_scale * 2^k, where one exponent k per backward
(grad_exponent) brings the entry gradient max|dfeat| * grad_scale / 49 into [2^7, 2^8)."""
import math

import numpy as np
import torch

GRAD_EXP_TOP, GRAD_EXP_MAX = 8, 100         # csrc/common.cuh


def split(x):
    """fp32 tensor -> (hi, lo) fp16 planes, both returned as fp32 values (what the MMA multiplies)."""
    hi = x.to(torch.float16)
    lo = (x - hi.to(torch.float32)).to(torch.float16)
    return hi.to(torch.float32), lo.to(torch.float32)


def weight_scale(w):
    """power of two that brings max|w| into [4096, 8192) (pack_all_kernel's absmax + split_all_kernel's frexpf)."""
    m = float(w.abs().max())
    if m == 0.0:
        return 1.0
    _, e = math.frexp(m)            # m = f * 2^e, f in [0.5, 1)
    return 2.0 ** (13 - e)


def grad_exponent(amax, grad_scale, hw=49):
    """k of the backward's gradient scale 2^k (grad_exponent_kernel in csrc/simt_glue.cu, same fp32 steps): amax * grad_scale
    * 2^k / hw in [2^(GRAD_EXP_TOP-1), 2^GRAD_EXP_TOP); 0 for amax 0, inf or NaN (the device also raises the overflow flag
    then); |k| <= GRAD_EXP_MAX."""
    a = np.float32(amax)
    if not np.isfinite(a) or a == 0:
        return 0
    fa, ea = math.frexp(float(a))
    fg, eg = math.frexp(float(np.float32(grad_scale)))
    _, e = math.frexp(float(np.float32(np.float32(fa) * np.float32(fg)) / np.float32(hw)))
    return max(-GRAD_EXP_MAX, min(GRAD_EXP_MAX, GRAD_EXP_TOP - (ea + eg + e)))


def split_error(dz, scale):
    """rel-L2 of the gradient the planes carry, (hi + lo) / scale, against the fp32 dz"""
    hi, lo = split((dz * scale).float())
    return float(((hi.double() + lo.double()) / scale - dz.double()).norm() / dz.double().norm())


def split_matmul(a, b, scale_weights=True, accumulate=torch.float32):
    """a [M,K] activations, b [K,N] weights -> a @ b through the three-term split product (small terms first)."""
    s = weight_scale(b) if scale_weights else 1.0
    a_hi, a_lo = split(a)
    b_hi, b_lo = split(b * s)
    t = accumulate
    acc = a_lo.to(t) @ b_hi.to(t)
    acc = acc + a_hi.to(t) @ b_lo.to(t)
    acc = acc + a_hi.to(t) @ b_hi.to(t)
    return (acc / s).to(torch.float32)


def fp16_matmul(a, b):
    """FAST_FP16: fp16 operands, fp32 accumulate."""
    return a.to(torch.float16).to(torch.float32) @ b.to(torch.float16).to(torch.float32)
