// Epilogue helpers shared by the tensor-core convolution kernels: the SSNB_EXACT_TC fp32 epilogue.
#pragma once
#include "umma_conv.cuh"
#include "umma_dev.cuh"

namespace ssnb {
namespace umma {

// 32 bytes = 8 words through two 128-bit accesses
struct U8 { uint32_t v[8]; };
__device__ __forceinline__ U8 ldg256(const void* p) {
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  return U8{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}
__device__ __forceinline__ U8 ldg256_nc(const void* p) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  return U8{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}
__device__ __forceinline__ void stg256(void* p, const U8& a) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}

// SSNB_EXACT_TC epilogue: one 16-column chunk of an accumulator row in fp32 -- alpha * acc (+ bias, ReLU | + old) ->
// 64 bytes of fp32, plus the value's fp16 hi / lo operand planes (2 x 32 bytes) for the convolutions that consume it
__device__ __forceinline__ void store_chunk32(const UmmaConvParams& p, float alpha, const uint32_t* r, const float* bias, float* dst, __half* hdst,
                                              const float* ymask, long long lo_off) {
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]) * alpha;
  if (p.bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + j);
      v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
    }
  }
  if (p.accumulate) {
    const U8 o0 = ldg256(dst), o1 = ldg256(dst + 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] += __uint_as_float(o0.v[j]); v[8 + j] += __uint_as_float(o1.v[j]); }
  }
  if (p.relu) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  if (ymask) {                               // ReLU gradient of the value this data gradient completes: keep where y > 0 (NaN -> 0)
    const U8 y0 = ldg256_nc(ymask), y1 = ldg256_nc(ymask + 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (!(__uint_as_float(y0.v[j]) > 0.f)) v[j] = 0.f;
      if (!(__uint_as_float(y1.v[j]) > 0.f)) v[8 + j] = 0.f;
    }
  }
  U8 q0, q1;
#pragma unroll
  for (int j = 0; j < 8; ++j) { q0.v[j] = __float_as_uint(v[j]); q1.v[j] = __float_as_uint(v[8 + j]); }
  stg256(dst, q0);
  stg256(dst + 8, q1);
  if (hdst) {
    if (p.flag || p.plane_scale != 1.0f) {   // gradient planes: scaled by the loss scale, guarded against the fp16 range
      float m = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) { v[j] *= p.plane_scale; m = fmaxf(m, fabsf(v[j])); if (v[j] != v[j]) m = INFINITY; }
      if (p.flag && !(m <= 65504.f)) *p.flag = 1;
    }
    U8 qh, ql;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __half2 h = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
      qh.v[j] = *reinterpret_cast<const uint32_t*>(&h);
      ql.v[j] = *reinterpret_cast<const uint32_t*>(&l);
    }
    stg256(hdst, qh);
    stg256(reinterpret_cast<char*>(hdst) + lo_off, ql);
  }
}

}  // namespace umma
}  // namespace ssnb
