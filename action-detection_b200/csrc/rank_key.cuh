// Descending-score radix keys shared by the sorting kernels (proposals.cu, detect.cu, detection_ap.cu).
#pragma once
#include <stdint.h>

namespace ssnb {

// descending score as an ascending radix key; -0 and +0 share a key, as they compare equal.  Every NaN, whatever its
// sign or payload, gets key 0, ahead of +inf (key 0x007fffff): NaN scores rank first, as numpy's argsort()[::-1] puts
// NaN first; a stable sort keeps equal keys (NaN among them) in input order.  key_score(0) is the NaN 0x7fffffff.
__device__ __forceinline__ uint32_t score_key(float s) {
  if (s != s) return 0u;
  uint32_t u = __float_as_uint(s == 0.f ? 0.f : s);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~u;
}
__device__ __forceinline__ float key_score(uint32_t key) {
  const uint32_t u = ~key;
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// score_key for a double score (proposal_ar.cu): the same rule on 64 bits.  Every NaN gets key 0, -0 and +0 share a key.
__device__ __forceinline__ uint64_t score_key64(double s) {
  if (s != s) return 0ull;
  uint64_t u = (uint64_t)__double_as_longlong(s == 0.0 ? 0.0 : s);
  u = (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
  return ~u;
}

}  // namespace ssnb
