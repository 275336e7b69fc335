// FAST-mode (fp16 NHWC) memory-bound glue, vectorised: every thread moves 8 channels (16 bytes) so a
// warp covers 256 contiguous channels / 512 bytes per pixel row.  Same semantics as the generic
// kernels in simt_glue.cu (Caffe ceil-mode pooling, layer_factory.py:41-53; first-max-wins argmax).
#include <cstdlib>

#include "common.cuh"

namespace ssnb {
namespace {

struct H8 { uint4 v; };
__device__ __forceinline__ void unpack8(const uint4& r, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return r;
}
__device__ __forceinline__ uint4 ldg16(const __half* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// max pooling on packed halves: compares and selects run as half2 mask operations (no fp32 round trip; the first
// version spent ~400 instructions per thread on conversions and was issue-bound at 2.6 TB/s).  Semantics unchanged:
// first maximum wins, NaN propagates (ATen's rule).
// K > 0: compile-time window (the network's max pools are all 3x3): the K*K loads are issued before the first compare
template <int K>
__global__ void maxpool_fwd_h8(const __half* __restrict__ src, int H, int W, int C, int spitch, int scoff,
                               __half* __restrict__ dst, int OH, int OW, int dpitch, int dcoff, int F, int k_rt, int stride,
                               int pad, uint8_t* __restrict__ argmax) {
  const int k = K ? K : k_rt;
  const int G = C / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * OH * OW * G) return;
  // 32-bit index arithmetic (thread count < 2^31); 64-bit only for the final byte offsets
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ox = (int)(pu % (unsigned)OW), oy = (int)((pu / (unsigned)OW) % (unsigned)OH);
  const long long p = pu;
  const long long f = pu / (unsigned)(OW * OH);
  uint32_t best[4] = {0u, 0u, 0u, 0u};     // 4 x half2
  uint32_t bi[4] = {0u, 0u, 0u, 0u};       // 4 x (two 16-bit tap indices, same lanes as the half2 values)
  bool first = true;
  const __half* base = src + (f * H * W) * spitch + scoff + g * 8;
  // one tap: NaN-propagating maximum; the tap index moves where the maximum changed (v > best, or a NaN arrived), or when
  // nothing was taken yet: 3 instructions per half2
  auto take = [&](const uint4& q, uint32_t t) {
    const uint32_t v[4] = {q.x, q.y, q.z, q.w};
    const uint32_t tag = t * 0x00010001u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hv = *reinterpret_cast<const __half2*>(&v[j]);
      const __half2 hb = *reinterpret_cast<const __half2*>(&best[j]);
      const __half2 hn = __hmax2_nan(hb, hv);
      const uint32_t m = first ? 0xFFFFFFFFu : __hneu2_mask(hn, hb);
      best[j] = first ? v[j] : *reinterpret_cast<const uint32_t*>(&hn);
      bi[j] = (tag & m) | (bi[j] & ~m);
    }
    first = false;
  };
  if (K) {
    constexpr int K1 = K ? K : 1, KK = K1 * K1;
    uint4 q[KK]; bool ok[KK];
#pragma unroll
    for (int t = 0; t < KK; ++t) {
      const int iy = oy * stride + t / K1 - pad, ix = ox * stride + t % K1 - pad;
      ok[t] = iy >= 0 && iy < H && ix >= 0 && ix < W;
      q[t] = ok[t] ? ldg16(base + ((long long)iy * W + ix) * spitch) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int t = 0; t < KK; ++t)
      if (ok[t]) take(q[t], (uint32_t)t);
  } else {
    for (int r = 0; r < k; ++r) {
      const int iy = oy * stride + r - pad;
      if (iy < 0 || iy >= H) continue;
      for (int s = 0; s < k; ++s) {
        const int ix = ox * stride + s - pad;
        if (ix < 0 || ix >= W) continue;
        take(ldg16(base + ((long long)iy * W + ix) * spitch), (uint32_t)(r * k + s));
      }
    }
  }
  *reinterpret_cast<uint4*>(dst + p * dpitch + dcoff + g * 8) = make_uint4(best[0], best[1], best[2], best[3]);
  uint2 a;
  a.x = (bi[0] & 0xFFu) | ((bi[0] >> 8) & 0xFF00u) | ((bi[1] & 0xFFu) << 16) | ((bi[1] >> 16) << 24);
  a.y = (bi[2] & 0xFFu) | ((bi[2] >> 8) & 0xFF00u) | ((bi[3] & 0xFFu) << 16) | ((bi[3] >> 16) << 24);
  *reinterpret_cast<uint2*>(argmax + p * C + g * 8) = a;
}

__global__ void maxpool_bwd_h8(__half* __restrict__ dsrc, int H, int W, int C, int spitch, int scoff,
                               const __half* __restrict__ ddst, int OH, int OW, int dpitch, int dcoff, int F, int k,
                               int stride, int pad, const uint8_t* __restrict__ argmax, int accumulate) {
  const int G = C / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * H * W * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ix = (int)(pu % (unsigned)W), iy = (int)((pu / (unsigned)W) % (unsigned)H);
  const long long p = pu;
  const long long f = pu / (unsigned)(W * H);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // windows covering this pixel: oy in [ceil((iy+pad-k+1)/stride), floor((iy+pad)/stride)] (<= 2 per axis for k3/s2)
  const int ty0 = iy + pad - k + 1, tx0 = ix + pad - k + 1;
  const int oy_lo = ty0 > 0 ? (ty0 + stride - 1) / stride : 0, oy_hi = min((iy + pad) / stride, OH - 1);
  const int ox_lo = tx0 > 0 ? (tx0 + stride - 1) / stride : 0, ox_hi = min((ix + pad) / stride, OW - 1);
  if (oy_hi - oy_lo <= 1 && ox_hi - ox_lo <= 1) {
    // stride-2 pools: at most 2x2 covering windows -> issue every load before the first use (memory-level parallelism)
    uint2 am[4]; uint4 dv[4]; uint32_t tg[4]; bool ok[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int oy = oy_lo + (q >> 1), ox = ox_lo + (q & 1);
      ok[q] = oy <= oy_hi && ox <= ox_hi;
      const long long op = (f * OH + (ok[q] ? oy : oy_lo)) * OW + (ok[q] ? ox : ox_lo);
      tg[q] = (uint32_t)((iy + pad - oy * stride) * k + (ix + pad - ox * stride));
      am[q] = __ldg(reinterpret_cast<const uint2*>(argmax + op * C + g * 8));
      dv[q] = ldg16(ddst + op * dpitch + dcoff + g * 8);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!ok[q]) continue;
      float v[8];
      unpack8(dv[q], v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (((am[q].x >> (8 * j)) & 0xFFu) == tg[q]) acc[j] += v[j];
        if (((am[q].y >> (8 * j)) & 0xFFu) == tg[q]) acc[4 + j] += v[4 + j];
      }
    }
  } else {
  for (int oy = oy_lo; oy <= oy_hi; ++oy) {
    const int r = iy + pad - oy * stride;
    for (int ox = ox_lo; ox <= ox_hi; ++ox) {
      const int s = ix + pad - ox * stride;
      const long long op = (f * OH + oy) * OW + ox;
      const uint2 a = __ldg(reinterpret_cast<const uint2*>(argmax + op * C + g * 8));
      const uint32_t tag = (uint32_t)(r * k + s);
      const uint32_t t4 = tag * 0x01010101u;
      const uint32_t xa = a.x ^ t4, xb = a.y ^ t4;
      // zero byte test: does any of the 8 channels of this window point at this pixel?
      if (!(((xa - 0x01010101u) & ~xa & 0x80808080u) | ((xb - 0x01010101u) & ~xb & 0x80808080u))) continue;
      float v[8];
      unpack8(ldg16(ddst + op * dpitch + dcoff + g * 8), v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (((a.x >> (8 * j)) & 0xFFu) == tag) acc[j] += v[j];
        if (((a.y >> (8 * j)) & 0xFFu) == tag) acc[4 + j] += v[4 + j];
      }
    }
  }
  }
  __half* q = dsrc + p * spitch + scoff + g * 8;
  if (accumulate) {
    float o[8];
    unpack8(*reinterpret_cast<const uint4*>(q), o);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += o[j];
  }
  *reinterpret_cast<uint4*>(q) = pack8(acc);
}

// 3x3 stride-1 pad-1 average (count_include_pad: always /9; its own adjoint), 8 channels per thread, walking down a
// column with a rolling window of row sums.  Two adjacent columns per thread share the loads, the fp16->fp32
// conversions and the middle partial sum b + c: ~65 instead of ~100 instructions per output (the kernel is issue-bound).
__global__ void avgpool3_pair_h8(const __half* __restrict__ src, int H, int W, int C, int spitch, int scoff,
                                 __half* __restrict__ dst, int dpitch, int dcoff, int F, int accumulate) {
  const int G = C / 8, W2 = (W + 1) / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * W2 * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const int x = 2 * (int)((iu / (unsigned)G) % (unsigned)W2);
  const long long f = iu / (unsigned)(G * W2);
  const bool has1 = x + 1 < W;                       // second column of the pair exists
  float p0[8], c0[8], n0[8], p1[8], c1[8], n1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { p0[j] = c0[j] = p1[j] = c1[j] = 0.f; }
  auto rowsum = [&](int y, float* o0, float* o1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { o0[j] = 0.f; o1[j] = 0.f; }
    if (y >= H) return;
    const __half* base = src + ((f * H + y) * W) * spitch + scoff + g * 8;
    float a[8], b[8], c[8], d[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] = 0.f; c[j] = 0.f; d[j] = 0.f; }
    if (x - 1 >= 0) unpack8(ldg16(base + (long long)(x - 1) * spitch), a);
    unpack8(ldg16(base + (long long)x * spitch), b);
    if (x + 1 < W) unpack8(ldg16(base + (long long)(x + 1) * spitch), c);
    if (x + 2 < W) unpack8(ldg16(base + (long long)(x + 2) * spitch), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float m = b[j] + c[j];
      o0[j] = a[j] + m;
      o1[j] = m + d[j];
    }
  };
  rowsum(0, c0, c1);
  for (int y = 0; y < H; ++y) {
    rowsum(y + 1, n0, n1);
    float s0[8], s1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s0[j] = (p0[j] + c0[j] + n0[j]) * (1.0f / 9.0f);
      s1[j] = (p1[j] + c1[j] + n1[j]) * (1.0f / 9.0f);
    }
    __half* o = dst + ((f * H + y) * W + x) * dpitch + dcoff + g * 8;
    if (accumulate) {
      float old[8];
      unpack8(*reinterpret_cast<const uint4*>(o), old);
#pragma unroll
      for (int j = 0; j < 8; ++j) s0[j] += old[j];
      if (has1) {
        unpack8(*reinterpret_cast<const uint4*>(o + dpitch), old);
#pragma unroll
        for (int j = 0; j < 8; ++j) s1[j] += old[j];
      }
    }
    *reinterpret_cast<uint4*>(o) = pack8(s0);
    if (has1) *reinterpret_cast<uint4*>(o + dpitch) = pack8(s1);
#pragma unroll
    for (int j = 0; j < 8; ++j) { p0[j] = c0[j]; c0[j] = n0[j]; p1[j] = c1[j]; c1[j] = n1[j]; }
  }
}

// fused ReLU gradient mask + bias-gradient column sums: dz = dy * (y > 0) in place; partial[cta][c] = sum_rows dz
constexpr int MB_THREADS = 256;
// the last CTA to finish reduces the per-CTA partials in CTA order (deterministic) into db
__device__ __forceinline__ void colsum_tail(float* __restrict__ partial, unsigned* __restrict__ counter, int C,
                                            const float* __restrict__ mult, float out_scale, const float* __restrict__ unscale,
                                            float* __restrict__ db, bool* is_last, int accumulate) {
  if (!db) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!*is_last) return;
  __threadfence();
  const int n = (int)gridDim.x;
  if (unscale) out_scale *= __ldg(unscale);
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {      // coalesced across threads, 4 independent chains per thread
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int i = 0;
    for (; i + 3 < n; i += 4) {
      s0 += __ldcg(partial + (long long)i * C + c);       s1 += __ldcg(partial + (long long)(i + 1) * C + c);
      s2 += __ldcg(partial + (long long)(i + 2) * C + c); s3 += __ldcg(partial + (long long)(i + 3) * C + c);
    }
    for (; i < n; ++i) s0 += __ldcg(partial + (long long)i * C + c);
    db[c] = (accumulate ? db[c] : 0.f) + ((s0 + s1) + (s2 + s3)) * mult[c] * out_scale;
  }
  if (threadIdx.x == 0) *counter = 0;             // ready for the next launch on this stream
}
__global__ void __launch_bounds__(MB_THREADS) mask_bias_h8(__half* __restrict__ dy, int dpitch, int dcoff,
                                                           const __half* __restrict__ y, int ypitch, int ycoff,
                                                           long long rows, int C, long long rows_per_cta,
                                                           float* __restrict__ partial, unsigned* __restrict__ counter,
                                                           const float* __restrict__ mult, float out_scale,
                                                           const float* __restrict__ unscale, float* __restrict__ db, int accumulate) {
  extern __shared__ float red[];                 // [lanes][C]
  __shared__ bool is_last;
  const int G = C / 8;
  const int lanes = MB_THREADS / G;               // row lanes per CTA (G <= 64)
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = (r0 + rows_per_cta < rows) ? r0 + rows_per_cta : rows;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (rl < lanes) {
    constexpr int U = 8;                          // rows in flight per thread
    for (long long rb = r0 + rl; rb < r1; rb += (long long)lanes * U) {
      uint4 dv[U], yv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r < r1) {
          dv[u] = *reinterpret_cast<const uint4*>(dy + r * dpitch + dcoff + g * 8);
          if (y) yv[u] = ldg16(y + r * ypitch + ycoff + g * 8);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r >= r1) continue;
        float d[8], a[8];
        unpack8(dv[u], d);
        bool changed = false;
        if (y) {                                  // y == nullptr: the producer already masked dy (column sums only)
          unpack8(yv[u], a);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (!(a[j] > 0.f)) { changed = changed || (d[j] != 0.f); d[j] = 0.f; }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += d[j];
        if (changed) *reinterpret_cast<uint4*>(dy + r * dpitch + dcoff + g * 8) = pack8(d);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl * C + g * 8 + j] = acc[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
  colsum_tail(partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

// Same pass for a convolution whose only consumer is a stride-2 max pool (conv1 -> pool1, conv2_3x3 -> pool2):
// the pool's backward gather is folded in, so the full-resolution dy tensor is never written or re-read:
//   dz[p] = (sum over covering windows whose arg-max is p of dpool) * (y[p] > 0);  partial = column sums of dz
__global__ void __launch_bounds__(MB_THREADS) pool_mask_bias_h8(__half* __restrict__ dz, int dpitch, int dcoff,
                                                                const __half* __restrict__ y, int ypitch, int ycoff, int H,
                                                                int W, const __half* __restrict__ dpool, int OH, int OW,
                                                                int ppitch, int pcoff, const uint8_t* __restrict__ argmax,
                                                                int k, int stride, int pad, long long rows, int C,
                                                                long long rows_per_cta, float* __restrict__ partial,
                                                                unsigned* __restrict__ counter, const float* __restrict__ mult,
                                                                float out_scale, const float* __restrict__ unscale, float* __restrict__ db,
                                                                int accumulate) {
  extern __shared__ float red[];
  __shared__ bool is_last;
  const int G = C / 8;
  const int lanes = MB_THREADS / G;
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = (r0 + rows_per_cta < rows) ? r0 + rows_per_cta : rows;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (rl < lanes) {
    for (long long r = r0 + rl; r < r1; r += lanes) {
      const unsigned ru = (unsigned)r;                       // rows < 2^31
      const int ix = (int)(ru % (unsigned)W), iy = (int)((ru / (unsigned)W) % (unsigned)H);
      const long long f = ru / (unsigned)(W * H);
      const int ty0 = iy + pad - k + 1, tx0 = ix + pad - k + 1;
      const int oy_lo = ty0 > 0 ? (ty0 + stride - 1) / stride : 0, oy_hi = min((iy + pad) / stride, OH - 1);
      const int ox_lo = tx0 > 0 ? (tx0 + stride - 1) / stride : 0, ox_hi = min((ix + pad) / stride, OW - 1);
      uint2 am[4]; uint4 dv[4]; uint32_t tg[4]; bool ok[4];
      const uint4 yv = ldg16(y + r * ypitch + ycoff + g * 8);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int oy = oy_lo + (q >> 1), ox = ox_lo + (q & 1);
        ok[q] = oy <= oy_hi && ox <= ox_hi;
        const long long op = (f * OH + (ok[q] ? oy : oy_lo)) * OW + (ok[q] ? ox : ox_lo);
        tg[q] = (uint32_t)((iy + pad - oy * stride) * k + (ix + pad - ox * stride));
        am[q] = __ldg(reinterpret_cast<const uint2*>(argmax + op * C + g * 8));
        dv[q] = ldg16(dpool + op * ppitch + pcoff + g * 8);
      }
      float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, a[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!ok[q]) continue;
        float v[8];
        unpack8(dv[q], v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (((am[q].x >> (8 * j)) & 0xFFu) == tg[q]) d[j] += v[j];
          if (((am[q].y >> (8 * j)) & 0xFFu) == tg[q]) d[4 + j] += v[4 + j];
        }
      }
      unpack8(yv, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (!(a[j] > 0.f)) d[j] = 0.f;
        // round to storage precision first so the bias gradient sums exactly what the weight gradient reads
        d[j] = __half2float(__float2half_rn(d[j]));
        acc[j] += d[j];
      }
      *reinterpret_cast<uint4*>(dz + r * dpitch + dcoff + g * 8) = pack8(d);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl * C + g * 8 + j] = acc[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
  colsum_tail(partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}


// k3/s2/pad0 variant of the pass above working on 2x2 input blocks: the block (2i..2i+1, 2j..2j+1) is covered by the
// four windows (i-1..i, j-1..j) only, so one thread loads 4 windows + 4 activations for 4 outputs (the per-pixel version
// loads 4 windows per pixel: 2.8x the L1/L2 traffic) and has 12 independent loads in flight.
__global__ void __launch_bounds__(MB_THREADS) pool_mask_bias2x2_h8(__half* __restrict__ dz, int dpitch, int dcoff,
                                                                   const __half* __restrict__ y, int ypitch, int ycoff, int H, int W,
                                                                   const __half* __restrict__ dpool, int OH, int OW, int ppitch, int pcoff,
                                                                   const uint8_t* __restrict__ argmax, long long blocks, int C,
                                                                   long long blocks_per_cta, float* __restrict__ partial,
                                                                   unsigned* __restrict__ counter, const float* __restrict__ mult,
                                                                   float out_scale, const float* __restrict__ unscale, float* __restrict__ db,
                                                                   int accumulate) {
  extern __shared__ float red[];
  __shared__ bool is_last;
  const int G = C / 8;
  const int lanes = MB_THREADS / G;
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const int BH = (H + 1) / 2, BW = (W + 1) / 2;
  const long long b0 = (long long)blockIdx.x * blocks_per_cta;
  const long long b1 = (b0 + blocks_per_cta < blocks) ? b0 + blocks_per_cta : blocks;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (rl < lanes) {
    for (long long b = b0 + rl; b < b1; b += lanes) {
      const unsigned bu = (unsigned)b;
      const int bj = (int)(bu % (unsigned)BW), bi = (int)((bu / (unsigned)BW) % (unsigned)BH);
      const long long f = bu / (unsigned)(BW * BH);
      uint2 am[4]; uint4 dv[4], yv[4]; bool wok[4], pok[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int oy = bi - 1 + (q >> 1), ox = bj - 1 + (q & 1);
        wok[q] = oy >= 0 && oy < OH && ox >= 0 && ox < OW;
        if (wok[q]) {
          const long long op = (f * OH + oy) * OW + ox;
          am[q] = __ldg(reinterpret_cast<const uint2*>(argmax + op * C + g * 8));
          dv[q] = ldg16(dpool + op * ppitch + pcoff + g * 8);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int iy = 2 * bi + (q >> 1), ix = 2 * bj + (q & 1);
        pok[q] = iy < H && ix < W;
        if (pok[q]) yv[q] = ldg16(y + ((f * H + iy) * W + ix) * ypitch + ycoff + g * 8);
      }
      // packed-half arithmetic (the fp32 version of this loop was issue-bound: 65 % issue utilisation at 1.9 TB/s):
      // byte-compare the arg-max tags, widen the byte masks to half lanes, AND-select the pooled gradient, add as half2
      uint32_t bsum[4] = {0u, 0u, 0u, 0u};                       // half2 sums of the block's dz (bias gradient)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!pok[q]) continue;
        const int a = q >> 1, c = q & 1;
        uint32_t d2[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int wq = 0; wq < 4; ++wq) {
          const int u = wq >> 1, v = wq & 1;
          if (!((u == 1 || a == 0) && (v == 1 || c == 0))) continue;      // compile-time: this window never covers the pixel
          if (!wok[wq]) continue;
          const uint32_t tag4 = (uint32_t)((a + 2 - 2 * u) * 3 + (c + 2 - 2 * v)) * 0x01010101u;
          const uint32_t mx = __vcmpeq4(am[wq].x, tag4), my = __vcmpeq4(am[wq].y, tag4);
          const uint32_t k[4] = {__byte_perm(mx, 0u, 0x1100), __byte_perm(mx, 0u, 0x3322), __byte_perm(my, 0u, 0x1100), __byte_perm(my, 0u, 0x3322)};
          const uint32_t t[4] = {dv[wq].x, dv[wq].y, dv[wq].z, dv[wq].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t sel = t[j] & k[j];
            const __half2 r = __hadd2(*reinterpret_cast<const __half2*>(&d2[j]), *reinterpret_cast<const __half2*>(&sel));
            d2[j] = *reinterpret_cast<const uint32_t*>(&r);
          }
        }
        const uint32_t yy[4] = {yv[q].x, yv[q].y, yv[q].z, yv[q].w};
        const __half2 zero = __float2half2_rn(0.f);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          d2[j] &= __hgt2_mask(*reinterpret_cast<const __half2*>(&yy[j]), zero);       // ReLU gradient: keep where y > 0
          const __half2 r = __hadd2(*reinterpret_cast<const __half2*>(&bsum[j]), *reinterpret_cast<const __half2*>(&d2[j]));
          bsum[j] = *reinterpret_cast<const uint32_t*>(&r);
        }
        const int iy = 2 * bi + a, ix = 2 * bj + c;
        *reinterpret_cast<uint4*>(dz + ((f * H + iy) * W + ix) * dpitch + dcoff + g * 8) = make_uint4(d2[0], d2[1], d2[2], d2[3]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&bsum[j]));
        acc[2 * j] += t.x; acc[2 * j + 1] += t.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[rl * C + g * 8 + j] = acc[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
  colsum_tail(partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

}  // namespace

#define HP(v) reinterpret_cast<__half*>((v).base)
static inline unsigned nblk(long long n, int t) { return (unsigned)((n + t - 1) / t); }

int launch_maxpool_fwd_h8(View src, View dst, int F, int k, int stride, int pad, uint8_t* argmax, cudaStream_t s) {
  const long long n = (long long)F * dst.H * dst.W * (src.C / 8);
  if (k == 3)
    maxpool_fwd_h8<3><<<nblk(n, 256), 256, 0, s>>>(HP(src), src.H, src.W, src.C, src.pitch, src.coff, HP(dst), dst.H, dst.W, dst.pitch,
                                             dst.coff, F, k, stride, pad, argmax);
  else
    maxpool_fwd_h8<0><<<nblk(n, 256), 256, 0, s>>>(HP(src), src.H, src.W, src.C, src.pitch, src.coff, HP(dst), dst.H, dst.W, dst.pitch,
                                             dst.coff, F, k, stride, pad, argmax);
  SSNB_LAUNCH_CHECK("maxpool_fwd_h8");
  return 0;
}
int launch_maxpool_bwd_h8(View dsrc, View ddst, int F, int k, int stride, int pad, const uint8_t* argmax, int accumulate,
                          cudaStream_t s) {
  const long long n = (long long)F * dsrc.H * dsrc.W * (dsrc.C / 8);
  maxpool_bwd_h8<<<nblk(n, 256), 256, 0, s>>>(HP(dsrc), dsrc.H, dsrc.W, dsrc.C, dsrc.pitch, dsrc.coff, HP(ddst), ddst.H, ddst.W,
                                             ddst.pitch, ddst.coff, F, k, stride, pad, argmax, accumulate);
  SSNB_LAUNCH_CHECK("maxpool_bwd_h8");
  return 0;
}
int launch_avgpool3_h8(View src, View dst, int F, int accumulate, cudaStream_t s) {
  const long long n2 = (long long)F * ((src.W + 1) / 2) * (src.C / 8);
  avgpool3_pair_h8<<<nblk(n2, 128), 128, 0, s>>>(HP(src), src.H, src.W, src.C, src.pitch, src.coff, HP(dst), dst.pitch, dst.coff, F, accumulate);
  SSNB_LAUNCH_CHECK("avgpool3_pair_h8");
  return 0;
}
// partial must hold max_ctas * C floats; db may be nullptr (mask only)
int launch_mask_bias_h8(View dy, View y, int F, const float* mult, float out_scale, const float* unscale, float* partial, int max_ctas,
                        float* db, int accumulate, cudaStream_t s) {
  const long long rows = (long long)F * dy.H * dy.W;
  const int C = dy.C;
  if (C % 8 || C / 8 > 64) { set_thread_error("mask_bias: C must be a multiple of 8 and <= 512"); return 1; }
  int ctas = (int)((rows + 255) / 256);
  if (ctas > 444) ctas = 444;                      // three CTAs per SM: enough to saturate HBM, short final reduction
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  const long long rpc = (rows + ctas - 1) / ctas;
  ctas = (int)((rows + rpc - 1) / rpc);
  const int lanes = MB_THREADS / (C / 8);
  unsigned* counter = reinterpret_cast<unsigned*>(partial);          // first 256 bytes of the scratch: completion counter
  float* part = partial + 64;
  mask_bias_h8<<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(HP(dy), dy.pitch, dy.coff, HP(y), y.pitch, y.coff, rows, C, rpc, part,
                                                              counter, mult, out_scale, unscale, db, accumulate);
  SSNB_LAUNCH_CHECK("mask_bias_h8");
  return 0;
}


// conv output y/dz views at full resolution; dpool = gradient of the max pool's output, argmax from its forward
int launch_pool_mask_bias_h8(View dz, View y, View dpool, int F, int k, int stride, int pad, const uint8_t* argmax,
                             const float* mult, float out_scale, const float* unscale, float* partial, int max_ctas, float* db, int accumulate,
                             cudaStream_t s) {
  const long long rows = (long long)F * dz.H * dz.W;
  const int C = dz.C;
  if (C % 8 || C / 8 > 64 || stride != 2 || k != 3) { set_thread_error("pool_mask_bias: k3/s2 pools, C multiple of 8 and <= 512"); return 1; }
  const int lanes = MB_THREADS / (C / 8);
  unsigned* counter = reinterpret_cast<unsigned*>(partial);
  float* part = partial + 64;
  if (pad == 0) {                                   // 2x2-block version (every BNInception stride-2 pool)
    const long long blocks = (long long)F * ((dz.H + 1) / 2) * ((dz.W + 1) / 2);
    int ctas = (int)((blocks + 63) / 64);
    if (ctas > 888) ctas = 888;
    if (ctas > max_ctas) ctas = max_ctas;
    if (ctas < 1) ctas = 1;
    const long long bpc = (blocks + ctas - 1) / ctas;
    ctas = (int)((blocks + bpc - 1) / bpc);
    pool_mask_bias2x2_h8<<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(HP(dz), dz.pitch, dz.coff, HP(y), y.pitch, y.coff, dz.H, dz.W, HP(dpool),
                                                                        dpool.H, dpool.W, dpool.pitch, dpool.coff, argmax, blocks, C, bpc, part,
                                                                        counter, mult, out_scale, unscale, db, accumulate);
    SSNB_LAUNCH_CHECK("pool_mask_bias2x2_h8");
    return 0;
  }
  int ctas = (int)((rows + 255) / 256);
  if (ctas > 888) ctas = 888;
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  const long long rpc = (rows + ctas - 1) / ctas;
  ctas = (int)((rows + rpc - 1) / rpc);
  pool_mask_bias_h8<<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(HP(dz), dz.pitch, dz.coff, HP(y), y.pitch, y.coff, dz.H, dz.W, HP(dpool),
                                                                   dpool.H, dpool.W, dpool.pitch, dpool.coff, argmax, k, stride, pad, rows, C,
                                                                   rpc, part, counter, mult, out_scale, unscale, db, accumulate);
  SSNB_LAUNCH_CHECK("pool_mask_bias_h8");
  return 0;
}

}  // namespace ssnb
