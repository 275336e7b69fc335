// Memory-bound glue of every precision over NHWC views, vectorised: every thread moves 16 bytes of channels, 4 fp32
// channels in SSNB_EXACT_FP32 and SSNB_EXACT_TC, 8 fp16 channels in SSNB_FAST_FP16.  Caffe ceil-mode pooling
// (model_zoo/bninception/layer_factory.py:41-53) with a first-max-wins arg-max, the 3x3 average with count_include_pad, and
// the ReLU mask + bias-gradient pass of a convolution's backward.  Each kernel is written once over the storage type; Vec<T>
// holds what differs between the two.  In EXACT_TC the kernels that produce a convolution operand also write its fp16 hi / lo
// planes, so no separate split pass runs; EXACT_FP32 passes no planes.
#include <type_traits>

#include "common.cuh"

namespace ssnb {
namespace {

// 0x80 in every byte of x that is zero
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) { return (x - 0x01010101u) & ~x & 0x80808080u; }

template <typename T> struct Vec;

// EXACT_FP32 and EXACT_TC: fp32 arithmetic throughout; in EXACT_TC the outputs that feed a tensor-core product also go out as
// hi / lo planes
template <> struct Vec<float> {
  static constexpr int N = VEC_WIDTH<float>;
  static constexpr bool PLANES = true;
  static constexpr int MASK_CTAS = 592;                 // four CTAs per SM
  using Raw = float4;
  using Tags = uint32_t;                                // N 8-bit arg-max tap indices
  static __device__ __forceinline__ void unpack(const float4& r, float* f) { f[0] = r.x; f[1] = r.y; f[2] = r.z; f[3] = r.w; }
  static __device__ __forceinline__ float4 pack(const float* f) { return make_float4(f[0], f[1], f[2], f[3]); }
  // acc += the lanes of v whose arg-max tag is t
  static __device__ __forceinline__ void add_tagged(float* acc, Tags am, const float* v, uint32_t t) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (((am >> (8 * j)) & 0xFFu) == t) acc[j] += v[j];
  }
  static __device__ __forceinline__ uint32_t any_tag(Tags a, uint32_t t4) { return zero_bytes(a ^ t4); }
  // running maximum of a window, per lane: first max wins, NaN propagates and the last NaN holds the arg-max (ATen)
  struct Max {
    float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    uint32_t bi = 0u;
    __device__ __forceinline__ void take(const float4& q, uint32_t t, bool first) {
      const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (first || v[j] > best[j] || v[j] != v[j]) { best[j] = v[j]; bi = (bi & ~(0xFFu << (8 * j))) | (t << (8 * j)); }
    }
    __device__ __forceinline__ float4 value() const { return make_float4(best[0], best[1], best[2], best[3]); }
    __device__ __forceinline__ Tags tags() const { return bi; }
  };
  static __device__ __forceinline__ float avg9(float s) { return s / 9.0f; }      // a true division, as ATen's s / 9
  static __device__ __forceinline__ void planes(__half* hi, long long lo_off, const float4& v) { store_planes4(hi, lo_off, v); }
  // planes of a gradient times the loss scale; amax = largest magnitude so far (inf after a NaN)
  static __device__ __forceinline__ void grad_planes(__half* hi, long long lo_off, const float4& d, float scale, float& amax) {
    const float4 sv = make_float4(d.x * scale, d.y * scale, d.z * scale, d.w * scale);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(sv.x), fabsf(sv.y)), fmaxf(fabsf(sv.z), fabsf(sv.w))));
    if (sv.x != sv.x || sv.y != sv.y || sv.z != sv.z || sv.w != sv.w) amax = INFINITY;
    store_planes4(hi, lo_off, sv);
  }
  // 2x2 pool-gather pass: d += the lanes of the window gradient w whose arg-max is tap t; ReLU mask; bias sums added per pixel
  static __device__ __forceinline__ void gather(float4& d, Tags am, const float4& w, uint32_t t) {
    const float v[4] = {w.x, w.y, w.z, w.w};
    add_tagged(reinterpret_cast<float*>(&d), am, v, t);
  }
  struct BlockSum {
    // ReLU-mask d by y, add it to the bias sums
    __device__ __forceinline__ void mask_add(float* acc, float4& d, const float4& y) {
      float* dd = reinterpret_cast<float*>(&d);
      const float yy[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!(yy[j] > 0.f)) dd[j] = 0.f;
        acc[j] += dd[j];
      }
    }
    __device__ __forceinline__ void flush(float*) {}
  };
};

// FAST: packed halves; the pools compare and the pool-gather pass selects and adds as half2 (their fp32 versions were issue-bound)
template <> struct Vec<__half> {
  static constexpr int N = VEC_WIDTH<__half>;
  static constexpr bool PLANES = false;
  static constexpr int MASK_CTAS = 444;                 // three CTAs per SM: enough to saturate HBM, short final reduction
  using Raw = uint4;
  using Tags = uint2;
  static __device__ __forceinline__ void unpack(const uint4& r, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint4 r;
    __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return r;
  }
  static __device__ __forceinline__ void add_tagged(float* acc, Tags am, const float* v, uint32_t t) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (((am.x >> (8 * j)) & 0xFFu) == t) acc[j] += v[j];
      if (((am.y >> (8 * j)) & 0xFFu) == t) acc[4 + j] += v[4 + j];
    }
  }
  static __device__ __forceinline__ uint32_t any_tag(Tags a, uint32_t t4) { return zero_bytes(a.x ^ t4) | zero_bytes(a.y ^ t4); }
  // NaN-propagating half2 maximum; value and tap index (16-bit, in the lanes of the half2 values) move together where
  // v > best or v is NaN (so a later NaN takes them from an earlier one, as in ATen), or when nothing was taken yet.  The
  // value is the taken tap's bits: __hmax2_nan would give +0 for a window whose first maximum is -0.
  struct Max {
    uint32_t best[4] = {0u, 0u, 0u, 0u};
    uint32_t bi[4] = {0u, 0u, 0u, 0u};
    __device__ __forceinline__ void take(const uint4& q, uint32_t t, bool first) {
      const uint32_t v[4] = {q.x, q.y, q.z, q.w};
      const uint32_t tag = t * 0x00010001u;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __half2 hv = *reinterpret_cast<const __half2*>(&v[j]);
        const __half2 hb = *reinterpret_cast<const __half2*>(&best[j]);
        const uint32_t m = first ? 0xFFFFFFFFu : (__hgt2_mask(hv, hb) | __hneu2_mask(hv, hv));
        best[j] = (v[j] & m) | (best[j] & ~m);
        bi[j] = (tag & m) | (bi[j] & ~m);
      }
    }
    __device__ __forceinline__ uint4 value() const { return make_uint4(best[0], best[1], best[2], best[3]); }
    __device__ __forceinline__ Tags tags() const {        // 16-bit tags -> bytes
      return make_uint2((bi[0] & 0xFFu) | ((bi[0] >> 8) & 0xFF00u) | ((bi[1] & 0xFFu) << 16) | ((bi[1] >> 16) << 24),
                        (bi[2] & 0xFFu) | ((bi[2] >> 8) & 0xFF00u) | ((bi[3] & 0xFFu) << 16) | ((bi[3] >> 16) << 24));
    }
  };
  static __device__ __forceinline__ float avg9(float s) { return s * (1.0f / 9.0f); }
  static __device__ __forceinline__ void planes(__half*, long long, const uint4&) {}
  static __device__ __forceinline__ void grad_planes(__half*, long long, const uint4&, float, float&) {}
  // byte-compare the arg-max tags, widen the byte masks to half lanes, AND-select the window gradient, add as half2
  static __device__ __forceinline__ void gather(uint4& d, Tags am, const uint4& w, uint32_t t) {
    uint32_t* dd = reinterpret_cast<uint32_t*>(&d);
    const uint32_t t4 = t * 0x01010101u;
    const uint32_t mx = __vcmpeq4(am.x, t4), my = __vcmpeq4(am.y, t4);
    const uint32_t k[4] = {__byte_perm(mx, 0u, 0x1100), __byte_perm(mx, 0u, 0x3322), __byte_perm(my, 0u, 0x1100), __byte_perm(my, 0u, 0x3322)};
    const uint32_t v[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t sel = v[j] & k[j];
      const __half2 r = __hadd2(*reinterpret_cast<const __half2*>(&dd[j]), *reinterpret_cast<const __half2*>(&sel));
      dd[j] = *reinterpret_cast<const uint32_t*>(&r);
    }
  }
  // the bias sums of a 2x2 block add up in half2 and reach the fp32 lane sums once per block
  struct BlockSum {
    uint32_t s[4] = {0u, 0u, 0u, 0u};
    __device__ __forceinline__ void mask_add(float*, uint4& d, const uint4& y) {
      uint32_t* dd = reinterpret_cast<uint32_t*>(&d);
      const uint32_t yy[4] = {y.x, y.y, y.z, y.w};
      const __half2 zero = __float2half2_rn(0.f);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        dd[j] &= __hgt2_mask(*reinterpret_cast<const __half2*>(&yy[j]), zero);
        const __half2 r = __hadd2(*reinterpret_cast<const __half2*>(&s[j]), *reinterpret_cast<const __half2*>(&dd[j]));
        s[j] = *reinterpret_cast<const uint32_t*>(&r);
      }
    }
    __device__ __forceinline__ void flush(float* acc) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&s[j]));
        acc[2 * j] += t.x; acc[2 * j + 1] += t.y;
      }
    }
  };
};

template <typename T> __device__ __forceinline__ typename Vec<T>::Raw ldv(const T* p) {
  return __ldg(reinterpret_cast<const typename Vec<T>::Raw*>(p));
}

// ---- max pooling ---------------------------------------------------------------------------------------------
// every max pool of the network is 3x3: all nine loads are issued before the first compare; the compare order -- and with
// it the first-max-wins / NaN rule -- is that of a row-major loop over the window
template <typename T>
__global__ void maxpool_fwd_vec(const T* __restrict__ src, int H, int W, int C, int spitch, int scoff, T* __restrict__ dst, int OH, int OW,
                                int dpitch, int dcoff, __half* __restrict__ hi, long long lo_off, int stride, int pad, int F,
                                uint8_t* __restrict__ argmax) {
  using V = Vec<T>;
  constexpr int N = V::N, K = 3;
  const int G = C / N;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * OH * OW * G) return;
  // 32-bit index arithmetic (thread count < 2^31); 64-bit only for the final offsets
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ox = (int)(pu % (unsigned)OW), oy = (int)((pu / (unsigned)OW) % (unsigned)OH);
  const long long p = pu;
  const long long f = pu / (unsigned)(OW * OH);
  const T* base = src + (f * H * W) * spitch + scoff + g * N;
  typename V::Raw q[K * K];
  bool ok[K * K];
#pragma unroll
  for (int t = 0; t < K * K; ++t) {
    const int iy = oy * stride + t / K - pad, ix = ox * stride + t % K - pad;
    ok[t] = iy >= 0 && iy < H && ix >= 0 && ix < W;
    q[t] = ok[t] ? ldv(base + ((long long)iy * W + ix) * spitch) : typename V::Raw{};
  }
  typename V::Max m;
  bool first = true;
#pragma unroll
  for (int t = 0; t < K * K; ++t) {
    if (!ok[t]) continue;
    m.take(q[t], (uint32_t)t, first);
    first = false;
  }
  const typename V::Raw o = m.value();
  *reinterpret_cast<typename V::Raw*>(dst + p * dpitch + dcoff + g * N) = o;
  if (hi) V::planes(hi + p * dpitch + dcoff + g * N, lo_off, o);
  *reinterpret_cast<typename V::Tags*>(argmax + p * C + g * N) = m.tags();
}

template <typename T>
__global__ void maxpool_bwd_vec(T* __restrict__ dsrc, int H, int W, int C, int spitch, int scoff, const T* __restrict__ ddst, int OH, int OW,
                                int dpitch, int dcoff, int F, int k, int stride, int pad, const uint8_t* __restrict__ argmax, int accumulate) {
  using V = Vec<T>;
  using Raw = typename V::Raw;
  using Tags = typename V::Tags;
  constexpr int N = V::N;
  const int G = C / N;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * H * W * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ix = (int)(pu % (unsigned)W), iy = (int)((pu / (unsigned)W) % (unsigned)H);
  const long long p = pu;
  const long long f = pu / (unsigned)(W * H);
  float acc[N] = {};
  // windows covering this pixel: oy in [ceil((iy+pad-k+1)/stride), floor((iy+pad)/stride)]
  const int ty0 = iy + pad - k + 1, tx0 = ix + pad - k + 1;
  const int oy_lo = ty0 > 0 ? (ty0 + stride - 1) / stride : 0, oy_hi = min((iy + pad) / stride, OH - 1);
  const int ox_lo = tx0 > 0 ? (tx0 + stride - 1) / stride : 0, ox_hi = min((ix + pad) / stride, OW - 1);
  if (oy_hi - oy_lo <= 1 && ox_hi - ox_lo <= 1) {
    // stride-2 pools: at most 2x2 covering windows -> every load is issued before the first use
    Tags am[4]; Raw dv[4]; uint32_t tg[4]; bool ok[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int oy = oy_lo + (q >> 1), ox = ox_lo + (q & 1);
      ok[q] = oy <= oy_hi && ox <= ox_hi;
      const long long op = (f * OH + (ok[q] ? oy : oy_lo)) * OW + (ok[q] ? ox : ox_lo);
      tg[q] = (uint32_t)((iy + pad - oy * stride) * k + (ix + pad - ox * stride));
      am[q] = __ldg(reinterpret_cast<const Tags*>(argmax + op * C + g * N));
      dv[q] = ldv(ddst + op * dpitch + dcoff + g * N);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!ok[q]) continue;
      float v[N];
      V::unpack(dv[q], v);
      V::add_tagged(acc, am[q], v, tg[q]);
    }
  } else {
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      const int r = iy + pad - oy * stride;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int s = ix + pad - ox * stride;
        const long long op = (f * OH + oy) * OW + ox;
        const Tags a = __ldg(reinterpret_cast<const Tags*>(argmax + op * C + g * N));
        const uint32_t tag = (uint32_t)(r * k + s);
        if (!V::any_tag(a, tag * 0x01010101u)) continue;      // none of the channels of this window points here
        float v[N];
        V::unpack(ldv(ddst + op * dpitch + dcoff + g * N), v);
        V::add_tagged(acc, a, v, tag);
      }
    }
  }
  T* q = dsrc + p * spitch + scoff + g * N;
  if (accumulate) {
    float o[N];
    V::unpack(*reinterpret_cast<const Raw*>(q), o);
#pragma unroll
    for (int j = 0; j < N; ++j) acc[j] += o[j];
  }
  *reinterpret_cast<Raw*>(q) = V::pack(acc);
}

// ---- 3x3 stride-1 pad-1 average (count_include_pad: always /9; its own adjoint) ---------------------------------------
// one thread per (frame, column PAIR, channel group) walks down the rows keeping the horizontal 3-sums of the last three
// rows; the two columns share the loads, the conversions and the middle partial sum b + c: ~65 instead of ~100
// instructions per output in FAST (the kernel is issue-bound)
template <typename T>
__global__ void avgpool3_pair_vec(const T* __restrict__ src, int H, int W, int C, int spitch, int scoff, T* __restrict__ dst, int dpitch,
                                  int dcoff, __half* __restrict__ hi, long long lo_off, int F, int accumulate) {
  using V = Vec<T>;
  using Raw = typename V::Raw;
  constexpr int N = V::N;
  const int G = C / N, W2 = (W + 1) / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * W2 * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const int x = 2 * (int)((iu / (unsigned)G) % (unsigned)W2);
  const long long f = iu / (unsigned)(G * W2);
  const bool has1 = x + 1 < W;                       // second column of the pair exists
  float p0[N], c0[N], n0[N], p1[N], c1[N], n1[N];
#pragma unroll
  for (int j = 0; j < N; ++j) { p0[j] = c0[j] = p1[j] = c1[j] = 0.f; }
  auto rowsum = [&](int y, float* o0, float* o1) {
#pragma unroll
    for (int j = 0; j < N; ++j) { o0[j] = 0.f; o1[j] = 0.f; }
    if (y >= H) return;
    const T* base = src + ((f * H + y) * W) * spitch + scoff + g * N;
    float a[N] = {}, b[N], c[N] = {}, d[N] = {};
    if (x - 1 >= 0) V::unpack(ldv(base + (long long)(x - 1) * spitch), a);
    V::unpack(ldv(base + (long long)x * spitch), b);
    if (x + 1 < W) V::unpack(ldv(base + (long long)(x + 1) * spitch), c);
    if (x + 2 < W) V::unpack(ldv(base + (long long)(x + 2) * spitch), d);
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float m = b[j] + c[j];
      o0[j] = a[j] + m;
      o1[j] = m + d[j];
    }
  };
  rowsum(0, c0, c1);
  for (int y = 0; y < H; ++y) {
    rowsum(y + 1, n0, n1);
    float s0[N], s1[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
      s0[j] = V::avg9(p0[j] + c0[j] + n0[j]);
      s1[j] = V::avg9(p1[j] + c1[j] + n1[j]);
    }
    T* o = dst + ((f * H + y) * W + x) * dpitch + dcoff + g * N;
    if (accumulate) {
      float old[N];
      V::unpack(*reinterpret_cast<const Raw*>(o), old);
#pragma unroll
      for (int j = 0; j < N; ++j) s0[j] += old[j];
      if (has1) {
        V::unpack(*reinterpret_cast<const Raw*>(o + dpitch), old);
#pragma unroll
        for (int j = 0; j < N; ++j) s1[j] += old[j];
      }
    }
    *reinterpret_cast<Raw*>(o) = V::pack(s0);
    if (has1) *reinterpret_cast<Raw*>(o + dpitch) = V::pack(s1);
    if (hi) {
      __half* hp = hi + ((f * H + y) * W + x) * dpitch + dcoff + g * N;
      V::planes(hp, lo_off, V::pack(s0));
      if (has1) V::planes(hp + dpitch, lo_off, V::pack(s1));
    }
#pragma unroll
    for (int j = 0; j < N; ++j) { p0[j] = c0[j]; c0[j] = n0[j]; p1[j] = c1[j]; c1[j] = n1[j]; }
  }
}

// ---- backward pass of a convolution's output gradient: ReLU mask + bias-gradient column sums (+ operand planes) ----------
//   dz = dy * (y > 0);  partial[cta][c] = sum_rows dz;  EXACT_TC: planes = hi/lo of dz * scale (the tensor-core weight / data
//   gradients read the planes; the fp32 dz is written back only on request)
constexpr int MB_THREADS = 256;
// the CTA's lane sums [lanes][C] -> partial[cta]; then the last CTA to finish reduces the per-CTA partials in CTA order
// (deterministic) into db
__device__ __forceinline__ void colsum_tail(const float* red, int lanes, float* __restrict__ partial, unsigned* __restrict__ counter, int C,
                                            const float* __restrict__ mult, float out_scale, const float* __restrict__ unscale,
                                            float* __restrict__ db, bool* is_last, int accumulate) {
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
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

template <typename T>
__global__ void __launch_bounds__(MB_THREADS) mask_bias_vec(T* __restrict__ dy, int dpitch, int dcoff, const T* __restrict__ y, int ypitch,
                                                            int ycoff, __half* __restrict__ hi, int hpitch, int hcoff, long long lo_off,
                                                            float scale, int write_back, int* __restrict__ flag, long long rows, int C,
                                                            long long rows_per_cta, float* __restrict__ partial, unsigned* __restrict__ counter,
                                                            const float* __restrict__ mult, float out_scale, const float* __restrict__ unscale,
                                                            float* __restrict__ db, int accumulate) {
  using V = Vec<T>;
  using Raw = typename V::Raw;
  constexpr int N = V::N;
  extern __shared__ float red[];                 // [lanes][C]
  __shared__ bool is_last;
  const int G = C / N;
  const int lanes = MB_THREADS / G;               // row lanes per CTA (G <= 256)
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = (r0 + rows_per_cta < rows) ? r0 + rows_per_cta : rows;
  float acc[N] = {};
  float amax = 0.f;
  if (rl < lanes) {
    constexpr int U = 8;                          // rows in flight per thread
    for (long long rb = r0 + rl; rb < r1; rb += (long long)lanes * U) {
      Raw dv[U], yv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r < r1) {
          dv[u] = *reinterpret_cast<const Raw*>(dy + r * dpitch + dcoff + g * N);
          if (y) yv[u] = ldv(y + r * ypitch + ycoff + g * N);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r >= r1) continue;
        float d[N];
        V::unpack(dv[u], d);
        bool changed = false;
        if (y) {                                  // y == nullptr: dy is already masked or no ReLU follows (column sums / planes only)
          float a[N];
          V::unpack(yv[u], a);
#pragma unroll
          for (int j = 0; j < N; ++j)
            if (!(a[j] > 0.f)) { changed = changed || (d[j] != 0.f); d[j] = 0.f; }
        }
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] += d[j];
        if (write_back && changed) *reinterpret_cast<Raw*>(dy + r * dpitch + dcoff + g * N) = V::pack(d);
        if (hi) V::grad_planes(hi + r * hpitch + hcoff + g * N, lo_off, V::pack(d), scale, amax);
      }
    }
#pragma unroll
    for (int j = 0; j < N; ++j) red[rl * C + g * N + j] = acc[j];
  }
  if (flag && !(amax <= HALF_MAX)) *flag = 1;      // the loss scale pushed a gradient beyond the fp16 range (or a NaN arrived)
  colsum_tail(red, lanes, partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

// Same pass for a convolution whose only consumer is a k3/s2/pad0 max pool (conv1 -> pool1, conv2_3x3 -> pool2): the pool's
// backward gather is folded in, so the full-resolution dy tensor is neither written by a pooling kernel nor re-read:
//   dz[p] = (sum over covering windows whose arg-max is p of dpool) * (y[p] > 0)
// Works on 2x2 input blocks: block (2i..2i+1, 2j..2j+1) is covered by the four windows (i-1..i, j-1..j) only, so one thread
// loads 4 windows + 4 activations for 4 outputs (a per-pixel version loads 4 windows per pixel: 2.8x the L1/L2 traffic) and
// has 12 independent loads in flight.
template <typename T>
__global__ void __launch_bounds__(MB_THREADS) pool_mask_bias2x2_vec(T* __restrict__ dz, int dpitch, int dcoff, const T* __restrict__ y,
                                                                    int ypitch, int ycoff, int H, int W, const T* __restrict__ dpool, int OH,
                                                                    int OW, int ppitch, int pcoff, const uint8_t* __restrict__ argmax,
                                                                    __half* __restrict__ hi, int hpitch, int hcoff, long long lo_off, float scale,
                                                                    int write_back, int* __restrict__ flag, long long blocks, int C,
                                                                    long long blocks_per_cta, float* __restrict__ partial,
                                                                    unsigned* __restrict__ counter, const float* __restrict__ mult,
                                                                    float out_scale, const float* __restrict__ unscale, float* __restrict__ db,
                                                                    int accumulate) {
  using V = Vec<T>;
  using Raw = typename V::Raw;
  constexpr int N = V::N;
  extern __shared__ float red[];
  __shared__ bool is_last;
  const int G = C / N;
  const int lanes = MB_THREADS / G;
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const int BH = (H + 1) / 2, BW = (W + 1) / 2;
  const long long b0 = (long long)blockIdx.x * blocks_per_cta;
  const long long b1 = (b0 + blocks_per_cta < blocks) ? b0 + blocks_per_cta : blocks;
  float acc[N] = {};
  float amax = 0.f;
  if (rl < lanes) {
    for (long long b = b0 + rl; b < b1; b += lanes) {
      const unsigned bu = (unsigned)b;
      const int bj = (int)(bu % (unsigned)BW), bi = (int)((bu / (unsigned)BW) % (unsigned)BH);
      const long long f = bu / (unsigned)(BW * BH);
      typename V::Tags am[4]; Raw dv[4], yv[4]; bool wok[4], pok[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int oy = bi - 1 + (q >> 1), ox = bj - 1 + (q & 1);
        wok[q] = oy >= 0 && oy < OH && ox >= 0 && ox < OW;
        if (wok[q]) {
          const long long op = (f * OH + oy) * OW + ox;
          am[q] = __ldg(reinterpret_cast<const typename V::Tags*>(argmax + op * C + g * N));
          dv[q] = ldv(dpool + op * ppitch + pcoff + g * N);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int iy = 2 * bi + (q >> 1), ix = 2 * bj + (q & 1);
        pok[q] = iy < H && ix < W;
        if (pok[q]) yv[q] = ldv(y + ((f * H + iy) * W + ix) * ypitch + ycoff + g * N);
      }
      typename V::BlockSum bsum;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!pok[q]) continue;
        const int a = q >> 1, c = q & 1;
        Raw d{};
#pragma unroll
        for (int wq = 0; wq < 4; ++wq) {
          const int u = wq >> 1, v = wq & 1;
          if (!((u == 1 || a == 0) && (v == 1 || c == 0))) continue;      // compile-time: this window never covers the pixel
          if (!wok[wq]) continue;
          V::gather(d, am[wq], dv[wq], (uint32_t)((a + 2 - 2 * u) * 3 + (c + 2 - 2 * v)));
        }
        bsum.mask_add(acc, d, yv[q]);
        const int iy = 2 * bi + a, ix = 2 * bj + c;
        const long long px = (f * H + iy) * W + ix;
        if (write_back) *reinterpret_cast<Raw*>(dz + px * dpitch + dcoff + g * N) = d;
        if (hi) V::grad_planes(hi + px * hpitch + hcoff + g * N, lo_off, d, scale, amax);
      }
      bsum.flush(acc);
    }
#pragma unroll
    for (int j = 0; j < N; ++j) red[rl * C + g * N + j] = acc[j];
  }
  if (flag && !(amax <= HALF_MAX)) *flag = 1;
  colsum_tail(red, lanes, partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

}  // namespace

// ---- launchers ---------------------------------------------------------------------------------------------------
// the names the per-launch timing records
template <typename T> static const char* name(const char* f4, const char* h8) { return std::is_same<T, float>::value ? f4 : h8; }
template <typename T> static T* ptr(const View& v) { return reinterpret_cast<T*>(v.base); }
static unsigned nblk(long long n, int t) { return (unsigned)((n + t - 1) / t); }
template <typename T> static bool aligned(const View& v) { return v.pitch % VEC_WIDTH<T> == 0 && v.coff % VEC_WIDTH<T> == 0; }
// a planes view (or none) the kernel can write: hi + lo planes in 16-byte groups, and only where the storage has planes
template <typename T> static bool planes_ok(const View& pl) { return !pl.base || (Vec<T>::PLANES && pl.lo_off && aligned<T>(pl)); }
// ... that the pools address with the offsets of their fp32 output
template <typename T> static bool planes_like(const View& pl, const View& v) {
  return planes_ok<T>(pl) && (!pl.base || (pl.pitch == v.pitch && pl.coff == v.coff && pl.C == v.C));
}
static int unsupported(const char* what) { set_thread_error(std::string(what) + ": unsupported view"); return 1; }
// CTAs of the column-sum passes: about `per` items each, at most `cap`, `max_ctas` (the partials' room) and `n`; none idle
static int colsum_ctas(long long n, int per, int cap, int max_ctas, long long* per_cta) {
  int ctas = (int)((n + per - 1) / per);
  if (ctas > cap) ctas = cap;
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  *per_cta = (n + ctas - 1) / ctas;
  return (int)((n + *per_cta - 1) / *per_cta);
}

template <typename T>
int launch_maxpool_fwd_vec(View src, View dst, View dst_planes, int F, int k, int stride, int pad, uint8_t* argmax, cudaStream_t s) {
  const char* what = name<T>("maxpool_fwd_f4", "maxpool_fwd_h8");
  if (k != 3 || src.C % VEC_WIDTH<T> || !aligned<T>(src) || !aligned<T>(dst) || !planes_like<T>(dst_planes, dst)) return unsupported(what);
  const long long n = (long long)F * dst.H * dst.W * (src.C / VEC_WIDTH<T>);
  maxpool_fwd_vec<T><<<nblk(n, 256), 256, 0, s>>>(ptr<T>(src), src.H, src.W, src.C, src.pitch, src.coff, ptr<T>(dst), dst.H, dst.W, dst.pitch,
                                                  dst.coff, ptr<__half>(dst_planes), dst_planes.lo_off, stride, pad, F, argmax);
  SSNB_LAUNCH_CHECK(what);
  return 0;
}
template <typename T>
int launch_maxpool_bwd_vec(View dsrc, View ddst, int F, int k, int stride, int pad, const uint8_t* argmax, int accumulate, cudaStream_t s) {
  const char* what = name<T>("maxpool_bwd_f4", "maxpool_bwd_h8");
  if (dsrc.C % VEC_WIDTH<T> || !aligned<T>(dsrc) || !aligned<T>(ddst)) return unsupported(what);
  const long long n = (long long)F * dsrc.H * dsrc.W * (dsrc.C / VEC_WIDTH<T>);
  maxpool_bwd_vec<T><<<nblk(n, 256), 256, 0, s>>>(ptr<T>(dsrc), dsrc.H, dsrc.W, dsrc.C, dsrc.pitch, dsrc.coff, ptr<T>(ddst), ddst.H, ddst.W,
                                                  ddst.pitch, ddst.coff, F, k, stride, pad, argmax, accumulate);
  SSNB_LAUNCH_CHECK(what);
  return 0;
}
template <typename T> int launch_avgpool3_vec(View src, View dst, View dst_planes, int F, int accumulate, cudaStream_t s) {
  const char* what = name<T>("avgpool3_pair_f4", "avgpool3_pair_h8");
  if (src.C % VEC_WIDTH<T> || !aligned<T>(src) || !aligned<T>(dst) || !planes_like<T>(dst_planes, dst)) return unsupported(what);
  const long long n2 = (long long)F * ((src.W + 1) / 2) * (src.C / VEC_WIDTH<T>);
  avgpool3_pair_vec<T><<<nblk(n2, 128), 128, 0, s>>>(ptr<T>(src), src.H, src.W, src.C, src.pitch, src.coff, ptr<T>(dst), dst.pitch, dst.coff,
                                                     ptr<__half>(dst_planes), dst_planes.lo_off, F, accumulate);
  SSNB_LAUNCH_CHECK(what);
  return 0;
}
template <typename T>
int launch_mask_bias_vec(View dy, View y, View planes, float scale, int write_back, int* flag, int F, const float* mult, float out_scale,
                         const float* unscale, float* partial, int max_ctas, float* db, int accumulate, cudaStream_t s) {
  const char* what = name<T>("mask_bias_split_f4", "mask_bias_h8");
  const int C = dy.C, N = VEC_WIDTH<T>;
  if (C % N || C / N > MB_THREADS || !aligned<T>(dy) || (y.base && !aligned<T>(y)) || !planes_ok<T>(planes)) return unsupported(what);
  const long long rows = (long long)F * dy.H * dy.W;
  long long rpc;
  const int ctas = colsum_ctas(rows, 256, Vec<T>::MASK_CTAS, max_ctas, &rpc);
  const int lanes = MB_THREADS / (C / N);
  mask_bias_vec<T><<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(ptr<T>(dy), dy.pitch, dy.coff, ptr<T>(y), y.pitch, y.coff, ptr<__half>(planes),
                                                                   planes.pitch, planes.coff, planes.lo_off, scale, write_back, flag, rows, C, rpc,
                                                                   partial + 64, reinterpret_cast<unsigned*>(partial), mult, out_scale, unscale,
                                                                   db, accumulate);
  SSNB_LAUNCH_CHECK(what);
  return 0;
}
template <typename T>
int launch_pool_mask_bias_vec(View dz, View y, View dpool, View planes, float scale, int write_back, int* flag, int F, int k, int stride, int pad,
                              const uint8_t* argmax, const float* mult, float out_scale, const float* unscale, float* partial, int max_ctas,
                              float* db, int accumulate, cudaStream_t s) {
  const char* what = name<T>("pool_mask_bias_split2x2_f4", "pool_mask_bias2x2_h8");
  const int C = dz.C, N = VEC_WIDTH<T>;
  if (k != 3 || stride != 2 || pad != 0 || C % N || C / N > MB_THREADS || !aligned<T>(dz) || !aligned<T>(y) || !aligned<T>(dpool) ||
      !planes_ok<T>(planes))
    return unsupported(what);
  const long long blocks = (long long)F * ((dz.H + 1) / 2) * ((dz.W + 1) / 2);
  long long bpc;
  const int ctas = colsum_ctas(blocks, 64, 888, max_ctas, &bpc);
  const int lanes = MB_THREADS / (C / N);
  pool_mask_bias2x2_vec<T><<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(ptr<T>(dz), dz.pitch, dz.coff, ptr<T>(y), y.pitch, y.coff, dz.H, dz.W,
                                                                           ptr<T>(dpool), dpool.H, dpool.W, dpool.pitch, dpool.coff, argmax,
                                                                           ptr<__half>(planes), planes.pitch, planes.coff, planes.lo_off, scale,
                                                                           write_back, flag, blocks, C, bpc, partial + 64,
                                                                           reinterpret_cast<unsigned*>(partial), mult, out_scale, unscale, db,
                                                                           accumulate);
  SSNB_LAUNCH_CHECK(what);
  return 0;
}

#define INST(T)                                                                                                                       \
  template int launch_maxpool_fwd_vec<T>(View, View, View, int, int, int, int, uint8_t*, cudaStream_t);                               \
  template int launch_maxpool_bwd_vec<T>(View, View, int, int, int, int, const uint8_t*, int, cudaStream_t);                          \
  template int launch_avgpool3_vec<T>(View, View, View, int, int, cudaStream_t);                                                     \
  template int launch_mask_bias_vec<T>(View, View, View, float, int, int*, int, const float*, float, const float*, float*, int, float*, \
                                       int, cudaStream_t);                                                                            \
  template int launch_pool_mask_bias_vec<T>(View, View, View, View, float, int, int*, int, int, int, int, const uint8_t*, const float*, \
                                            float, const float*, float*, int, float*, int, cudaStream_t);
INST(float)
INST(__half)

}  // namespace ssnb
