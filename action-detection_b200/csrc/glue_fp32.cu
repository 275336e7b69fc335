// SSNB_EXACT_TC memory-bound glue over fp32 NHWC views, vectorised: every thread moves 4 channels (16 bytes), and the
// kernels that produce a convolution operand also write its fp16 hi / lo planes (tc_glue.cu has the definition), so no
// separate split pass runs.  Same semantics as the generic kernels in simt_glue.cu (Caffe ceil-mode pooling,
// model_zoo/bninception/layer_factory.py:41-53; first-max-wins arg-max; 3x3 average with count_include_pad) -- these are
// the fp32 counterparts of glue_fp16.cu.
#include "common.cuh"

namespace ssnb {
namespace {

constexpr float HALF_MAX = 65504.f;

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// 4 fp32 values -> 8 bytes of hi + 8 bytes of lo at the same element offset of the two planes
__device__ __forceinline__ void store_planes4(__half* hi, long long lo_off, const float4& v) {
  uint2 h, l;
  split2(v.x, v.y, h.x, l.x);
  split2(v.z, v.w, h.y, l.y);
  *reinterpret_cast<uint2*>(hi) = h;
  *reinterpret_cast<uint2*>(reinterpret_cast<char*>(hi) + lo_off) = l;
}

// ---- max pooling ---------------------------------------------------------------------------------------------
// K > 0: compile-time window size (every max pool of the network is 3x3): all K*K loads are issued before the first compare
// (the generic loop waits for each load in turn); the compare order -- and with it the first-max-wins / NaN rule -- is the same
template <int K>
__global__ void maxpool_fwd_f4(const float* __restrict__ src, int H, int W, int C, int spitch, int scoff, float* __restrict__ dst, int OH,
                               int OW, int dpitch, int dcoff, __half* __restrict__ hi, long long lo_off, int F, int k_rt, int stride, int pad,
                               uint8_t* __restrict__ argmax) {
  const int k = K ? K : k_rt;
  const int G = C / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * OH * OW * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ox = (int)(pu % (unsigned)OW), oy = (int)((pu / (unsigned)OW) % (unsigned)OH);
  const long long p = pu;
  const long long f = pu / (unsigned)(OW * OH);
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  uint32_t bi = 0u;                                   // four 8-bit tap indices
  bool first = true;
  const float* base = src + (f * H * W) * spitch + scoff + g * 4;
  if (K) {
    constexpr int KK = K ? K * K : 1;
    float4 q[KK]; bool ok[KK];
#pragma unroll
    for (int t = 0; t < KK; ++t) {
      const int iy = oy * stride + t / (K ? K : 1) - pad, ix = ox * stride + t % (K ? K : 1) - pad;
      ok[t] = iy >= 0 && iy < H && ix >= 0 && ix < W;
      q[t] = ok[t] ? ldg4(base + ((long long)iy * W + ix) * spitch) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int t = 0; t < KK; ++t) {
      if (!ok[t]) continue;
      const float v[4] = {q[t].x, q[t].y, q[t].z, q[t].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (first || v[j] > best[j] || v[j] != v[j]) { best[j] = v[j]; bi = (bi & ~(0xFFu << (8 * j))) | ((uint32_t)t << (8 * j)); }   // first max wins (ATen)
      first = false;
    }
  } else {
  for (int r = 0; r < k; ++r) {
    const int iy = oy * stride + r - pad;
    if (iy < 0 || iy >= H) continue;
    for (int s = 0; s < k; ++s) {
      const int ix = ox * stride + s - pad;
      if (ix < 0 || ix >= W) continue;
      const float4 q = ldg4(base + ((long long)iy * W + ix) * spitch);
      const float v[4] = {q.x, q.y, q.z, q.w};
      const uint32_t tag = (uint32_t)(r * k + s);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (first || v[j] > best[j] || v[j] != v[j]) { best[j] = v[j]; bi = (bi & ~(0xFFu << (8 * j))) | (tag << (8 * j)); }   // first max wins (ATen)
      first = false;
    }
  }
  }
  const float4 o = make_float4(best[0], best[1], best[2], best[3]);
  *reinterpret_cast<float4*>(dst + p * dpitch + dcoff + g * 4) = o;
  if (hi) store_planes4(hi + p * dpitch + dcoff + g * 4, lo_off, o);
  *reinterpret_cast<uint32_t*>(argmax + p * C + g * 4) = bi;
}

__global__ void maxpool_bwd_f4(float* __restrict__ dsrc, int H, int W, int C, int spitch, int scoff, const float* __restrict__ ddst, int OH,
                               int OW, int dpitch, int dcoff, int F, int k, int stride, int pad, const uint8_t* __restrict__ argmax,
                               int accumulate) {
  const int G = C / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * H * W * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int ix = (int)(pu % (unsigned)W), iy = (int)((pu / (unsigned)W) % (unsigned)H);
  const long long p = pu;
  const long long f = pu / (unsigned)(W * H);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  // windows covering this pixel: oy in [ceil((iy+pad-k+1)/stride), floor((iy+pad)/stride)]
  const int ty0 = iy + pad - k + 1, tx0 = ix + pad - k + 1;
  const int oy_lo = ty0 > 0 ? (ty0 + stride - 1) / stride : 0, oy_hi = min((iy + pad) / stride, OH - 1);
  const int ox_lo = tx0 > 0 ? (tx0 + stride - 1) / stride : 0, ox_hi = min((ix + pad) / stride, OW - 1);
  if (oy_hi - oy_lo <= 1 && ox_hi - ox_lo <= 1) {
    // stride-2 pools: at most 2x2 covering windows -> every load is issued before the first use
    uint32_t am[4]; float4 dv[4]; uint32_t tg[4]; bool ok[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int oy = oy_lo + (q >> 1), ox = ox_lo + (q & 1);
      ok[q] = oy <= oy_hi && ox <= ox_hi;
      const long long op = (f * OH + (ok[q] ? oy : oy_lo)) * OW + (ok[q] ? ox : ox_lo);
      tg[q] = (uint32_t)((iy + pad - oy * stride) * k + (ix + pad - ox * stride));
      am[q] = __ldg(reinterpret_cast<const uint32_t*>(argmax + op * C + g * 4));
      dv[q] = ldg4(ddst + op * dpitch + dcoff + g * 4);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!ok[q]) continue;
      const float v[4] = {dv[q].x, dv[q].y, dv[q].z, dv[q].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (((am[q] >> (8 * j)) & 0xFFu) == tg[q]) acc[j] += v[j];
    }
  } else {
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      const int r = iy + pad - oy * stride;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const int s = ix + pad - ox * stride;
        const long long op = (f * OH + oy) * OW + ox;
        const uint32_t a = __ldg(reinterpret_cast<const uint32_t*>(argmax + op * C + g * 4));
        const uint32_t tag = (uint32_t)(r * k + s);
        const uint32_t xa = a ^ (tag * 0x01010101u);
        if (!((xa - 0x01010101u) & ~xa & 0x80808080u)) continue;      // none of the 4 channels of this window points here
        const float4 d4 = ldg4(ddst + op * dpitch + dcoff + g * 4);
        const float v[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (((a >> (8 * j)) & 0xFFu) == tag) acc[j] += v[j];
      }
    }
  }
  float* q = dsrc + p * spitch + scoff + g * 4;
  if (accumulate) {
    const float4 o = *reinterpret_cast<const float4*>(q);
    acc[0] += o.x; acc[1] += o.y; acc[2] += o.z; acc[3] += o.w;
  }
  *reinterpret_cast<float4*>(q) = make_float4(acc[0], acc[1], acc[2], acc[3]);
}

// ---- 3x3 stride-1 pad-1 average (count_include_pad: always /9; its own adjoint) ---------------------------------------
// one thread per (frame, column PAIR, 4-channel group) walks down the rows keeping the horizontal 3-sums of the last
// three rows; the two columns share the loads and the middle partial sum (see glue_fp16.cu).  The division is a true
// fp32 division by 9 like ATen's (s / 9), applied to the 9-term sum.
__global__ void avgpool3_pair_f4(const float* __restrict__ src, int H, int W, int C, int spitch, int scoff, float* __restrict__ dst,
                                 int dpitch, int dcoff, __half* __restrict__ hi, long long lo_off, int F, int accumulate) {
  const int G = C / 4, W2 = (W + 1) / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * W2 * G) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const int x = 2 * (int)((iu / (unsigned)G) % (unsigned)W2);
  const long long f = iu / (unsigned)(G * W2);
  const bool has1 = x + 1 < W;
  float p0[4], c0[4], n0[4], p1[4], c1[4], n1[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { p0[j] = c0[j] = p1[j] = c1[j] = 0.f; }
  auto rowsum = [&](int y, float* o0, float* o1) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { o0[j] = 0.f; o1[j] = 0.f; }
    if (y >= H) return;
    const float* base = src + ((f * H + y) * W) * spitch + scoff + g * 4;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a = x - 1 >= 0 ? ldg4(base + (long long)(x - 1) * spitch) : z;
    const float4 b = ldg4(base + (long long)x * spitch);
    const float4 c = x + 1 < W ? ldg4(base + (long long)(x + 1) * spitch) : z;
    const float4 d = x + 2 < W ? ldg4(base + (long long)(x + 2) * spitch) : z;
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w}, cv[4] = {c.x, c.y, c.z, c.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float m = bv[j] + cv[j];
      o0[j] = av[j] + m;
      o1[j] = m + dv[j];
    }
  };
  rowsum(0, c0, c1);
  for (int y = 0; y < H; ++y) {
    rowsum(y + 1, n0, n1);
    float s0[4], s1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      s0[j] = (p0[j] + c0[j] + n0[j]) / 9.0f;
      s1[j] = (p1[j] + c1[j] + n1[j]) / 9.0f;
    }
    float* o = dst + ((f * H + y) * W + x) * dpitch + dcoff + g * 4;
    if (accumulate) {
      const float4 old = *reinterpret_cast<const float4*>(o);
      s0[0] += old.x; s0[1] += old.y; s0[2] += old.z; s0[3] += old.w;
      if (has1) {
        const float4 old1 = *reinterpret_cast<const float4*>(o + dpitch);
        s1[0] += old1.x; s1[1] += old1.y; s1[2] += old1.z; s1[3] += old1.w;
      }
    }
    const float4 v0 = make_float4(s0[0], s0[1], s0[2], s0[3]), v1 = make_float4(s1[0], s1[1], s1[2], s1[3]);
    *reinterpret_cast<float4*>(o) = v0;
    if (has1) *reinterpret_cast<float4*>(o + dpitch) = v1;
    if (hi) {
      __half* hp = hi + ((f * H + y) * W + x) * dpitch + dcoff + g * 4;
      store_planes4(hp, lo_off, v0);
      if (has1) store_planes4(hp + dpitch, lo_off, v1);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { p0[j] = c0[j]; c0[j] = n0[j]; p1[j] = c1[j]; c1[j] = n1[j]; }
  }
}

// ---- backward pass of a convolution's output gradient: ReLU mask + bias-gradient column sums + operand planes ----------
//   dz = dy * (y > 0);  partial[cta][c] = sum_rows dz;  planes = hi/lo of dz * scale  (the tensor-core weight / data
//   gradients read the planes; the fp32 dz is written back only on request)
constexpr int MB_THREADS = 256;
// the last CTA to finish reduces the per-CTA partials in CTA order (deterministic) into db
__device__ __forceinline__ void colsum_tail(float* __restrict__ partial, unsigned* __restrict__ counter, int C, const float* __restrict__ mult,
                                            float out_scale, const float* __restrict__ unscale, float* __restrict__ db, bool* is_last,
                                            int accumulate) {
  if (!db) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!*is_last) return;
  __threadfence();
  const int n = (int)gridDim.x;
  if (unscale) out_scale *= __ldg(unscale);
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
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

__global__ void __launch_bounds__(MB_THREADS) mask_bias_split_f4(float* __restrict__ dy, int dpitch, int dcoff, const float* __restrict__ y,
                                                                 int ypitch, int ycoff, __half* __restrict__ hi, int hpitch, int hcoff,
                                                                 long long lo_off, float scale, int write_f32, int* __restrict__ flag,
                                                                 long long rows, int C, long long rows_per_cta, float* __restrict__ partial,
                                                                 unsigned* __restrict__ counter, const float* __restrict__ mult,
                                                                 float out_scale, const float* __restrict__ unscale, float* __restrict__ db,
                                                                 int accumulate) {
  extern __shared__ float red[];                 // [lanes][C]
  __shared__ bool is_last;
  const int G = C / 4;
  const int lanes = MB_THREADS / G;               // row lanes per CTA (G <= 256)
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = (r0 + rows_per_cta < rows) ? r0 + rows_per_cta : rows;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float amax = 0.f;
  if (rl < lanes) {
    constexpr int U = 8;                          // rows in flight per thread
    for (long long rb = r0 + rl; rb < r1; rb += (long long)lanes * U) {
      float4 dv[U], yv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r < r1) {
          dv[u] = *reinterpret_cast<const float4*>(dy + r * dpitch + dcoff + g * 4);
          if (y) yv[u] = ldg4(y + r * ypitch + ycoff + g * 4);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long r = rb + (long long)u * lanes;
        if (r >= r1) continue;
        float d[4] = {dv[u].x, dv[u].y, dv[u].z, dv[u].w};
        bool changed = false;
        if (y) {                                  // y == nullptr: no ReLU behind this convolution (column sums / planes only)
          const float a[4] = {yv[u].x, yv[u].y, yv[u].z, yv[u].w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (!(a[j] > 0.f)) { changed = changed || (d[j] != 0.f); d[j] = 0.f; }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += d[j];
        if (write_f32 && changed) *reinterpret_cast<float4*>(dy + r * dpitch + dcoff + g * 4) = make_float4(d[0], d[1], d[2], d[3]);
        if (hi) {
          const float4 sv = make_float4(d[0] * scale, d[1] * scale, d[2] * scale, d[3] * scale);
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(sv.x), fabsf(sv.y)), fmaxf(fabsf(sv.z), fabsf(sv.w))));
          if (sv.x != sv.x || sv.y != sv.y || sv.z != sv.z || sv.w != sv.w) amax = INFINITY;
          store_planes4(hi + r * hpitch + hcoff + g * 4, lo_off, sv);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) red[rl * C + g * 4 + j] = acc[j];
  }
  if (flag && !(amax <= HALF_MAX)) *flag = 1;      // the loss scale pushed a gradient beyond the fp16 range (or a NaN arrived)
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
  colsum_tail(partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

// Same pass for a convolution whose only consumer is a k3/s2/pad0 max pool (conv1 -> pool1, conv2_3x3 -> pool2): the pool's
// backward gather is folded in, so the full-resolution fp32 dy tensor is neither written by a pooling kernel nor re-read:
//   dz[p] = (sum over covering windows whose arg-max is p of dpool) * (y[p] > 0)
// Works on 2x2 input blocks: block (2i..2i+1, 2j..2j+1) is covered by the four windows (i-1..i, j-1..j) only, so one thread
// loads 4 windows + 4 activations for 4 outputs with 12 independent loads in flight (see glue_fp16.cu).
__global__ void __launch_bounds__(MB_THREADS) pool_mask_bias_split2x2_f4(float* __restrict__ dz, int dpitch, int dcoff, const float* __restrict__ y,
                                                                         int ypitch, int ycoff, int H, int W, const float* __restrict__ dpool, int OH,
                                                                         int OW, int ppitch, int pcoff, const uint8_t* __restrict__ argmax,
                                                                         __half* __restrict__ hi, int hpitch, int hcoff, long long lo_off, float scale,
                                                                         int write_f32, int* __restrict__ flag, long long blocks, int C,
                                                                         long long blocks_per_cta, float* __restrict__ partial,
                                                                         unsigned* __restrict__ counter, const float* __restrict__ mult,
                                                                         float out_scale, const float* __restrict__ unscale, float* __restrict__ db,
                                                                         int accumulate) {
  extern __shared__ float red[];
  __shared__ bool is_last;
  const int G = C / 4;
  const int lanes = MB_THREADS / G;
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const int BH = (H + 1) / 2, BW = (W + 1) / 2;
  const long long b0 = (long long)blockIdx.x * blocks_per_cta;
  const long long b1 = (b0 + blocks_per_cta < blocks) ? b0 + blocks_per_cta : blocks;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float amax = 0.f;
  if (rl < lanes) {
    for (long long b = b0 + rl; b < b1; b += lanes) {
      const unsigned bu = (unsigned)b;
      const int bj = (int)(bu % (unsigned)BW), bi = (int)((bu / (unsigned)BW) % (unsigned)BH);
      const long long f = bu / (unsigned)(BW * BH);
      uint32_t am[4]; float4 dv[4], yv[4]; bool wok[4], pok[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int oy = bi - 1 + (q >> 1), ox = bj - 1 + (q & 1);
        wok[q] = oy >= 0 && oy < OH && ox >= 0 && ox < OW;
        if (wok[q]) {
          const long long op = (f * OH + oy) * OW + ox;
          am[q] = __ldg(reinterpret_cast<const uint32_t*>(argmax + op * C + g * 4));
          dv[q] = ldg4(dpool + op * ppitch + pcoff + g * 4);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int iy = 2 * bi + (q >> 1), ix = 2 * bj + (q & 1);
        pok[q] = iy < H && ix < W;
        if (pok[q]) yv[q] = ldg4(y + ((f * H + iy) * W + ix) * ypitch + ycoff + g * 4);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (!pok[q]) continue;
        const int a = q >> 1, c = q & 1;
        float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int wq = 0; wq < 4; ++wq) {
          const int u = wq >> 1, v = wq & 1;
          if (!((u == 1 || a == 0) && (v == 1 || c == 0))) continue;      // compile-time: this window never covers the pixel
          if (!wok[wq]) continue;
          const uint32_t tag = (uint32_t)((a + 2 - 2 * u) * 3 + (c + 2 - 2 * v));
          const float t[4] = {dv[wq].x, dv[wq].y, dv[wq].z, dv[wq].w};
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (((am[wq] >> (8 * j)) & 0xFFu) == tag) d[j] += t[j];
        }
        const float yy[4] = {yv[q].x, yv[q].y, yv[q].z, yv[q].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (!(yy[j] > 0.f)) d[j] = 0.f;
          acc[j] += d[j];
        }
        const int iy = 2 * bi + a, ix = 2 * bj + c;
        const long long px = (f * H + iy) * W + ix;
        if (write_f32) *reinterpret_cast<float4*>(dz + px * dpitch + dcoff + g * 4) = make_float4(d[0], d[1], d[2], d[3]);
        if (hi) {
          const float4 sv = make_float4(d[0] * scale, d[1] * scale, d[2] * scale, d[3] * scale);
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(sv.x), fabsf(sv.y)), fmaxf(fabsf(sv.z), fabsf(sv.w))));
          if (sv.x != sv.x || sv.y != sv.y || sv.z != sv.z || sv.w != sv.w) amax = INFINITY;
          store_planes4(hi + px * hpitch + hcoff + g * 4, lo_off, sv);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) red[rl * C + g * 4 + j] = acc[j];
  }
  if (flag && !(amax <= HALF_MAX)) *flag = 1;
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += MB_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * C + c];
    partial[(long long)blockIdx.x * C + c] = s;
  }
  colsum_tail(partial, counter, C, mult, out_scale, unscale, db, &is_last, accumulate);
}

}  // namespace

#define FP(v) reinterpret_cast<float*>((v).base)
static inline unsigned nblk(long long n, int t) { return (unsigned)((n + t - 1) / t); }
static inline bool planes_match(const View& f32, const View& pl) {
  return !pl.base || (pl.lo_off && pl.pitch == f32.pitch && pl.coff == f32.coff && pl.C == f32.C);
}

int launch_maxpool_fwd_f4(View src, View dst, View dst_planes, int F, int k, int stride, int pad, uint8_t* argmax, cudaStream_t s) {
  if (src.C % 4 || src.pitch % 4 || src.coff % 4 || dst.pitch % 4 || dst.coff % 4 || k * k > 255 || !planes_match(dst, dst_planes)) {
    set_thread_error("maxpool_fwd_f4: unsupported view"); return 1; }
  const long long n = (long long)F * dst.H * dst.W * (src.C / 4);
  if (k == 3)
    maxpool_fwd_f4<3><<<nblk(n, 256), 256, 0, s>>>(FP(src), src.H, src.W, src.C, src.pitch, src.coff, FP(dst), dst.H, dst.W, dst.pitch, dst.coff,
                                                  (__half*)dst_planes.base, dst_planes.lo_off, F, k, stride, pad, argmax);
  else
    maxpool_fwd_f4<0><<<nblk(n, 256), 256, 0, s>>>(FP(src), src.H, src.W, src.C, src.pitch, src.coff, FP(dst), dst.H, dst.W, dst.pitch, dst.coff,
                                                  (__half*)dst_planes.base, dst_planes.lo_off, F, k, stride, pad, argmax);
  SSNB_LAUNCH_CHECK("maxpool_fwd_f4");
  return 0;
}
int launch_maxpool_bwd_f4(View dsrc, View ddst, int F, int k, int stride, int pad, const uint8_t* argmax, int accumulate, cudaStream_t s) {
  if (dsrc.C % 4 || dsrc.pitch % 4 || dsrc.coff % 4 || ddst.pitch % 4 || ddst.coff % 4) { set_thread_error("maxpool_bwd_f4: unsupported view"); return 1; }
  const long long n = (long long)F * dsrc.H * dsrc.W * (dsrc.C / 4);
  maxpool_bwd_f4<<<nblk(n, 256), 256, 0, s>>>(FP(dsrc), dsrc.H, dsrc.W, dsrc.C, dsrc.pitch, dsrc.coff, FP(ddst), ddst.H, ddst.W, ddst.pitch,
                                             ddst.coff, F, k, stride, pad, argmax, accumulate);
  SSNB_LAUNCH_CHECK("maxpool_bwd_f4");
  return 0;
}
int launch_avgpool3_f4(View src, View dst, View dst_planes, int F, int accumulate, cudaStream_t s) {
  if (src.C % 4 || src.pitch % 4 || src.coff % 4 || dst.pitch % 4 || dst.coff % 4 || !planes_match(dst, dst_planes)) {
    set_thread_error("avgpool3_f4: unsupported view"); return 1; }
  const long long n2 = (long long)F * ((src.W + 1) / 2) * (src.C / 4);
  avgpool3_pair_f4<<<nblk(n2, 128), 128, 0, s>>>(FP(src), src.H, src.W, src.C, src.pitch, src.coff, FP(dst), dst.pitch, dst.coff,
                                                (__half*)dst_planes.base, dst_planes.lo_off, F, accumulate);
  SSNB_LAUNCH_CHECK("avgpool3_pair_f4");
  return 0;
}
// partial must hold 64 + max_ctas * C floats (first 256 bytes: completion counter); db may be nullptr (mask / planes only)
int launch_mask_bias_split_f4(View dy, View y, View planes, float scale, int write_f32, int* flag, int F, const float* mult, float out_scale,
                              const float* unscale, float* partial, int max_ctas, float* db, int accumulate, cudaStream_t s) {
  const long long rows = (long long)F * dy.H * dy.W;
  const int C = dy.C;
  if (C % 4 || C / 4 > MB_THREADS || dy.pitch % 4 || dy.coff % 4 || (y.base && (y.pitch % 4 || y.coff % 4)) || (planes.base && (!planes.lo_off || planes.pitch % 4 || planes.coff % 4))) {
    set_thread_error("mask_bias_split_f4: unsupported view"); return 1; }
  int ctas = (int)((rows + 255) / 256);
  if (ctas > 592) ctas = 592;                      // four CTAs per SM
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  const long long rpc = (rows + ctas - 1) / ctas;
  ctas = (int)((rows + rpc - 1) / rpc);
  const int lanes = MB_THREADS / (C / 4);
  unsigned* counter = reinterpret_cast<unsigned*>(partial);
  float* part = partial + 64;
  mask_bias_split_f4<<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(FP(dy), dy.pitch, dy.coff, FP(y), y.pitch, y.coff, (__half*)planes.base,
                                                                    planes.pitch, planes.coff, planes.lo_off, scale, write_f32, flag, rows, C, rpc,
                                                                    part, counter, mult, out_scale, unscale, db, accumulate);
  SSNB_LAUNCH_CHECK("mask_bias_split_f4");
  return 0;
}

// conv output y / dz views at full resolution; dpool = fp32 gradient of the k3/s2/pad0 max pool's output, argmax from its forward
int launch_pool_mask_bias_split_f4(View dz, View y, View dpool, View planes, float scale, int write_f32, int* flag, int F, const uint8_t* argmax,
                                   const float* mult, float out_scale, const float* unscale, float* partial, int max_ctas, float* db, int accumulate,
                                   cudaStream_t s) {
  const int C = dz.C;
  if (C % 4 || C / 4 > MB_THREADS || dz.pitch % 4 || dz.coff % 4 || y.pitch % 4 || y.coff % 4 || dpool.pitch % 4 || dpool.coff % 4 ||
      (planes.base && (!planes.lo_off || planes.pitch % 4 || planes.coff % 4))) { set_thread_error("pool_mask_bias_split_f4: unsupported view"); return 1; }
  const long long blocks = (long long)F * ((dz.H + 1) / 2) * ((dz.W + 1) / 2);
  int ctas = (int)((blocks + 63) / 64);
  if (ctas > 888) ctas = 888;
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  const long long bpc = (blocks + ctas - 1) / ctas;
  ctas = (int)((blocks + bpc - 1) / bpc);
  const int lanes = MB_THREADS / (C / 4);
  unsigned* counter = reinterpret_cast<unsigned*>(partial);
  float* part = partial + 64;
  pool_mask_bias_split2x2_f4<<<ctas, MB_THREADS, (size_t)lanes * C * 4, s>>>(FP(dz), dz.pitch, dz.coff, FP(y), y.pitch, y.coff, dz.H, dz.W, FP(dpool),
                                                                            dpool.H, dpool.W, dpool.pitch, dpool.coff, argmax, (__half*)planes.base,
                                                                            planes.pitch, planes.coff, planes.lo_off, scale, write_f32, flag, blocks, C,
                                                                            bpc, part, counter, mult, out_scale, unscale, db, accumulate);
  SSNB_LAUNCH_CHECK("pool_mask_bias_split2x2_f4");
  return 0;
}

}  // namespace ssnb
