// STPP, the three linear heads, and the multi-task loss of SSN — all fp32 (HBM/latency-bound work).
// Reference: ops/ssn_ops.py:22-79 (STPP), :82-170 (STPPReorgainzed), :173-258 (losses);
// ssn_models.py:272-289 (heads + row selection); ssn_train.py:210-214 (loss mix).
#include <climits>
#include <cstring>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int MAX_PARTS = 32;
struct PartTable { int n; int lo[MAX_PARTS], hi[MAX_PARTS], norm[MAX_PARTS], col[MAX_PARTS]; int clo, chi; };

// one thread per (proposal, feature); sequential sums keep the reference's rounding order
__global__ void stpp_fwd_kernel(const float* __restrict__ ft, const float* __restrict__ scaling, int n, int S, int D,
                                PartTable pt, float* __restrict__ course, float* __restrict__ stpp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * D) return;
  const int d = (int)(i % D);
  const long long p = i / D;
  const float* row = ft + (p * S) * D + d;
  for (int q = 0; q < pt.n; ++q) {
    float s = 0.f;
    for (int t = pt.lo[q]; t < pt.hi[q]; ++t) s += row[(long long)t * D];
    float m = s / (float)(pt.hi[q] - pt.lo[q]);       // mean (0/0 = NaN for an empty part, like torch)
    m = m / (float)pt.norm[q];
    if (pt.col[q] >= 0) m = m * scaling[p * 2 + pt.col[q]];
    stpp[(p * pt.n + q) * D + d] = m;
  }
  float s = 0.f;
  for (int t = pt.clo; t < pt.chi; ++t) s += row[(long long)t * D];
  course[p * D + d] = s / (float)(pt.chi - pt.clo);
}

__global__ void stpp_bwd_kernel(const float* __restrict__ dcourse, const float* __restrict__ dstpp,
                                const float* __restrict__ scaling, int n, int S, int D, PartTable pt,
                                float* __restrict__ dft) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * S * D) return;
  const int d = (int)(i % D);
  const int t = (int)((i / D) % S);
  const long long p = i / ((long long)D * S);
  float g = 0.f;
  for (int q = 0; q < pt.n; ++q) {
    if (t < pt.lo[q] || t >= pt.hi[q]) continue;
    float v = dstpp[(p * pt.n + q) * D + d];
    if (pt.col[q] >= 0) v = v * scaling[p * 2 + pt.col[q]];
    v = v / (float)pt.norm[q];
    g += v / (float)(pt.hi[q] - pt.lo[q]);
  }
  if (dcourse && t >= pt.clo && t < pt.chi) g += dcourse[p * D + d] / (float)(pt.chi - pt.clo);
  dft[i] = g;
}

// fused 7x7 global average pool (+ dropout mask) + STPP: one thread per (proposal, channel) walks the
// S snippets, reducing each 49-pixel column in registers; reads the 5b output exactly once.
template <typename T>
__global__ void gpool_stpp_kernel(const T* __restrict__ src, int HW, int C, int pitch, int coff, int n, int S,
                                  const float* __restrict__ mask, const float* __restrict__ scaling, PartTable pt,
                                  float* __restrict__ feat, float* __restrict__ course, float* __restrict__ stpp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * C) return;
  const int c = (int)(i % C);
  const long long p = i / C;
  float pooled[32];
  for (int t = 0; t < S; ++t) {
    const long long f = p * S + t;
    float s = 0.f;
    for (int q = 0; q < HW; ++q) s += to_f<T>(src[(f * HW + q) * pitch + coff + c]);
    float v = s / (float)HW;
    if (mask) v = v * mask[f * C + c];
    pooled[t] = v;
    feat[f * C + c] = v;
  }
  for (int q = 0; q < pt.n; ++q) {
    float s = 0.f;
    for (int t = pt.lo[q]; t < pt.hi[q]; ++t) s += pooled[t];
    float m = s / (float)(pt.hi[q] - pt.lo[q]);
    m = m / (float)pt.norm[q];
    if (pt.col[q] >= 0) m = m * scaling[p * 2 + pt.col[q]];
    stpp[(p * pt.n + q) * C + c] = m;
  }
  float s = 0.f;
  for (int t = pt.clo; t < pt.chi; ++t) s += pooled[t];
  course[p * C + c] = s / (float)(pt.chi - pt.clo);
}


// ---- vectorised STPP (S <= SMAX segments per proposal, D % 4 == 0) --------------------------------------------------
// One thread owns 4 features of one proposal: the S segment vectors are loaded ONCE (S independent 16-byte loads in
// flight) and every pyramid part + the course feature is formed from registers in the reference's order (sequential sum
// over the part's segments, / len, / norm, * scaling: ops/ssn_ops.py:49-64), then stored as 16-byte vectors.  Algorithmic
// traffic only: 61,448 B per proposal for (1,(1,2),1) at D = 1024 (SURVEY section 8d); the scalar kernel above re-read
// every segment once per part that contains it.
template <int SMAX>
__global__ void stpp_fwd_v4_kernel(const float* __restrict__ ft, const float* __restrict__ scaling, int n, int S, int D,
                                   PartTable pt, float* __restrict__ course, float* __restrict__ stpp) {
  const int D4 = D / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * D4) return;
  const int d = (int)(i % D4) * 4;
  const long long p = i / D4;
  const float* row = ft + (p * S) * D + d;
  float4 v[SMAX];
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
    if (t < S) v[t] = __ldg(reinterpret_cast<const float4*>(row + (long long)t * D));
  const float s0 = pt.n ? scaling[p * 2] : 0.f, s1 = pt.n ? scaling[p * 2 + 1] : 0.f;     // no parts: scaling may be NULL
  auto part = [&](int lo, int hi) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < SMAX; ++t)
      if (t < S && t >= lo && t < hi) { s.x += v[t].x; s.y += v[t].y; s.z += v[t].z; s.w += v[t].w; }
    const float len = (float)(hi - lo);             // 0/0 = NaN for an empty part, like torch
    return make_float4(s.x / len, s.y / len, s.z / len, s.w / len);
  };
  for (int q = 0; q < pt.n; ++q) {
    float4 m = part(pt.lo[q], pt.hi[q]);
    const float nm = (float)pt.norm[q];
    m.x /= nm; m.y /= nm; m.z /= nm; m.w /= nm;
    if (pt.col[q] >= 0) { const float sc = pt.col[q] == 0 ? s0 : s1; m.x *= sc; m.y *= sc; m.z *= sc; m.w *= sc; }
    *reinterpret_cast<float4*>(stpp + (p * pt.n + q) * D + d) = m;
  }
  *reinterpret_cast<float4*>(course + p * D + d) = part(pt.clo, pt.chi);
}

// backward: every part gradient is loaded once, each of the S segment gradients is formed in the scalar kernel's order
template <int SMAX, int PMAX>
__global__ void stpp_bwd_v4_kernel(const float* __restrict__ dcourse, const float* __restrict__ dstpp, const float* __restrict__ scaling,
                                   int n, int S, int D, PartTable pt, float* __restrict__ dft) {
  const int D4 = D / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * D4) return;
  const int d = (int)(i % D4) * 4;
  const long long p = i / D4;
  const float s0 = pt.n ? scaling[p * 2] : 0.f, s1 = pt.n ? scaling[p * 2 + 1] : 0.f;     // no parts: scaling may be NULL
  float4 g[PMAX];
#pragma unroll
  for (int q = 0; q < PMAX; ++q)
    if (q < pt.n) {
      float4 v = __ldg(reinterpret_cast<const float4*>(dstpp + (p * pt.n + q) * D + d));
      if (pt.col[q] >= 0) { const float sc = pt.col[q] == 0 ? s0 : s1; v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc; }
      const float nm = (float)pt.norm[q], len = (float)(pt.hi[q] - pt.lo[q]);
      g[q] = make_float4(v.x / nm / len, v.y / nm / len, v.z / nm / len, v.w / nm / len);
    }
  float4 gc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (dcourse) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(dcourse + p * D + d));
    const float len = (float)(pt.chi - pt.clo);
    gc = make_float4(v.x / len, v.y / len, v.z / len, v.w / len);
  }
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    if (t >= S) break;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < PMAX; ++q)
      if (q < pt.n && t >= pt.lo[q] && t < pt.hi[q]) { a.x += g[q].x; a.y += g[q].y; a.z += g[q].z; a.w += g[q].w; }
    if (dcourse && t >= pt.clo && t < pt.chi) { a.x += gc.x; a.y += gc.y; a.z += gc.z; a.w += gc.w; }
    *reinterpret_cast<float4*>(dft + (p * S + t) * D + d) = a;
  }
}

// ---- fused 7x7 global average pool (+ dropout mask) + STPP, second generation ------------------------------------------
// CTA = (proposal, SLAB-channel slab), 256 threads = (16-byte channel groups of the slab) x (pixel lanes): every thread
// accumulates its pixel subset of all S frames in registers (S independent 16-byte loads in flight per pixel step, consecutive
// threads on consecutive 16-byte chunks of a pixel row), the pixel lanes are reduced through shared memory, then thread c forms
// the parts of channel c from the S pooled values.  Reads the 5b output exactly once with n x C/SLAB CTAs in flight (256 at the
// bench shape); the first-generation kernel gave every thread a serial chain of S x HW 2-byte loads.
template <typename T, int SMAX, int SLAB>
__global__ void __launch_bounds__(256) gpool_stpp_v2_kernel(const T* __restrict__ src, int HW, int C, int pitch, int coff, int n, int S,
                                                            const float* __restrict__ mask, const float* __restrict__ scaling, PartTable pt,
                                                            float* __restrict__ feat, float* __restrict__ course, float* __restrict__ stpp) {
  constexpr int VEC = 16 / sizeof(T);              // channels per 16-byte load: 8 (fp16) or 4 (fp32)
  constexpr int G = SLAB / VEC;                    // channel groups per slab
  constexpr int L = 256 / G;                       // pixel lanes
  extern __shared__ float red[];                   // [L][SMAX][SLAB]
  const long long p = blockIdx.x;
  const int c0 = blockIdx.y * SLAB;
  const int g = threadIdx.x % G, l = threadIdx.x / G;
  float acc[SMAX][VEC];
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[t][j] = 0.f;
  const bool live = c0 + g * VEC < C;
  if (live) {
    const T* base = src + (p * S * HW) * pitch + coff + c0 + g * VEC;
    // pixel loop outside, frame loop unrolled inside: S independent 16-byte loads in flight per iteration
    for (int q = l; q < HW; q += L) {
      uint4 r[SMAX];
#pragma unroll
      for (int t = 0; t < SMAX; ++t)
        if (t < S) r[t] = __ldg(reinterpret_cast<const uint4*>(base + ((long long)t * HW + q) * pitch));
#pragma unroll
      for (int t = 0; t < SMAX; ++t) {
        if (t >= S) continue;
        if (sizeof(T) == 2) {
          const __half2* h = reinterpret_cast<const __half2*>(&r[t]);
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float2 f2 = __half22float2(h[j]); acc[t][(2 * j) % VEC] += f2.x; acc[t][(2 * j + 1) % VEC] += f2.y; }
        } else {
          acc[t][0] += __uint_as_float(r[t].x); acc[t][1 % VEC] += __uint_as_float(r[t].y); acc[t][2 % VEC] += __uint_as_float(r[t].z); acc[t][3 % VEC] += __uint_as_float(r[t].w);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
#pragma unroll
    for (int j = 0; j < VEC; ++j) red[(l * SMAX + t) * SLAB + g * VEC + j] = acc[t][j];
  __syncthreads();
  if (threadIdx.x >= SLAB) return;
  const int c = c0 + threadIdx.x;
  if (c >= C) return;
  float pooled[SMAX];
#pragma unroll
  for (int t = 0; t < SMAX; ++t) {
    float s = 0.f;
#pragma unroll
    for (int ll = 0; ll < L; ++ll) s += red[(ll * SMAX + t) * SLAB + threadIdx.x];
    float v = s / (float)HW;
    if (t < S) {
      const long long f = p * S + t;
      if (mask) v = v * mask[f * C + c];
      feat[f * C + c] = v;
    }
    pooled[t] = v;
  }
  for (int q = 0; q < pt.n; ++q) {
    float s = 0.f;
#pragma unroll
    for (int t = 0; t < SMAX; ++t)
      if (t < S && t >= pt.lo[q] && t < pt.hi[q]) s += pooled[t];
    float m = s / (float)(pt.hi[q] - pt.lo[q]);
    m = m / (float)pt.norm[q];
    if (pt.col[q] >= 0) m = m * scaling[p * 2 + pt.col[q]];
    stpp[(p * pt.n + q) * C + c] = m;
  }
  float s = 0.f;
#pragma unroll
  for (int t = 0; t < SMAX; ++t)
    if (t < S && t >= pt.clo && t < pt.chi) s += pooled[t];
  course[p * C + c] = s / (float)(pt.chi - pt.clo);
}

// ---- STPPReorgainzed ------------------------------------------------------------------------------
struct ReorgCfg { int nstage; int nlev[3]; int lev[3][8]; int cnt[3]; };

// python slice semantics for raw[pl:pr] over T rows
__device__ __forceinline__ void py_slice(int pl, int pr, int T, int& a, int& b) {
  a = pl < 0 ? max(pl + T, 0) : min(pl, T);
  b = pr < 0 ? max(pr + T, 0) : min(pr, T);
  if (b < a) b = a;
}

// int(np.arange(left, right + 1e-5, step)[q]) (ops/ssn_ops.py:144-147): numpy stores p[0] = left and p[1] = left + step, then
// fills p[q] = left + q * (p[1] - p[0]) for q >= 2, each operation rounded on its own (no DFMA), which is not left + q * step
// when the part count is not a power of two
__device__ __forceinline__ int reorg_tick(int left, double step, int q) {
  const double l = (double)left;
  if (q == 0) return left;
  const double t1 = __dadd_rn(l, step);
  if (q == 1) return (int)t1;
  return (int)__dadd_rn(l, __dmul_rn((double)q, __dsub_rn(t1, l)));
}

// ---- STPPReorgainzed through column prefix sums ---------------------------------------------------------------------------
// Every pooled part is a mean over a contiguous row range of the [T, D] score table, and the 1000 proposals of a video overlap
// heavily: one exclusive scan down the rows (fp64, so that P[b] - P[a] is exact to fp32 rounding of the part's own sum), then
// each part costs two loads instead of (b - a).  P has T + 1 rows.
// Many videos per launch: video v's ticks are rows tick_off[v] .. tick_off[v+1]-1 of the packed scores and its table is rows
// tick_off[v] + v .. tick_off[v+1] + v of P; its proposals are rows off[v] .. off[v+1]-1.  tick_off == NULL: one video of
// T ticks (and off == NULL: its N proposals), the single-video call.
struct ReorgVideo { const double* P; int T; };

__device__ __forceinline__ ReorgVideo reorg_video(const double* P, int T, int D, const int64_t* tick_off, int v) {
  if (!tick_off) return {P, T};
  const long long t0 = tick_off[v];
  return {P + (t0 + v) * D, (int)(tick_off[v + 1] - t0)};
}

// grid (V, ceil(D / 128)): one thread per (video, column)
__global__ void colscan_f64_kernel(const float* __restrict__ scores, int T, int D, const int64_t* __restrict__ tick_off,
                                   double* __restrict__ P) {
  const int d = blockIdx.y * blockDim.x + threadIdx.x;
  if (d >= D) return;
  const int v = blockIdx.x;
  const long long t0 = tick_off ? tick_off[v] : 0;
  const int Tv = tick_off ? (int)(tick_off[v + 1] - t0) : T;
  double* Pv = P + (t0 + v) * D;
  const float* sv = scores + t0 * D;
  double s = 0.0;
  Pv[d] = 0.0;
  for (int r = 0; r < Tv; ++r) {
    s += (double)sv[(long long)r * D + d];
    Pv[(long long)(r + 1) * D + d] = s;
  }
}

// ssn_test.py:89-92 de-normalisation of the regression columns by the checkpoint's reg_stats (means, stds): column 2k is
// location, 2k + 1 size; torch's two fp32 ops, each rounded on its own (no FMA)
struct RegStats { int on; float mean[2]; float std[2]; };

__device__ void pspool_prefix_dev(const double* __restrict__ P, int T, int D, int col0, int score_len, const int* tk, float s0, float s1,
                                  const ReorgCfg& cfg, float* __restrict__ out, RegStats stats) {
  for (int j = threadIdx.x; j < score_len; j += blockDim.x) {
    float acc = 0.f;
    int offset = 0;
    for (int si = 0; si < 3; ++si) {
      const float s = si == 0 ? s0 : (si == 2 ? s1 : 1.0f);
      const int left = tk[si];
      const int right = max(tk[si] + 1, tk[si + 1]);
      if (right <= 0 || left >= T) { offset += cfg.cnt[si]; continue; }
      for (int l = 0; l < cfg.nlev[si]; ++l) {
        const int np_ = cfg.lev[si][l];
        const double step = (double)(right - left) / (double)np_;
        for (int q = 0; q < np_; ++q) {
          const int pl = reorg_tick(left, step, q);
          const int pr = reorg_tick(left, step, q + 1);
          if (pr - pl >= 1) {
            int a, b;
            py_slice(pl, pr, T, a, b);
            const int col = col0 + offset * score_len + j;
            const float sum = (float)(P[(long long)b * D + col] - P[(long long)a * D + col]);
            acc += (sum / (float)(b - a)) * s;
          }
          ++offset;
        }
      }
    }
    if (stats.on) {
      const bool size = j & 1;
      acc = __fadd_rn(__fmul_rn(acc, size ? stats.std[1] : stats.std[0]), size ? stats.mean[1] : stats.mean[0]);
    }
    out[j] = acc;
  }
}

// one CTA per proposal row i of the packed proposals; its video is the last v with off[v] <= i (empty videos own no row)
__global__ void stpp_reorg_prefix_kernel(const double* __restrict__ Pall, int T_one, int D, const int64_t* __restrict__ tick_off,
                                         const int64_t* __restrict__ off, int V, const int32_t* __restrict__ ticks,
                                         const float* __restrict__ scaling, int N, int act_len, int comp_len, int reg_len, ReorgCfg cfg, int mult,
                                         RegStats stats, float* __restrict__ out_act, float* __restrict__ out_comp, float* __restrict__ out_reg) {
  const int i = blockIdx.x;
  if (i >= N) return;
  int v = 0;
  if (off) {
    int lo = 0, hi = V - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    v = lo;
  }
  const ReorgVideo vid = reorg_video(Pall, T_one, D, tick_off, v);
  const double* P = vid.P;
  const int T = vid.T;
  const long long i4 = (long long)i * 4, i2 = (long long)i * 2;
  int tk[4] = {ticks[i4], ticks[i4 + 1], ticks[i4 + 2], ticks[i4 + 3]};
  const float s0 = scaling[i2], s1 = scaling[i2 + 1];
  {
    int a, b;
    py_slice(tk[1], max(tk[1] + 1, tk[2]), T, a, b);
    for (int j = threadIdx.x; j < act_len; j += blockDim.x)
      out_act[(long long)i * act_len + j] = (float)(P[(long long)b * D + j] - P[(long long)a * D + j]) / (float)(b - a);
  }
  pspool_prefix_dev(P, T, D, act_len, comp_len, tk, s0, s1, cfg, out_comp + (long long)i * comp_len, RegStats{0, {0.f, 0.f}, {0.f, 0.f}});
  pspool_prefix_dev(P, T, D, act_len + comp_len * mult, reg_len, tk, s0, s1, cfg, out_reg + (long long)i * reg_len, stats);
}

// ---- linear ---------------------------------------------------------------------------------------
__global__ void linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                  int n, int in_dim, int out_dim, float* __restrict__ y) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (warp >= n * out_dim) return;
  const int i = warp / out_dim, j = warp % out_dim;
  const float* xr = x + (long long)i * in_dim;
  const float* wr = w + (long long)j * in_dim;
  float s = 0.f;
  for (int d = lane; d < in_dim; d += 32) s = fmaf(xr[d], wr[d], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) y[warp] = s + (b ? b[j] : 0.f);
}
// test-time scores with the crop mean folded in (ssn_test.py:80-86: rst.view(num_crop, -1, D).mean(0) after test_fc):
//   y[t, j] = b[j] + w[j, :] . (1/crops * sum_c x[c*nt + t, :])      (the mean commutes with the linear layer)
// one CTA per tick t: phase 1 averages the crops' features into shared memory, phase 2 = one warp per output row
__global__ void linear_cropmean_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                       int crops, int nt, int in_dim, int out_dim, float* __restrict__ y) {
  extern __shared__ float xm[];
  const int t = blockIdx.x;
  const float inv = 1.0f / (float)crops;
  for (int d = threadIdx.x; d < in_dim; d += blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < crops; ++c) s += x[((long long)c * nt + t) * in_dim + d];
    xm[d] = s * inv;
  }
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, nw = blockDim.x / 32;
  for (int j = warp; j < out_dim; j += nw) {
    const float* wr = w + (long long)j * in_dim;
    float s = 0.f;
    for (int d = lane; d < in_dim; d += 32) s = fmaf(xm[d], __ldg(wr + d), s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) y[(long long)t * out_dim + j] = s + (b ? b[j] : 0.f);
  }
}
__global__ void linear_bwd_w_kernel(const float* __restrict__ x, const float* __restrict__ dy, int n, int in_dim,
                                    int out_dim, float* __restrict__ dw, float* __restrict__ db) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < out_dim && db) {
    float s = 0.f;
    for (int r = 0; r < n; ++r) s += dy[(long long)r * out_dim + i];
    db[i] = s;
  }
  if (i >= (long long)out_dim * in_dim) return;
  const int d = (int)(i % in_dim), j = (int)(i / in_dim);
  float s = 0.f;
  for (int r = 0; r < n; ++r) s = fmaf(dy[(long long)r * out_dim + j], x[(long long)r * in_dim + d], s);
  dw[i] = s;
}
__global__ void linear_bwd_x_kernel(const float* __restrict__ w, const float* __restrict__ dy, int n, int in_dim,
                                    int out_dim, float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * in_dim) return;
  const int d = (int)(i % in_dim), r = (int)(i / in_dim);
  float s = 0.f;
  for (int j = 0; j < out_dim; ++j) s = fmaf(dy[(long long)r * out_dim + j], w[(long long)j * in_dim + d], s);
  dx[i] = s;
}

// ---- OHEM hinge -------------------------------------------------------------------------------------
__device__ __forceinline__ int wrap_label(long long lab, int K) {   // labels[i]-1 with Python negative wrap
  long long c = lab - 1;
  if (c < 0) c += K;
  return (int)c;
}

__global__ void ohem_fwd_kernel(const float* __restrict__ pred, const int64_t* __restrict__ labels, int m, int K,
                                float y, int group, int keep, float* __restrict__ loss, uint8_t* __restrict__ kept,
                                float* __restrict__ slopes, float* __restrict__ scratch) {
  // scratch [m] holds the per-row hinge losses
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const float l = fmaxf(0.f, 1.f - y * pred[(long long)i * K + wrap_label(labels[i], K)]);
    scratch[i] = l;
    slopes[i] = (l != 0.f) ? -y : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    const int g0 = (i / group) * group;
    const float li = scratch[i];
    int rank = 0;
    for (int j = g0; j < g0 + group; ++j) {
      const float lj = scratch[j];
      rank += (lj > li) || (lj == li && j < i);
    }
    kept[i] = rank < keep;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float total = 0.f;
    for (int g0 = 0; g0 < m; g0 += group) {
      float s = 0.f;
      // descending order inside the group, like sorted_losses[i, :keep].sum()
      for (int r = 0; r < keep; ++r) {
        for (int j = g0; j < g0 + group; ++j) {
          if (!kept[j]) continue;
          int rank = 0;
          for (int q = g0; q < g0 + group; ++q) rank += (scratch[q] > scratch[j]) || (scratch[q] == scratch[j] && q < j);
          if (rank == r) s += scratch[j];
        }
      }
      total += s;
    }
    loss[0] = total;
  }
}
__global__ void ohem_bwd_kernel(const int64_t* __restrict__ labels, const uint8_t* __restrict__ kept,
                                const float* __restrict__ slopes, const float* __restrict__ gout, int m, int K,
                                float* __restrict__ gpred) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)m * K) return;
  const int r = (int)(i / K), c = (int)(i % K);
  gpred[i] = (kept[r] && c == wrap_label(labels[r], K)) ? slopes[r] * gout[0] : 0.f;
}

__device__ __forceinline__ float smooth_l1(float d) { const float a = fabsf(d); return a < 1.f ? 0.5f * d * d : a - 0.5f; }
__device__ __forceinline__ float smooth_l1_grad(float d) { return d >= 1.f ? 1.f : (d <= -1.f ? -1.f : d); }

__global__ void reg_fwd_kernel(const float* __restrict__ pred, const int64_t* __restrict__ labels,
                               const float* __restrict__ tg, int n, int K, float* __restrict__ loss) {
  if (threadIdx.x || blockIdx.x) return;
  float s = 0.f;
  for (int i = 0; i < n; ++i) {
    const int c = wrap_label(labels[i], K);
    for (int q = 0; q < 2; ++q) s += smooth_l1(pred[((long long)i * K + c) * 2 + q] - tg[i * 2 + q]);
  }
  loss[0] = s / (float)(2 * n) * 2.f;
}
__global__ void reg_bwd_kernel(const float* __restrict__ pred, const int64_t* __restrict__ labels,
                               const float* __restrict__ tg, const float* __restrict__ gout, int n, int K,
                               float* __restrict__ gpred) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * K * 2) return;
  const int q = (int)(i % 2), c = (int)((i / 2) % K), r = (int)(i / (2 * K));
  float g = 0.f;
  if (c == wrap_label(labels[r], K)) g = smooth_l1_grad(pred[i] - tg[r * 2 + q]) / (float)(2 * n) * 2.f * gout[0];
  gpred[i] = g;
}

// ---- fused heads + multi-task loss, forward and backward in one launch --------------------------------
constexpr int HL_THREADS = 256, HL_SLICE = 128;
constexpr int HL_ROWS = 32;        // proposals per shared-memory pass
constexpr int HL_DLCOLS = 64;      // logit columns of one slice kind held in shared memory (K+1 or 3K); wider heads use the generic path

struct HeadsArgs {
  ssnb_heads_cfg cfg;
  const float *course, *stpp, *aw, *ab, *cw, *cb, *rw, *rb;
  const int64_t *ptype, *target;
  const float* rtarget;
  float *raw_act, *raw_comp, *raw_reg, *losses, *dcourse, *dstpp, *daw, *dab, *dcw, *dcb, *drw, *drb;
  float* partial;      // [slices][n][ncols]
  float* dlogit;       // [n][ncols]
  int* rowlist;        // [3][n] selected rows: act, comp, reg
  unsigned* barrier;
};

__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    while (*((volatile unsigned*)ctr) < target) { __nanosleep(64); }
    __threadfence();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(HL_THREADS) heads_loss_kernel(HeadsArgs a) {
  const ssnb_heads_cfg& c = a.cfg;
  const int n = c.n, K = c.num_class, D = c.feat_dim, MD = c.feat_dim * c.feat_mult;
  const int na = K + 1, ncols = na + 3 * K;        // columns: [act (K+1) | comp (K) | reg (2K)]
  const int slices_c = D / HL_SLICE, slices_s = MD / HL_SLICE;
  const int s = blockIdx.x;
  const bool is_course = s < slices_c;
  const int d0 = (is_course ? s : s - slices_c) * HL_SLICE;
  const float* feat = is_course ? a.course : a.stpp;
  const int fdim = is_course ? D : MD;
  const int jc0 = is_course ? 0 : na;               // first logit column this slice contributes to
  const int jcn = is_course ? na : 3 * K;
  auto wrow = [&](int j) -> const float* {          // weight row of global logit column j
    if (j < na) return a.aw + (long long)j * D;
    if (j < na + K) return a.cw + (long long)(j - na) * MD;
    return a.rw + (long long)(j - na - K) * MD;
  };
  // phase 1: partial logits of this feature slice.  The slice of the features ([32 rows][128] per pass) is staged in
  // shared memory; a warp owns logit columns, keeps its weight slice in registers and sweeps the rows -- one global
  // load latency per column instead of one per (row, column) pair (the first version spent ~150 of its 225 us here).
  // Arithmetic per (row, column) is unchanged: lane-strided FMAs, then an xor-shuffle tree.
  __shared__ float xs[HL_ROWS][HL_SLICE];
  __shared__ float dls[HL_ROWS][HL_DLCOLS];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, nw = HL_THREADS / 32;
  for (int r0 = 0; r0 < n; r0 += HL_ROWS) {
    const int nr = min(HL_ROWS, n - r0);
    __syncthreads();
    for (int e = threadIdx.x; e < nr * HL_SLICE; e += HL_THREADS) xs[e / HL_SLICE][e % HL_SLICE] = feat[(long long)(r0 + e / HL_SLICE) * fdim + d0 + e % HL_SLICE];
    __syncthreads();
    for (int jj = warp; jj < jcn; jj += nw) {
      const int j = jc0 + jj;
      const float* wr = wrow(j) + d0;
      float wv[HL_SLICE / 32];
#pragma unroll
      for (int q = 0; q < HL_SLICE / 32; ++q) wv[q] = wr[lane + 32 * q];
#pragma unroll 4
      for (int i = 0; i < nr; ++i) {
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < HL_SLICE / 32; ++q) v = fmaf(xs[i][lane + 32 * q], wv[q], v);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) a.partial[((long long)s * n + r0 + i) * ncols + j] = v;
      }
    }
  }
  grid_barrier(a.barrier, gridDim.x * 1);
  // phase 2a: reduce partials in slice order -> raw logits (+bias); distributed over the grid
  for (long long e = (long long)blockIdx.x * HL_THREADS + threadIdx.x; e < (long long)n * ncols;
       e += (long long)gridDim.x * HL_THREADS) {
    const int i = (int)(e / ncols), j = (int)(e % ncols);
    float v = 0.f;
    if (j < na) { for (int q = 0; q < slices_c; ++q) v += a.partial[((long long)q * n + i) * ncols + j]; v += a.ab[j]; a.raw_act[(long long)i * na + j] = v; }
    else {
      for (int q = slices_c; q < slices_c + slices_s; ++q) v += a.partial[((long long)q * n + i) * ncols + j];
      if (j < na + K) { v += a.cb[j - na]; a.raw_comp[(long long)i * K + (j - na)] = v; }
      else { v += a.rb[j - na - K]; a.raw_reg[(long long)i * 2 * K + (j - na - K)] = v; }
    }
    a.dlogit[e] = 0.f;
  }
  grid_barrier(a.barrier, gridDim.x * 2);
  // phase 2b: block 0 computes the three losses and d(loss)/d(logits).  Each thread sums its own rows / groups (ascending),
  // then thread 0 adds the per-thread partials in thread order: the losses are the same bits on every call
  if (blockIdx.x == 0) {
    __shared__ int cnt[3];
    __shared__ float lpart[3][HL_THREADS];
    float lsum[3] = {0.f, 0.f, 0.f};
    if (threadIdx.x == 0) {
      int ca = 0, cc = 0, cr = 0;
      for (int i = 0; i < n; ++i) {      // ascending flat order == nonzero() (ssn_models.py:276-282)
        const long long t = a.ptype[i];
        if (t == 0 || t == 2) a.rowlist[ca++] = i;
        if (t == 0 || t == 1) a.rowlist[n + cc++] = i;
        if (t == 0) a.rowlist[2 * n + cr++] = i;
      }
      cnt[0] = ca; cnt[1] = cc; cnt[2] = cr;
    }
    __syncthreads();
    const float gscale = c.loss_scale;
    // activity: cross entropy, mean over selected rows
    for (int q = threadIdx.x; q < cnt[0]; q += HL_THREADS) {
      const int i = a.rowlist[q];
      const float* z = a.raw_act + (long long)i * na;
      float mx = z[0];
      for (int j = 1; j < na; ++j) mx = fmaxf(mx, z[j]);
      float se = 0.f;
      for (int j = 0; j < na; ++j) se += expf(z[j] - mx);
      const int t = (int)a.target[i];
      const float lse = mx + logf(se);
      lsum[0] += lse - z[t];
      for (int j = 0; j < na; ++j)
        a.dlogit[(long long)i * ncols + j] = (expf(z[j] - lse) - (j == t ? 1.f : 0.f)) / (float)cnt[0] * gscale;
    }
    // completeness: OHEM hinge per video group (ops/ssn_ops.py:223-239)
    const int G = c.comp_group, P = c.fg_per_video, Ng = G - P;
    const int ngroups = cnt[1] / G;
    const int keep_neg = c.keep_neg;
    const float denom = c.comp_denom;
    for (int g = threadIdx.x; g < ngroups; g += HL_THREADS) {
      float ls = 0.f;
      for (int q = 0; q < P; ++q) {          // positives: ratio 1.0, all kept
        const int i = a.rowlist[n + g * G + q];
        const int col = wrap_label(a.target[i], K);
        const float l = fmaxf(0.f, 1.f - a.raw_comp[(long long)i * K + col]);
        ls += l;
        if (l != 0.f) a.dlogit[(long long)i * ncols + na + col] = -1.f / denom * c.comp_w * gscale;
      }
      float nl[64];
      for (int q = 0; q < Ng && q < 64; ++q) {
        const int i = a.rowlist[n + g * G + P + q];
        nl[q] = fmaxf(0.f, 1.f + a.raw_comp[(long long)i * K + wrap_label(a.target[i], K)]);
      }
      for (int q = 0; q < Ng && q < 64; ++q) {
        int rank = 0;
        for (int r = 0; r < Ng && r < 64; ++r) rank += (nl[r] > nl[q]) || (nl[r] == nl[q] && r < q);
        if (rank < keep_neg) {
          const int i = a.rowlist[n + g * G + P + q];
          ls += nl[q];
          if (nl[q] != 0.f) a.dlogit[(long long)i * ncols + na + wrap_label(a.target[i], K)] = 1.f / denom * c.comp_w * gscale;
        }
      }
      lsum[1] += ls;
    }
    // regression: class-wise smooth L1 (mean over 2*n_fg) * 2
    for (int q = threadIdx.x; q < cnt[2]; q += HL_THREADS) {
      const int i = a.rowlist[2 * n + q];
      const int col = wrap_label(a.target[i], K);
      float ls = 0.f;
      for (int t = 0; t < 2; ++t) {
        const float d = a.raw_reg[(long long)i * 2 * K + col * 2 + t] - a.rtarget[i * 2 + t];
        ls += smooth_l1(d);
        a.dlogit[(long long)i * ncols + na + K + col * 2 + t] = smooth_l1_grad(d) / (float)(2 * cnt[2]) * 2.f * c.reg_w * gscale;
      }
      lsum[2] += ls;
    }
    for (int k = 0; k < 3; ++k) lpart[k][threadIdx.x] = lsum[k];
    __syncthreads();
    if (threadIdx.x == 0) {
      const int busy[3] = {min(cnt[0], HL_THREADS), min(ngroups, HL_THREADS), min(cnt[2], HL_THREADS)};   // the rest hold 0
      for (int k = 0; k < 3; ++k) {
        float v = 0.f;
        for (int t = 0; t < busy[k]; ++t) v += lpart[k][t];
        lsum[k] = v;
      }
      const float la = cnt[0] ? lsum[0] / (float)cnt[0] : 0.f;
      // the completeness rows must come in whole groups of comp_group per video (the reference's pred.view(-1, group, K) raises
      // otherwise, ops/ssn_ops.py:225): signalled as a NaN completeness / total loss instead of silently dropping the tail rows
      const float lc = (cnt[1] % G) ? __int_as_float(0x7fc00000) : lsum[1] / denom;
      const float lr = cnt[2] ? lsum[2] / (float)(2 * cnt[2]) * 2.f : 0.f;
      a.losses[0] = la; a.losses[1] = lc; a.losses[2] = lr; a.losses[3] = la + lc * c.comp_w + lr * c.reg_w;
    }
  }
  grid_barrier(a.barrier, gridDim.x * 3);
  // phase 3: gradients restricted to this feature slice — no cross-CTA reduction needed.  Features and d(logits) sit
  // in shared memory in passes of 32 rows x 64 logit columns; sums run in the same order as before (rows ascending /
  // columns ascending), so results are unchanged.
  {
    constexpr int WPT = HL_DLCOLS * HL_SLICE / HL_THREADS;                           // dW outputs per thread and column chunk
    constexpr int RSTEP = HL_THREADS / HL_SLICE, RPT = HL_ROWS / RSTEP;              // dfeat rows per thread and pass
    const int dcol = threadIdx.x % HL_SLICE, rsub = threadIdx.x / HL_SLICE;
    auto stage_x = [&](int r0, int nr) {
      for (int e = threadIdx.x; e < nr * HL_SLICE; e += HL_THREADS) xs[e / HL_SLICE][e % HL_SLICE] = feat[(long long)(r0 + e / HL_SLICE) * fdim + d0 + e % HL_SLICE];
    };
    auto stage_dl = [&](int r0, int nr, int jb, int nj) {
      for (int e = threadIdx.x; e < nr * nj; e += HL_THREADS) dls[e / nj][e % nj] = a.dlogit[(long long)(r0 + e / nj) * ncols + jc0 + jb + e % nj];
    };
    // (A) dW[j][d0+d] = sum_i dlogit[i][j] * feat[i][d]
    for (int jb = 0; jb < jcn; jb += HL_DLCOLS) {
      const int nj = min(HL_DLCOLS, jcn - jb);
      float accw[WPT];
#pragma unroll
      for (int o = 0; o < WPT; ++o) accw[o] = 0.f;
      for (int r0 = 0; r0 < n; r0 += HL_ROWS) {
        const int nr = min(HL_ROWS, n - r0);
        __syncthreads();
        stage_x(r0, nr); stage_dl(r0, nr, jb, nj);
        __syncthreads();
#pragma unroll
        for (int o = 0; o < WPT; ++o) {
          const int e = threadIdx.x + o * HL_THREADS, jj = e / HL_SLICE, d = e % HL_SLICE;
          if (jj < nj) {
            float v = accw[o];
            for (int i = 0; i < nr; ++i) v = fmaf(dls[i][jj], xs[i][d], v);
            accw[o] = v;
          }
        }
      }
#pragma unroll
      for (int o = 0; o < WPT; ++o) {
        const int e = threadIdx.x + o * HL_THREADS, jj = e / HL_SLICE, d = e % HL_SLICE;
        if (jj < nj) {
          const int j = jc0 + jb + jj;
          float* dst = j < na ? a.daw + (long long)j * D : (j < na + K ? a.dcw + (long long)(j - na) * MD : a.drw + (long long)(j - na - K) * MD);
          dst[d0 + d] = accw[o];
        }
      }
    }
    // (B) dfeat[i][d0+d] = sum_j dlogit[i][j] * W[j][d0+d]
    for (int r0 = 0; r0 < n; r0 += HL_ROWS) {
      const int nr = min(HL_ROWS, n - r0);
      float accf[RPT];
#pragma unroll
      for (int q = 0; q < RPT; ++q) accf[q] = 0.f;
      for (int jb = 0; jb < jcn; jb += HL_DLCOLS) {
        const int nj = min(HL_DLCOLS, jcn - jb);
        __syncthreads();
        stage_dl(r0, nr, jb, nj);
        __syncthreads();
        for (int jj = 0; jj < nj; ++jj) {
          const float wv = wrow(jc0 + jb + jj)[d0 + dcol];
#pragma unroll
          for (int q = 0; q < RPT; ++q) accf[q] = fmaf(dls[rsub + q * RSTEP][jj], wv, accf[q]);      // rows >= nr hold stale data: not stored
        }
      }
#pragma unroll
      for (int q = 0; q < RPT; ++q) {
        const int i = rsub + q * RSTEP;
        if (i < nr) (is_course ? a.dcourse : a.dstpp)[(long long)(r0 + i) * fdim + d0 + dcol] = accf[q];
      }
    }
  }
  if (blockIdx.x == 0)                                                    // bias gradients
    for (int j = threadIdx.x; j < ncols; j += HL_THREADS) {
      float v = 0.f;
      for (int i = 0; i < n; ++i) v += a.dlogit[(long long)i * ncols + j];
      if (j < na) a.dab[j] = v; else if (j < na + K) a.dcb[j - na] = v; else a.drb[j - na - K] = v;
    }
}

// one launch for the whole model: the flat buffer is cut into segments (one per parameter tensor) carrying their group's
// learning rate and weight decay (ssn_train.py:391-398 lr_mult / decay_mult); the segment of an element is found by
// binary search over the cumulative ends staged in shared memory
constexpr int SGD_MAX_SEG = 512;
__global__ void sgd_groups_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, long long n,
                                  const long long* __restrict__ seg_end, const float* __restrict__ seg_lr, const float* __restrict__ seg_wd,
                                  int nseg, float mom, float gm) {
  __shared__ long long s_end[SGD_MAX_SEG];
  __shared__ float s_lr[SGD_MAX_SEG], s_wd[SGD_MAX_SEG];
  for (int i = threadIdx.x; i < nseg; i += blockDim.x) { s_end[i] = seg_end[i]; s_lr[i] = seg_lr[i]; s_wd[i] = seg_wd[i]; }
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = nseg - 1;                 // first segment whose end is > i
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_end[mid] > i) hi = mid; else lo = mid + 1; }
  const float w = p[i];
  const float gr = g[i] * gm + s_wd[lo] * w;
  const float b = mom * buf[i] + gr;
  buf[i] = b;
  p[i] = w - s_lr[lo] * b;
}

// n_parts == 0: the course mean alone (BinaryClassifier's segment mean, binary_model.py:229-230); no part array is read
int fill_parts(PartTable& pt, int n_parts, const int* lo, const int* hi, const int* norm, const int* col, int clo, int chi, int S) {
  if (n_parts < 0 || n_parts > MAX_PARTS) { set_thread_error("stpp: 0..32 parts supported"); return SSNB_EINVAL; }
  pt.n = n_parts;
  for (int i = 0; i < n_parts; ++i) {
    if (lo[i] < 0 || hi[i] > S || hi[i] < lo[i] || norm[i] <= 0 || col[i] > 1) { set_thread_error("stpp: bad part table"); return SSNB_EINVAL; }
    pt.lo[i] = lo[i]; pt.hi[i] = hi[i]; pt.norm[i] = norm[i]; pt.col[i] = col[i];
  }
  if (clo < 0 || chi > S || chi < clo) { set_thread_error("stpp: bad course range"); return SSNB_EINVAL; }
  pt.clo = clo; pt.chi = chi;
  return 0;
}

}  // namespace
}  // namespace ssnb

namespace ssnb { int engine_tail_view(ssnb_handle h, View* v, int* F, int* fp16); }
using namespace ssnb;

extern "C" {

int ssnb_stpp_fwd(const float* ft, const float* scaling, int n, int n_seg, int D, int n_parts, const int* part_lo,
                  const int* part_hi, const int* part_norm, const int* part_scale_col, int course_lo, int course_hi,
                  float* course_ft, float* stpp_ft, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!ft || !course_ft || n < 0 || D <= 0 || (n_parts != 0 && (!scaling || !stpp_ft))) { set_thread_error("stpp_fwd: bad argument"); return SSNB_EINVAL; }
  PartTable pt;
  if (int rc = fill_parts(pt, n_parts, part_lo, part_hi, part_norm, part_scale_col, course_lo, course_hi, n_seg)) return rc;
  if (n == 0) return SSNB_OK;
  const long long tot = (long long)n * D;
  const bool vec = D % 4 == 0 && ((uintptr_t)ft | (uintptr_t)course_ft | (uintptr_t)stpp_ft) % 16 == 0;
  if (vec && n_seg <= 9) {
    stpp_fwd_v4_kernel<9><<<(unsigned)((tot / 4 + 255) / 256), 256, 0, s>>>(ft, scaling, n, n_seg, D, pt, course_ft, stpp_ft);
    SSNB_LAUNCH_CHECK("stpp_fwd_v4_kernel");
  } else if (vec && n_seg <= 16) {
    stpp_fwd_v4_kernel<16><<<(unsigned)((tot / 4 + 255) / 256), 256, 0, s>>>(ft, scaling, n, n_seg, D, pt, course_ft, stpp_ft);
    SSNB_LAUNCH_CHECK("stpp_fwd_v4_kernel");
  } else {
    stpp_fwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(ft, scaling, n, n_seg, D, pt, course_ft, stpp_ft);
    SSNB_LAUNCH_CHECK("stpp_fwd_kernel");
  }
  return SSNB_OK;
}

int ssnb_stpp_bwd(const float* d_course, const float* d_stpp, const float* scaling, int n, int n_seg, int D, int n_parts,
                  const int* part_lo, const int* part_hi, const int* part_norm, const int* part_scale_col, int course_lo,
                  int course_hi, float* d_ft, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!d_ft || n < 0 || D <= 0 || (n_parts != 0 && (!d_stpp || !scaling)) || (n_parts == 0 && !d_course)) {
    set_thread_error("stpp_bwd: bad argument"); return SSNB_EINVAL; }
  PartTable pt;
  if (int rc = fill_parts(pt, n_parts, part_lo, part_hi, part_norm, part_scale_col, course_lo, course_hi, n_seg)) return rc;
  if (n == 0) return SSNB_OK;
  const long long tot = (long long)n * n_seg * D;
  const bool vec = D % 4 == 0 && ((uintptr_t)d_course | (uintptr_t)d_stpp | (uintptr_t)d_ft) % 16 == 0;
  if (vec && n_seg <= 9 && pt.n <= 8) {
    stpp_bwd_v4_kernel<9, 8><<<(unsigned)(((long long)n * D / 4 + 255) / 256), 256, 0, s>>>(d_course, d_stpp, scaling, n, n_seg, D, pt, d_ft);
    SSNB_LAUNCH_CHECK("stpp_bwd_v4_kernel");
  } else if (vec && n_seg <= 16 && pt.n <= 16) {
    stpp_bwd_v4_kernel<16, 16><<<(unsigned)(((long long)n * D / 4 + 255) / 256), 256, 0, s>>>(d_course, d_stpp, scaling, n, n_seg, D, pt, d_ft);
    SSNB_LAUNCH_CHECK("stpp_bwd_v4_kernel");
  } else {
    stpp_bwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(d_course, d_stpp, scaling, n, n_seg, D, pt, d_ft);
    SSNB_LAUNCH_CHECK("stpp_bwd_kernel");
  }
  return SSNB_OK;
}


int ssnb_gpool_stpp_fwd(ssnb_handle h, const float* drop_mask, const float* scaling, int n_seg, int n_parts,
                        const int* part_lo, const int* part_hi, const int* part_norm, const int* part_scale_col,
                        int course_lo, int course_hi, float* feat, float* course_ft, float* stpp_ft, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  View v; int F = 0, fp16 = 0;
  if (!h || !feat || !course_ft || (n_parts != 0 && (!scaling || !stpp_ft))) { set_thread_error("gpool_stpp: null argument"); return SSNB_EINVAL; }
  if (int rc = engine_tail_view(h, &v, &F, &fp16)) return rc;
  if (n_seg <= 0 || n_seg > 32 || F % n_seg) { set_thread_error("gpool_stpp: frames must be a multiple of n_seg (<= 32)"); return SSNB_EINVAL; }
  PartTable pt;
  if (int rc = fill_parts(pt, n_parts, part_lo, part_hi, part_norm, part_scale_col, course_lo, course_hi, n_seg)) return rc;
  const int n = F / n_seg;
  const long long tot = (long long)n * v.C;
  if (n_seg <= 9 && v.C % 8 == 0 && v.pitch % 8 == 0 && v.coff % 8 == 0) {
    // second-generation kernel: CTA = (proposal, 128-channel slab)
    constexpr int SLAB = 128;
    static bool attr_set[64][2] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    const size_t smem = (size_t)(fp16 ? 256 / (SLAB / 8) : 256 / (SLAB / 4)) * 9 * SLAB * 4;
    if (dev >= 0 && dev < 64 && !attr_set[dev][fp16 ? 1 : 0]) {
      cudaError_t e = fp16 ? cudaFuncSetAttribute(gpool_stpp_v2_kernel<__half, 9, SLAB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                           : cudaFuncSetAttribute(gpool_stpp_v2_kernel<float, 9, SLAB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) { cudaGetLastError(); set_thread_error("gpool_stpp: cannot raise the dynamic shared memory limit"); return SSNB_ECUDA; }
      attr_set[dev][fp16 ? 1 : 0] = true;
    }
    dim3 grid((unsigned)n, (unsigned)((v.C + SLAB - 1) / SLAB));
    if (fp16) gpool_stpp_v2_kernel<__half, 9, SLAB><<<grid, 256, smem, s>>>((const __half*)v.base, v.H * v.W, v.C, v.pitch, v.coff, n, n_seg, drop_mask, scaling, pt, feat, course_ft, stpp_ft);
    else gpool_stpp_v2_kernel<float, 9, SLAB><<<grid, 256, smem, s>>>((const float*)v.base, v.H * v.W, v.C, v.pitch, v.coff, n, n_seg, drop_mask, scaling, pt, feat, course_ft, stpp_ft);
    SSNB_LAUNCH_CHECK("gpool_stpp_v2_kernel");
    return SSNB_OK;
  }
  if (fp16) gpool_stpp_kernel<__half><<<(unsigned)((tot + 127) / 128), 128, 0, s>>>((const __half*)v.base, v.H * v.W, v.C, v.pitch, v.coff, n, n_seg, drop_mask, scaling, pt, feat, course_ft, stpp_ft);
  else gpool_stpp_kernel<float><<<(unsigned)((tot + 127) / 128), 128, 0, s>>>((const float*)v.base, v.H * v.W, v.C, v.pitch, v.coff, n, n_seg, drop_mask, scaling, pt, feat, course_ft, stpp_ft);
  SSNB_LAUNCH_CHECK("gpool_stpp_kernel");
  return SSNB_OK;
}

size_t ssnb_stpp_reorg_workspace_bytes(int T, int D) { return (size_t)(T > 0 ? T + 1 : 0) * (size_t)(D > 0 ? D : 0) * sizeof(double); }

// the three stages' pyramid levels (level_counts[3] + the flattened levels) -> cfg and M; D must be act + M * (comp + reg)
static int reorg_cfg(const int* level_counts, const int* levels, int D, int act_len, int comp_len, int reg_len, ReorgCfg& cfg, int& mult) {
  memset(&cfg, 0, sizeof(cfg));
  cfg.nstage = 3;
  int q = 0;
  mult = 0;
  for (int st = 0; st < 3; ++st) {
    if (level_counts[st] < 1 || level_counts[st] > 8) { set_thread_error("stpp_reorg: 1..8 pyramid levels per stage"); return SSNB_EINVAL; }
    cfg.nlev[st] = level_counts[st];
    for (int l = 0; l < level_counts[st]; ++l) { cfg.lev[st][l] = levels[q++]; cfg.cnt[st] += cfg.lev[st][l]; }
    mult += cfg.cnt[st];
  }
  if (D != act_len + mult * (comp_len + reg_len)) { set_thread_error("stpp_reorg: D does not match act+M*(comp+reg)"); return SSNB_EINVAL; }
  return SSNB_OK;
}

int ssnb_stpp_reorg_prefix(const float* scores, int T, int D, const int32_t* ticks, const float* scaling, int N, int act_len,
                           int comp_len, int reg_len, const int* level_counts, const int* levels, float* out_act,
                           float* out_comp, float* out_reg, void* workspace, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!scores || !ticks || !scaling || !out_act || !out_comp || !out_reg || !workspace || T <= 0) { set_thread_error("stpp_reorg_prefix: bad argument"); return SSNB_EINVAL; }
  ReorgCfg cfg;
  int mult = 0;
  if (int rc = reorg_cfg(level_counts, levels, D, act_len, comp_len, reg_len, cfg, mult)) return rc;
  if (N == 0) return SSNB_OK;
  // one video: the V = 1 case of the batch kernels, without offsets
  double* P = reinterpret_cast<double*>(workspace);
  colscan_f64_kernel<<<dim3(1, (D + 127) / 128), 128, 0, s>>>(scores, T, D, nullptr, P);
  SSNB_LAUNCH_CHECK("colscan_f64_kernel");
  stpp_reorg_prefix_kernel<<<N, 128, 0, s>>>(P, T, D, nullptr, nullptr, 1, ticks, scaling, N, act_len, comp_len, reg_len, cfg, mult,
                                             RegStats{0, {0.f, 0.f}, {0.f, 0.f}}, out_act, out_comp, out_reg);
  SSNB_LAUNCH_CHECK("stpp_reorg_prefix_kernel");
  return SSNB_OK;
}

// host offsets [V + 1]: offsets[0] = 0, non-decreasing; -> the total, or -1
static long long reorg_offsets_total(const int64_t* offsets, int V) {
  if (!offsets || offsets[0] != 0) return -1;
  for (int v = 0; v < V; ++v)
    if (offsets[v + 1] < offsets[v]) return -1;
  return offsets[V];
}

static constexpr int kReorgMaxD = 65535 * 128;       // column blocks of the scan on grid y

size_t ssnb_stpp_reorg_batch_workspace_bytes(const int64_t* tick_offsets, int n_videos, int D) {
  if (n_videos < 0 || D <= 0 || D > kReorgMaxD) return 0;
  const long long T = reorg_offsets_total(tick_offsets, n_videos);
  if (T < 0) return 0;
  return (size_t)(T + n_videos) * (size_t)D * sizeof(double);
}

int ssnb_stpp_reorg_batch(const float* scores, int D, const int64_t* tick_offsets, const int64_t* tick_offsets_dev, const int32_t* ticks,
                          const float* scaling, const int64_t* offsets, const int64_t* offsets_dev, int n_videos, int act_len, int comp_len,
                          int reg_len, const int* level_counts, const int* levels, const double* reg_stats, float* out_act, float* out_comp,
                          float* out_reg, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  const int V = n_videos;
  if (V < 0 || D <= 0 || act_len < 0 || comp_len < 0 || reg_len < 0 || !level_counts || !levels) {
    set_thread_error("stpp_reorg_batch: bad argument (n_videos, D, score lengths or level table)"); return SSNB_EINVAL; }
  if (D > kReorgMaxD) { set_thread_error("stpp_reorg_batch: D above 65535 * 128"); return SSNB_ENOSUPPORT; }
  const long long sumT = reorg_offsets_total(tick_offsets, V), sumN = reorg_offsets_total(offsets, V);
  if (sumT < 0 || sumN < 0) {
    set_thread_error("stpp_reorg_batch: tick_offsets and offsets must be host int64 [V + 1], starting at 0, non-decreasing"); return SSNB_EINVAL; }
  for (int v = 0; v < V; ++v)
    if (tick_offsets[v + 1] - tick_offsets[v] > INT_MAX) { set_thread_error("stpp_reorg_batch: a video with more than INT_MAX ticks"); return SSNB_ENOSUPPORT; }
  if (sumN > INT_MAX) { set_thread_error("stpp_reorg_batch: more than INT_MAX proposal rows; split the batch"); return SSNB_ENOSUPPORT; }
  ReorgCfg cfg;
  int mult = 0;
  if (int rc = reorg_cfg(level_counts, levels, D, act_len, comp_len, reg_len, cfg, mult)) return rc;
  for (int st = 0; st < 3; ++st)
    for (int l = 0; l < cfg.nlev[st]; ++l)
      if (cfg.lev[st][l] < 1) { set_thread_error("stpp_reorg_batch: a pyramid level with no part"); return SSNB_EINVAL; }
  if (reg_stats && reg_len % 2) { set_thread_error("stpp_reorg_batch: reg_stats needs (location, size) column pairs: reg_len even"); return SSNB_EINVAL; }
  if (sumN > 0 && (!tick_offsets_dev || !offsets_dev || !ticks || !scaling || !out_act || !out_comp || !out_reg || !workspace || (sumT > 0 && !scores))) {
    set_thread_error("stpp_reorg_batch: NULL input, output, offsets or workspace pointer"); return SSNB_EINVAL; }
  if (sumN > 0 && workspace_bytes < (size_t)(sumT + V) * (size_t)D * sizeof(double)) {
    set_thread_error("stpp_reorg_batch: workspace too small (ssnb_stpp_reorg_batch_workspace_bytes)"); return SSNB_EINVAL; }
  if (sumN == 0) return SSNB_OK;
  RegStats st{0, {0.f, 0.f}, {0.f, 0.f}};
  if (reg_stats) st = RegStats{1, {(float)reg_stats[0], (float)reg_stats[1]}, {(float)reg_stats[2], (float)reg_stats[3]}};
  double* P = reinterpret_cast<double*>(workspace);
  colscan_f64_kernel<<<dim3((unsigned)V, (D + 127) / 128), 128, 0, s>>>(scores, 0, D, tick_offsets_dev, P);
  SSNB_LAUNCH_CHECK("colscan_f64_kernel");
  stpp_reorg_prefix_kernel<<<(unsigned)sumN, 128, 0, s>>>(P, 0, D, tick_offsets_dev, offsets_dev, V, ticks, scaling, (int)sumN, act_len,
                                                          comp_len, reg_len, cfg, mult, st, out_act, out_comp, out_reg);
  SSNB_LAUNCH_CHECK("stpp_reorg_prefix_kernel");
  return SSNB_OK;
}

int ssnb_linear_fwd(const float* x, const float* w, const float* b, int n, int in_dim, int out_dim, float* y, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!x || !w || !y) { set_thread_error("linear_fwd: null"); return SSNB_EINVAL; }
  if (n == 0) return SSNB_OK;
  const long long warps = (long long)n * out_dim;
  linear_fwd_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, s>>>(x, w, b, n, in_dim, out_dim, y);
  SSNB_LAUNCH_CHECK("linear_fwd_kernel");
  return SSNB_OK;
}

int ssnb_test_fc_cropmean(const float* feat, const float* w, const float* b, int crops, int nt, int in_dim, int out_dim,
                          float* y, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!feat || !w || !y || crops <= 0 || nt < 0 || in_dim <= 0 || in_dim > 12000 || out_dim <= 0) { set_thread_error("test_fc_cropmean: bad argument"); return SSNB_EINVAL; }
  if (nt == 0) return SSNB_OK;
  linear_cropmean_kernel<<<(unsigned)nt, 256, (size_t)in_dim * 4, s>>>(feat, w, b, crops, nt, in_dim, out_dim, y);
  SSNB_LAUNCH_CHECK("linear_cropmean_kernel");
  return SSNB_OK;
}

int ssnb_linear_bwd(const float* x, const float* w, const float* dy, int n, int in_dim, int out_dim, float* dx, float* dw,
                    float* db, void* stream) {
  if (!x || !w || !dy) { set_thread_error("linear_bwd: null"); return SSNB_EINVAL; }
  cudaStream_t s = (cudaStream_t)stream;
  if (dw) {
    const long long tot = (long long)out_dim * in_dim;
    linear_bwd_w_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(x, dy, n, in_dim, out_dim, dw, db);
    SSNB_LAUNCH_CHECK("linear_bwd_w_kernel");
  }
  if (dx && n > 0) {
    const long long tot = (long long)n * in_dim;
    linear_bwd_x_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(w, dy, n, in_dim, out_dim, dx);
    SSNB_LAUNCH_CHECK("linear_bwd_x_kernel");
  }
  return SSNB_OK;
}

int ssnb_ohem_hinge_fwd(const float* pred, const int64_t* labels, int m, int K, int is_positive, int group_size,
                        int keep_num, float* loss, uint8_t* kept, float* slopes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!pred || !labels || !loss || !kept || !slopes || group_size <= 0 || m % group_size) { set_thread_error("ohem_fwd: bad argument"); return SSNB_EINVAL; }
  // slopes doubles as the loss scratch? no: keep a separate scratch appended after slopes by the caller
  ohem_fwd_kernel<<<1, 256, 0, s>>>(pred, labels, m, K, (float)is_positive, group_size, keep_num, loss, kept, slopes, slopes + m);
  SSNB_LAUNCH_CHECK("ohem_fwd_kernel");
  return SSNB_OK;
}

int ssnb_ohem_hinge_bwd(const int64_t* labels, const uint8_t* kept, const float* slopes, const float* grad_out, int m, int K,
                        float* grad_pred, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!labels || !kept || !slopes || !grad_out || !grad_pred) { set_thread_error("ohem_bwd: null"); return SSNB_EINVAL; }
  if (m == 0) return SSNB_OK;
  const long long tot = (long long)m * K;
  ohem_bwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(labels, kept, slopes, grad_out, m, K, grad_pred);
  SSNB_LAUNCH_CHECK("ohem_bwd_kernel");
  return SSNB_OK;
}

int ssnb_classwise_reg_fwd(const float* pred, const int64_t* labels, const float* targets, int n, int K, float* loss, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!pred || !labels || !targets || !loss) { set_thread_error("reg_fwd: null"); return SSNB_EINVAL; }
  reg_fwd_kernel<<<1, 32, 0, s>>>(pred, labels, targets, n, K, loss);
  SSNB_LAUNCH_CHECK("reg_fwd_kernel");
  return SSNB_OK;
}

int ssnb_classwise_reg_bwd(const float* pred, const int64_t* labels, const float* targets, const float* grad_out, int n, int K,
                           float* grad_pred, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!pred || !labels || !targets || !grad_out || !grad_pred) { set_thread_error("reg_bwd: null"); return SSNB_EINVAL; }
  if (n == 0) return SSNB_OK;
  const long long tot = (long long)n * K * 2;
  reg_bwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(pred, labels, targets, grad_out, n, K, grad_pred);
  SSNB_LAUNCH_CHECK("reg_bwd_kernel");
  return SSNB_OK;
}

static size_t hl_align(size_t v) { return (v + 255) / 256 * 256; }
size_t ssnb_heads_loss_workspace_bytes(const ssnb_heads_cfg* c) {
  if (!c) return 0;
  const int ncols = (c->num_class + 1) + 3 * c->num_class;
  const int slices = (c->feat_dim + c->feat_dim * c->feat_mult) / HL_SLICE;
  return hl_align(256) + hl_align((size_t)slices * c->n * ncols * 4) + hl_align((size_t)c->n * ncols * 4) + hl_align((size_t)3 * c->n * 4);
}

int ssnb_heads_loss_fwd_bwd(const ssnb_heads_cfg* cfg, const float* course_ft, const float* stpp_ft, const float* act_w,
                            const float* act_b, const float* comp_w, const float* comp_b, const float* reg_w, const float* reg_b,
                            const int64_t* prop_type, const int64_t* target, const float* reg_target, float* raw_act,
                            float* raw_comp, float* raw_reg, float* losses, float* d_course_ft, float* d_stpp_ft, float* d_act_w,
                            float* d_act_b, float* d_comp_w, float* d_comp_b, float* d_reg_w, float* d_reg_b, void* workspace,
                            void* stream) {
  if (!cfg || !workspace) { set_thread_error("heads_loss: null cfg/workspace"); return SSNB_EINVAL; }
  if (cfg->feat_dim % HL_SLICE || cfg->n <= 0 || cfg->comp_group <= cfg->fg_per_video || cfg->comp_group - cfg->fg_per_video > 64 || !(cfg->comp_denom > 0.f)) {
    set_thread_error("heads_loss: feat_dim must be a multiple of 128; 1..64 negatives per group"); return SSNB_EINVAL; }
  const int slices = (cfg->feat_dim + cfg->feat_dim * cfg->feat_mult) / HL_SLICE;
  // the three phases are separated by grid barriers: the launch is COOPERATIVE, so the runtime guarantees that all CTAs are
  // co-resident (or fails the launch) whatever else occupies the device; validate the grid against the occupancy first
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, heads_loss_kernel, HL_THREADS, 0) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("heads_loss: cannot query the device occupancy"); return SSNB_ECUDA; }
  if (slices > per_sm * sms) { set_thread_error("heads_loss: more feature slices than co-resident CTAs (grid barrier)"); return SSNB_ENOSUPPORT; }
  const int ncols = (cfg->num_class + 1) + 3 * cfg->num_class;
  char* w = (char*)workspace;
  HeadsArgs a;
  a.cfg = *cfg;
  a.barrier = (unsigned*)w; w += hl_align(256);
  a.partial = (float*)w; w += hl_align((size_t)slices * cfg->n * ncols * 4);
  a.dlogit = (float*)w; w += hl_align((size_t)cfg->n * ncols * 4);
  a.rowlist = (int*)w;
  a.course = course_ft; a.stpp = stpp_ft; a.aw = act_w; a.ab = act_b; a.cw = comp_w; a.cb = comp_b; a.rw = reg_w; a.rb = reg_b;
  a.ptype = prop_type; a.target = target; a.rtarget = reg_target;
  a.raw_act = raw_act; a.raw_comp = raw_comp; a.raw_reg = raw_reg; a.losses = losses;
  a.dcourse = d_course_ft; a.dstpp = d_stpp_ft; a.daw = d_act_w; a.dab = d_act_b; a.dcw = d_comp_w; a.dcb = d_comp_b;
  a.drw = d_reg_w; a.drb = d_reg_b;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(a.barrier, 0, 256, s) != cudaSuccess) { set_thread_error("heads_loss: memset failed"); return SSNB_ECUDA; }
  void* kargs[] = {(void*)&a};
  if (cudaLaunchCooperativeKernel((const void*)heads_loss_kernel, dim3(slices), dim3(HL_THREADS), kargs, 0, s) != cudaSuccess) {
    set_thread_error(std::string("heads_loss_kernel cooperative launch: ") + cudaGetErrorString(cudaGetLastError())); return SSNB_ECUDA; }
  SSNB_LAUNCH_CHECK("heads_loss_kernel");
  return SSNB_OK;
}

int ssnb_sgd_step_groups(float* param, const float* grad, float* momentum_buf, size_t n, const int64_t* seg_end, const float* seg_lr,
                         const float* seg_wd, int n_seg, float momentum, float grad_mult, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!param || !grad || !momentum_buf || !seg_end || !seg_lr || !seg_wd || n_seg < 1 || n_seg > SGD_MAX_SEG) { set_thread_error("sgd_groups: bad argument"); return SSNB_EINVAL; }
  if (n == 0) return SSNB_OK;
  sgd_groups_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(param, grad, momentum_buf, (long long)n, (const long long*)seg_end, seg_lr, seg_wd, n_seg,
                                                              momentum, grad_mult);
  SSNB_LAUNCH_CHECK("sgd_groups_kernel");
  return SSNB_OK;
}

}  // extern "C"
