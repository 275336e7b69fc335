// Video-level classification from snippet scores on the GPU: the aggregation and fusion functions of ops/video_funcs.py and the
// metrics of ops/metrics.py, many ragged videos per call.
//
// ssnb_video_aggregate  packed scores [sum T, crops, D] fp32 -> [V, K]
//   va_default_kernel     thread per (video, class): crop reduction (sequential over crops, as numpy reduces a middle axis),
//                         then the tick sum in tick order and one division: default_aggregation_func (video_funcs.py:8-18)
//   va_tpp_kernel         thread per (video, class): crop mean, the stage column int(t * (stage / T)) of each tick summed in
//                         float64 from 0, divided by T: tpp_aggregation_func (:60-70)
//   va_transpose_kernel   crop reduction into a per-video column-major copy [D, T_v] (a 32 x 32 tile through shared memory)
//   va_sort_kernel        warp per (video, class): the column (top_k) or the window maxima of each span (sliding window) sorted
//                         by a warp bitonic sort in shared memory, the top k summed from the k-th largest up, in the ascending
//                         order of numpy's np.sort(...)[-k:].mean(); spans averaged in span order:
//                         top_k_aggregation_func (:21-26), sliding_window_aggregation_func (:29-57)
//   va_softmax_kernel     warp per row: metrics.softmax (metrics.py:8-11), the exponentials summed by numpy's pairwise rule
// ssnb_video_fuse       default_fusion_func (:73-80): major + fp32(s * w) per stream in stream order, then the optional softmax
// ssnb_video_metrics    [V, K] scores and (video, label) pairs:
//   vm_gt_kernel          the label indicator gt[v, c]
//   vm_video_kernel       warp per video: the classes ranked (rank_key.cuh keys, ties by descending class), the top-k set,
//                         its hits and the label count (top_k_acc / top_k_hit, metrics.py:14-21); np.argmax and the
//                         confusion counts of mean_class_accuracy (:53-60)
//   cub segmented sort    each class's videos by descending score
//   vm_ap_kernel          CTA per class: sklearn's average_precision_score for one column (step AP over distinct thresholds)
//   vm_summary_kernel     one CTA: top_k_accuracy, the macro mean of the class APs, mean_class_accuracy
// Every fp32 operation the reference rounds is written with an explicit rounding intrinsic, so nvcc contracts nothing.
#include <cub/cub.cuh>

#include <climits>
#include <cmath>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

constexpr int kThreads = 128, kMaxSpans = 16, kMaxStreams = 8, kMaxSortLen = 32768, kMaxClass = 1024, kApThreads = 256;
constexpr int kSortSmem = 128 * 1024;   // dynamic shared memory of one sort block

int blocks(long long n, int t) { return (int)((n + t - 1) / t); }
int pow2_at_least(long long n) { int p = 32; while (p < n) p <<= 1; return p; }
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

__device__ __forceinline__ float nan_max(float m, float x) { return (x > m || x != x) ? x : m; }   // np.max: NaN wins

struct AggParams {
  int V, crops, D, K, mode, crop_max, n_spans, stage;
  int top_k;
  int span[kMaxSpans], step[kMaxSpans];
};

__device__ __forceinline__ float crop_reduce(const float* __restrict__ x, int crops, int D, bool use_max) {
  float a = x[0];
  for (int j = 1; j < crops; ++j) a = use_max ? nan_max(a, x[(size_t)j * D]) : __fadd_rn(a, x[(size_t)j * D]);
  return use_max ? a : __fdiv_rn(a, (float)crops);
}

__global__ void va_default_kernel(const float* __restrict__ s, const int64_t* __restrict__ toff, AggParams p, float* __restrict__ out) {
  const int v = blockIdx.x, c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= p.D) return;
  const long long t0 = toff[v], T = toff[v + 1] - t0;
  const size_t row = (size_t)p.crops * p.D;
  float acc = 0.f;
  for (long long t = 0; t < T; ++t) {
    const float r = crop_reduce(s + (size_t)(t0 + t) * row + c, p.crops, p.D, p.crop_max);
    acc = t ? __fadd_rn(acc, r) : r;
  }
  out[(size_t)v * p.D + c] = __fdiv_rn(acc, (float)T);
}

__global__ void va_tpp_kernel(const float* __restrict__ s, const int64_t* __restrict__ toff, AggParams p, double* __restrict__ out) {
  const int v = blockIdx.x, c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= p.K) return;
  const long long t0 = toff[v], T = toff[v + 1] - t0;
  const size_t row = (size_t)p.crops * p.D;
  const double step = __ddiv_rn((double)p.stage, (double)T);     // float(stage) / length
  double acc = 0.0;                                               // np.zeros(num_class)
  for (long long t = 0; t < T; ++t) {
    const int k = (int)__dmul_rn((double)t, step);
    acc = __dadd_rn(acc, (double)crop_reduce(s + (size_t)(t0 + t) * row + (size_t)k * p.K + c, p.crops, p.D, false));
  }
  out[(size_t)v * p.K + c] = __ddiv_rn(acc, (double)T);
}

// crop reduction of 32 ticks x 32 columns, written column-major per video: ws[t0_v * D + c * T_v + (t - t0_v)]
__global__ void va_transpose_kernel(const float* __restrict__ s, const int64_t* __restrict__ toff, AggParams p, long long ticks,
                                    float* __restrict__ ws) {
  __shared__ float tile[32][33];
  const long long tb = (long long)blockIdx.x * 32;
  const int cb = blockIdx.y * 32;
  const size_t row = (size_t)p.crops * p.D;
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const long long t = tb + y;
    const int c = cb + threadIdx.x;
    if (t < ticks && c < p.D) tile[y][threadIdx.x] = crop_reduce(s + (size_t)t * row + c, p.crops, p.D, p.crop_max);
  }
  __syncthreads();
  const long long t = tb + threadIdx.x;
  if (t >= ticks) return;
  int lo = 0, hi = p.V;                                   // the video of tick t: the last v with toff[v] <= t
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (toff[mid] <= t) lo = mid; else hi = mid;
  }
  const long long t0 = toff[lo], T = toff[lo + 1] - t0;
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const int c = cb + y;
    if (c < p.D) ws[(size_t)t0 * p.D + (size_t)c * T + (t - t0)] = tile[threadIdx.x][y];
  }
}

// score_key, except that -0 takes the one key no float has (0x80000000, between +0 and the negative subnormals), so a key gives
// its value back bit for bit (key_score returns +0 for both zeros) and a sum of -0 stays -0 as numpy's does
__device__ __forceinline__ uint32_t value_key(float x) { return (x == 0.f && signbit(x)) ? 0x80000000u : score_key(x); }
__device__ __forceinline__ float key_value(uint32_t k) { return k == 0x80000000u ? -0.f : key_score(k); }

// ascending warp bitonic sort of n (a power of two, >= 32) keys in shared memory
template <typename Less, typename Swap>
__device__ __forceinline__ void warp_bitonic(int n, Less less, Swap swap) {
  const int lane = threadIdx.x & 31;
  for (int k = 2; k <= n; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < (n >> 1); i += 32) {
        const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo + j;
        const bool up = (lo & k) == 0;
        if (less(hi, lo) == up) swap(lo, hi);
      }
      __syncwarp();
    }
}

// the k largest of the n keys in buf (n keys written, sorted here), summed from the k-th largest up, divided by min(k, n)
__device__ float top_k_mean(uint32_t* buf, int n, int k) {
  const int lane = threadIdx.x & 31, np2 = max(32, 1 << (32 - __clz(max(n - 1, 1))));
  for (int i = n + lane; i < np2; i += 32) buf[i] = 0xffffffffu;          // below every value, -inf included
  __syncwarp();
  warp_bitonic(np2, [&](int a, int b) { return buf[a] < buf[b]; },
               [&](int a, int b) { const uint32_t t = buf[a]; buf[a] = buf[b]; buf[b] = t; });
  const int kk = min(k, n);
  float acc = key_value(buf[kk - 1]);
  for (int i = kk - 2; i >= 0; --i) acc = __fadd_rn(acc, key_value(buf[i]));
  __syncwarp();
  return __fdiv_rn(acc, (float)kk);
}

__global__ void va_sort_kernel(const float* __restrict__ cols, const int64_t* __restrict__ toff, AggParams p, float* __restrict__ out,
                               int buf_len) {
  extern __shared__ uint32_t sbuf[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int v = blockIdx.x, c = blockIdx.y * (blockDim.x >> 5) + warp;
  if (c >= p.D) return;
  uint32_t* buf = sbuf + (size_t)warp * buf_len;
  const long long t0 = toff[v];
  const int T = (int)(toff[v + 1] - t0);
  const float* col = cols + (size_t)t0 * p.D + (size_t)c * T;
  float r = 0.f;
  if (p.mode == SSNB_VAGG_TOP_K) {
    for (int i = lane; i < T; i += 32) buf[i] = value_key(col[i]);
    __syncwarp();
    r = top_k_mean(buf, T, p.top_k);
  } else {
    for (int s = 0; s < p.n_spans; ++s) {
      const int span = p.span[s], step = p.step[s], n = (T + step - 1) / step;
      for (int i = lane; i < n; i += 32) {
        const int b = i * step, e = min(b + span, T);
        float m = col[b];
        for (int t = b + 1; t < e; ++t) m = nan_max(m, col[t]);
        buf[i] = value_key(m);
      }
      __syncwarp();
      const float x = top_k_mean(buf, n, max(15, n / 4));
      r = s ? __fadd_rn(r, x) : x;
    }
    r = __fdiv_rn(r, (float)p.n_spans);
  }
  if (lane == 0) out[(size_t)v * p.D + c] = r;
}

// numpy's pairwise sum of a contiguous float32 run (numpy/_core/src/umath/loops_utils.h.src, PW_BLOCKSIZE 128)
__device__ float pairwise_sum(const float* a, int n) {
  if (n < 8) {
    float r = 0.f;
    for (int i = 0; i < n; ++i) r = __fadd_rn(r, a[i]);
    return r;
  }
  if (n <= 128) {
    float r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[i + j]);
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, a[i]);
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return __fadd_rn(pairwise_sum(a, n2), pairwise_sum(a + n2, n - n2));
}

// softmax of each row of x [rows, K] in place: exp((x - max) * T) / sum, max NaN-propagating as np.max
__global__ void va_softmax_kernel(float* __restrict__ x, long long rows, int K, float temp) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  float* row = x + (size_t)r * K;
  float m = row[0];
  for (int i = lane; i < K; i += 32) m = nan_max(m, row[i]);
  for (int o = 16; o; o >>= 1) m = nan_max(m, __shfl_xor_sync(0xffffffffu, m, o));
  for (int i = lane; i < K; i += 32) row[i] = expf(__fmul_rn(__fsub_rn(row[i], m), temp));
  __syncwarp();
  float sum = 0.f;
  if (lane == 0) sum = pairwise_sum(row, K);
  sum = __shfl_sync(0xffffffffu, sum, 0);
  for (int i = lane; i < K; i += 32) row[i] = __fdiv_rn(row[i], sum);
}

struct FuseParams {
  const float* other[kMaxStreams];
  float w[kMaxStreams];
  int n;
};

__global__ void va_fuse_kernel(const float* __restrict__ major, FuseParams f, long long n, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a = major[i];
  for (int s = 0; s < f.n; ++s) a = __fadd_rn(a, __fmul_rn(f.other[s][i], f.w[s]));
  out[i] = a;
}

int launch_softmax(float* x, long long rows, int K, float temp, cudaStream_t s) {
  if (rows == 0) return SSNB_OK;
  va_softmax_kernel<<<blocks(rows, kThreads / 32), kThreads, 0, s>>>(x, rows, K, temp);
  SSNB_LAUNCH_CHECK("va_softmax_kernel");
  return SSNB_OK;
}

struct AggPlan {
  long long ticks;
  int max_T, buf_len, warps;
  size_t ws;
};

const char* agg_check(const int64_t* toff, int V, int crops, int D, int mode, int crop_agg, int top_k, const int32_t* spans, int n_spans,
                      double overlap, int fps, int num_class, AggParams* p, AggPlan* plan) {
  if (V < 1) return "no video";
  if (!toff) return "NULL tick_offsets";
  if (crops < 1 || D < 1) return "crops and D must be >= 1";
  if (mode < SSNB_VAGG_DEFAULT || mode > SSNB_VAGG_TPP) return "unknown mode";
  if (crop_agg != SSNB_CROP_MEAN && crop_agg != SSNB_CROP_MAX) return "crop_agg must be SSNB_CROP_MEAN or SSNB_CROP_MAX";
  if ((mode == SSNB_VAGG_SLIDING || mode == SSNB_VAGG_TPP) && crop_agg != SSNB_CROP_MEAN)
    return "sliding-window and tpp aggregation take the crop mean";
  if (toff[0] != 0) return "tick_offsets[0] must be 0";
  int max_T = 0;
  for (int v = 0; v < V; ++v) {
    const long long T = toff[v + 1] - toff[v];
    if (T < 1) return "every video needs at least one tick";
    if (T > INT_MAX) return "a video has more than INT_MAX ticks";
    max_T = std::max(max_T, (int)T);
  }
  const long long ticks = toff[V];
  if ((unsigned long long)ticks * (unsigned long long)crops * (unsigned long long)D >= (1ull << 62)) return "scores too large";
  *p = AggParams{};
  p->V = V; p->crops = crops; p->D = D; p->K = D; p->mode = mode; p->crop_max = crop_agg == SSNB_CROP_MAX; p->top_k = top_k;
  plan->ticks = ticks; plan->max_T = max_T; plan->buf_len = 0; plan->warps = 0; plan->ws = 0;
  if (mode == SSNB_VAGG_TOP_K && top_k < 1) return "top_k must be >= 1";
  if (mode == SSNB_VAGG_TPP) {
    if (num_class < 1 || D % num_class) return "tpp: D must be a positive multiple of num_class";
    p->K = num_class; p->stage = D / num_class;
  }
  if (mode == SSNB_VAGG_SLIDING) {
    if (!spans || n_spans < 1 || n_spans > kMaxSpans) return "sliding window: 1..16 spans";
    if (fps < 1) return "sliding window: fps must be >= 1";
    if (!(overlap >= 0.0 && overlap < 1.0)) return "sliding window: overlap must be in [0, 1)";
    p->n_spans = n_spans;
    for (int i = 0; i < n_spans; ++i) {
      const long long span = (long long)spans[i] * fps;
      if (spans[i] < 1 || span > INT_MAX) return "sliding window: spans must be >= 1";
      const double st = std::ceil((double)span * (1.0 - overlap));   // int(np.ceil(span * (1 - overlap)))
      if (!(st >= 1.0) || st > INT_MAX) return "sliding window: a span's step is below 1";
      p->span[i] = (int)span; p->step[i] = (int)st;
    }
  }
  if (mode == SSNB_VAGG_TOP_K || mode == SSNB_VAGG_SLIDING) {
    if (max_T > kMaxSortLen) return "top-k and sliding-window aggregation take at most 32768 ticks per video";
    plan->buf_len = pow2_at_least(max_T);
    plan->warps = std::max(1, std::min(kThreads / 32, kSortSmem / (4 * plan->buf_len)));
    plan->ws = align256((size_t)ticks * D * sizeof(float));
  }
  return nullptr;
}

struct MetricsLayout {
  size_t gt, ka, kb, va, vb, seg, conf, cub, total;
};

size_t vm_cub_bytes(int V, int K) {
  size_t b = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b, k, v, V * K, K, (const int*)nullptr, (const int*)nullptr, 0, 64);
  return std::max(b, (size_t)1);
}

MetricsLayout vm_layout(int V, int K) {
  MetricsLayout L{};
  size_t o = 0;
  const size_t n = (size_t)V * K;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.gt = take(n); L.ka = take(8 * n); L.kb = take(8 * n); L.va = take(4 * n); L.vb = take(4 * n); L.seg = take(4 * ((size_t)K + 1));
  L.conf = take(12 * (size_t)K); L.cub = take(vm_cub_bytes(V, K));
  L.total = o;
  return L;
}

const char* vm_check(int V, int K, int64_t n_labels, int top_k) {
  if (V < 1) return "no video";
  if (K < 1 || K > kMaxClass) return "num_class must be in 1..1024";
  if ((long long)V * K >= INT_MAX) return "n_videos * num_class must be below INT_MAX";
  if (n_labels < 0 || n_labels > INT_MAX) return "n_labels outside 0..INT_MAX";
  if (top_k < 1) return "top_k must be >= 1";
  return nullptr;
}

template <typename S> __device__ __forceinline__ uint64_t desc_key(S s);
template <> __device__ __forceinline__ uint64_t desc_key<float>(float s) { return score_key(s); }
template <> __device__ __forceinline__ uint64_t desc_key<double>(double s) { return score_key64(s); }

__global__ void vm_gt_kernel(const int32_t* __restrict__ lv, const int32_t* __restrict__ lab, int n, int V, int K, uint8_t* __restrict__ gt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = lv[i], c = lab[i];
  if (v >= 0 && v < V && c >= 0 && c < K) gt[(size_t)v * K + c] = 1;
}

// warp per video: rank the classes (descending key, ties by descending class), the top_k set, its hits, the label count;
// np.argmax (the first NaN, else the first maximum) and the confusion counts of the video's class label
template <typename S>
__global__ void vm_video_kernel(const S* __restrict__ score, const uint8_t* __restrict__ gt, const int32_t* __restrict__ class_label, int V,
                                int K, int top_k, int buf_len, int32_t* __restrict__ hits, int32_t* __restrict__ count,
                                int32_t* __restrict__ topk, int32_t* __restrict__ conf) {
  extern __shared__ unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int v = blockIdx.x * (blockDim.x >> 5) + warp;
  if (v >= V) return;
  uint64_t* key = (uint64_t*)smem + (size_t)warp * buf_len;
  int* cls = (int*)((uint64_t*)smem + (size_t)(blockDim.x >> 5) * buf_len) + (size_t)warp * buf_len;
  const S* row = score + (size_t)v * K;
  const uint8_t* g = gt + (size_t)v * K;
  const int np2 = max(32, 1 << (32 - __clz(max(K - 1, 1))));
  int best = INT_MAX, nan_at = INT_MAX, n_lab = 0;
  S bv = row[0];
  for (int i = lane; i < np2; i += 32) {
    if (i < K) {
      const S x = row[i];
      key[i] = desc_key<S>(x);
      cls[i] = i;
      n_lab += g[i];
      if (x != x) nan_at = min(nan_at, i);
      else if (best == INT_MAX || x > bv) { best = i; bv = x; }
    } else {
      key[i] = ~0ull;                                     // above every score key
      cls[i] = -1;
    }
  }
  for (int o = 16; o; o >>= 1) {
    n_lab += __shfl_xor_sync(0xffffffffu, n_lab, o);
    nan_at = min(nan_at, __shfl_xor_sync(0xffffffffu, nan_at, o));
    const S ob = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best, o);
    if (oi != INT_MAX && (best == INT_MAX || ob > bv || (ob == bv && oi < best))) { best = oi; bv = ob; }
  }
  __syncwarp();
  // ascending (key, descending class): NaN first, then descending score, equal scores the higher class first
  warp_bitonic(np2, [&](int a, int b) { return key[a] < key[b] || (key[a] == key[b] && cls[a] > cls[b]); },
               [&](int a, int b) {
                 const uint64_t t = key[a]; key[a] = key[b]; key[b] = t;
                 const int u = cls[a]; cls[a] = cls[b]; cls[b] = u;
               });
  const int kk = min(top_k, K);
  int h = 0;
  for (int i = lane; i < kk; i += 32) {
    const int c = cls[i];
    h += g[c];
    if (topk) topk[(size_t)v * kk + i] = c;
  }
  for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if (lane) return;
  hits[v] = h;
  count[v] = n_lab;
  if (class_label) {
    const int pred = nan_at != INT_MAX ? nan_at : best, l = class_label[v];
    if (l >= 0 && l < K) {
      atomicAdd(&conf[l], 1);
      atomicAdd(&conf[K + pred], 1);
      if (l == pred) atomicAdd(&conf[2 * K + l], 1);
    }
  }
}

// segment c of the class-major keys holds column c: its videos keyed by descending score
template <typename S>
__global__ void vm_ap_keys_kernel(const S* __restrict__ score, int V, int K, uint64_t* __restrict__ keys, int* __restrict__ vals,
                                  int* __restrict__ seg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= K) seg[i] = (int)(i * V);
  if (i >= (long long)V * K) return;
  const int c = (int)(i / V), v = (int)(i % V);
  keys[i] = desc_key<S>(score[(size_t)v * K + c]);
  vals[i] = v;
}

// sklearn's _binary_uninterpolated_average_precision for column c: the distinct thresholds in descending order, each adding
// (tps - tps at the previous threshold) / P * tps / (rank + 1); no positive: 0.  Per-thread sums in rank order, then a block
// reduction: a fixed order, repeatable to the bit.
__global__ void __launch_bounds__(kApThreads) vm_ap_kernel(const uint64_t* __restrict__ keys, const int* __restrict__ vals,
                                                           const uint8_t* __restrict__ gt, int V, int K, double* __restrict__ ap) {
  using IScan = cub::BlockScan<int, kApThreads>;
  using DRed = cub::BlockReduce<double, kApThreads>;
  __shared__ union {
    typename IScan::TempStorage scan;
    typename DRed::TempStorage red;
  } tmp;
  const int c = blockIdx.x;
  const uint64_t* k = keys + (size_t)c * V;
  const int* vv = vals + (size_t)c * V;
  int carry_tp = 0, carry_end = 0;              // positives so far; tps at the last threshold so far
  double acc = 0.0;
  for (int b = 0; b < V; b += kApThreads) {
    const int i = b + threadIdx.x;
    const int y = i < V ? gt[(size_t)vv[i] * K + c] : 0;
    const bool end = i < V && (i == V - 1 || k[i] != k[i + 1]);
    int tps, agg;
    IScan(tmp.scan).InclusiveSum(y, tps, agg);
    __syncthreads();
    tps += carry_tp;
    int prev, agg2;
    IScan(tmp.scan).ExclusiveScan(end ? tps : -1, prev, -1, cub::Max(), agg2);
    __syncthreads();
    prev = max(prev, carry_end);
    if (end && tps > prev) acc = __dadd_rn(acc, __dmul_rn((double)(tps - prev), __ddiv_rn((double)tps, (double)(i + 1))));
    carry_tp += agg;
    carry_end = max(carry_end, agg2);
  }
  const double sum = DRed(tmp.red).Sum(acc);
  if (threadIdx.x == 0) ap[c] = carry_tp ? __ddiv_rn(sum, (double)carry_tp) : 0.0;
}

__global__ void __launch_bounds__(1024) vm_summary_kernel(const int32_t* __restrict__ hits, const double* __restrict__ ap,
                                                          const int32_t* __restrict__ conf, int V, int K, int has_class,
                                                          double* __restrict__ top_k_accuracy, double* __restrict__ mean_ap,
                                                          double* __restrict__ mean_class_acc) {
  using IRed = cub::BlockReduce<int, 1024>;
  using DRed = cub::BlockReduce<double, 1024>;
  __shared__ union {
    typename IRed::TempStorage ir;
    typename DRed::TempStorage dr;
  } tmp;
  int n_hit = 0;
  for (int v = threadIdx.x; v < V; v += 1024) n_hit += hits[v] > 0;
  n_hit = IRed(tmp.ir).Sum(n_hit);
  __syncthreads();
  double a = 0.0, r = 0.0;
  int n_cls = 0;
  for (int c = threadIdx.x; c < K; c += 1024) {
    a = __dadd_rn(a, ap[c]);
    if (has_class && (conf[c] || conf[K + c])) {
      ++n_cls;
      r = __dadd_rn(r, __ddiv_rn((double)conf[2 * K + c], (double)conf[c]));    // 0 / 0 = NaN, as numpy's cls_hit / cls_cnt
    }
  }
  a = DRed(tmp.dr).Sum(a);
  __syncthreads();
  r = DRed(tmp.dr).Sum(r);
  __syncthreads();
  n_cls = IRed(tmp.ir).Sum(n_cls);
  if (threadIdx.x == 0) {
    top_k_accuracy[0] = __ddiv_rn((double)n_hit, (double)V);
    mean_ap[0] = __ddiv_rn(a, (double)K);
    mean_class_acc[0] = has_class && n_cls ? __ddiv_rn(r, (double)n_cls) : __longlong_as_double(0x7ff8000000000000LL);
  }
}

template <typename S>
int run_metrics(const S* score, int V, int K, const int32_t* lv, const int32_t* lab, int n_lab, const int32_t* class_label, int top_k,
                int32_t* hits, int32_t* count, int32_t* topk, double* top_k_accuracy, double* ap, double* mean_ap, int32_t* conf_out,
                double* mean_class_acc, char* ws, cudaStream_t s) {
  const MetricsLayout L = vm_layout(V, K);
  uint8_t* gt = (uint8_t*)(ws + L.gt);
  int32_t* conf = (int32_t*)(ws + L.conf);
  if (cudaMemsetAsync(gt, 0, (size_t)V * K, s) != cudaSuccess || cudaMemsetAsync(conf, 0, 12 * (size_t)K, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("video_metrics: memset failed"); return SSNB_ECUDA; }
  if (n_lab > 0) {
    vm_gt_kernel<<<blocks(n_lab, 256), 256, 0, s>>>(lv, lab, n_lab, V, K, gt);
    SSNB_LAUNCH_CHECK("vm_gt_kernel");
  }
  const int buf_len = pow2_at_least(K), warps = kThreads / 32;
  vm_video_kernel<S><<<blocks(V, warps), kThreads, (size_t)warps * buf_len * 12, s>>>(score, gt, class_label, V, K, top_k, buf_len, hits, count,
                                                                                     topk, conf);
  SSNB_LAUNCH_CHECK("vm_video_kernel");
  const int n = V * K;
  cub::DoubleBuffer<unsigned long long> kb((unsigned long long*)(ws + L.ka), (unsigned long long*)(ws + L.kb));
  cub::DoubleBuffer<int> vb((int*)(ws + L.va), (int*)(ws + L.vb));
  int* seg = (int*)(ws + L.seg);
  vm_ap_keys_kernel<S><<<blocks((long long)n + 1, 256), 256, 0, s>>>(score, V, K, (uint64_t*)kb.Current(), vb.Current(), seg);
  SSNB_LAUNCH_CHECK("vm_ap_keys_kernel");
  size_t cub_bytes = vm_cub_bytes(V, K);
  if (cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, n, K, seg, seg + 1, 0, sizeof(S) == 4 ? 32 : 64, s) !=
      cudaSuccess) {
    cudaGetLastError(); set_thread_error("video_metrics: class sort failed"); return SSNB_ECUDA; }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  vm_ap_kernel<<<K, kApThreads, 0, s>>>((const uint64_t*)kb.Current(), vb.Current(), gt, V, K, ap);
  SSNB_LAUNCH_CHECK("vm_ap_kernel");
  vm_summary_kernel<<<1, 1024, 0, s>>>(hits, ap, conf, V, K, class_label != nullptr, top_k_accuracy, mean_ap, mean_class_acc);
  SSNB_LAUNCH_CHECK("vm_summary_kernel");
  if (conf_out && cudaMemcpyAsync(conf_out, conf, 12 * (size_t)K, cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("video_metrics: confusion copy failed"); return SSNB_ECUDA; }
  return SSNB_OK;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_video_aggregate_workspace_bytes(const int64_t* tick_offsets, int n_videos, int crops, int D, int mode, int crop_agg, int top_k,
                                            const int32_t* spans, int n_spans, double overlap, int fps, int num_class) {
  AggParams p;
  AggPlan plan;
  if (agg_check(tick_offsets, n_videos, crops, D, mode, crop_agg, top_k, spans, n_spans, overlap, fps, num_class, &p, &plan)) return 0;
  return std::max(plan.ws, (size_t)1);
}

int ssnb_video_aggregate(const float* scores, const int64_t* tick_offsets, const int64_t* tick_offsets_dev, int n_videos, int crops, int D,
                         int mode, int crop_agg, int normalize, int top_k, const int32_t* spans, int n_spans, double overlap, int fps,
                         int num_class, void* out, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("video_aggregate: " + m); return (int)SSNB_EINVAL; };
  AggParams p;
  AggPlan plan;
  if (const char* bad = agg_check(tick_offsets, n_videos, crops, D, mode, crop_agg, top_k, spans, n_spans, overlap, fps, num_class, &p, &plan))
    return fail(bad);
  if (!scores || !tick_offsets_dev || !out) return fail("NULL scores, tick_offsets_dev or out");
  if (mode == SSNB_VAGG_TPP && normalize) return fail("tpp aggregation has no normalisation");
  if (plan.ws && (!workspace || workspace_bytes < plan.ws)) return fail("workspace too small (ssnb_video_aggregate_workspace_bytes)");
  float* o = (float*)out;
  if (mode == SSNB_VAGG_DEFAULT) {
    va_default_kernel<<<dim3(p.V, blocks(p.D, kThreads)), kThreads, 0, s>>>(scores, tick_offsets_dev, p, o);
    SSNB_LAUNCH_CHECK("va_default_kernel");
  } else if (mode == SSNB_VAGG_TPP) {
    va_tpp_kernel<<<dim3(p.V, blocks(p.K, kThreads)), kThreads, 0, s>>>(scores, tick_offsets_dev, p, (double*)out);
    SSNB_LAUNCH_CHECK("va_tpp_kernel");
  } else {
    float* cols = (float*)workspace;
    va_transpose_kernel<<<dim3((unsigned)blocks(plan.ticks, 32), blocks(p.D, 32)), dim3(32, 8), 0, s>>>(scores, tick_offsets_dev, p, plan.ticks,
                                                                                                      cols);
    SSNB_LAUNCH_CHECK("va_transpose_kernel");
    const size_t smem = (size_t)plan.warps * plan.buf_len * 4;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(va_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSortSmem) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("video_aggregate: shared memory attribute failed"); return SSNB_ECUDA; }
    va_sort_kernel<<<dim3(p.V, blocks(p.D, plan.warps)), plan.warps * 32, smem, s>>>(cols, tick_offsets_dev, p, o, plan.buf_len);
    SSNB_LAUNCH_CHECK("va_sort_kernel");
  }
  if (normalize) return launch_softmax(o, p.V, p.K, 1.f, s);
  return SSNB_OK;
}

int ssnb_video_fuse(const float* major, const float* const* others, const double* weights, int n_others, int64_t rows, int num_class,
                    int normalize, double temperature, float* out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("video_fuse: " + m); return (int)SSNB_EINVAL; };
  if (rows < 0 || num_class < 1) return fail("rows must be >= 0 and num_class >= 1");
  if (n_others < 0 || n_others > kMaxStreams) return fail("0..8 other streams");
  if (!major || !out || (n_others && (!others || !weights))) return fail("NULL major, out, others or weights");
  FuseParams f{};
  f.n = n_others;
  for (int i = 0; i < n_others; ++i) {
    if (!others[i]) return fail("NULL stream");
    f.other[i] = others[i];
    f.w[i] = (float)weights[i];                  // a Python float weight meets an fp32 array as fp32 (numpy's weak scalars)
  }
  const long long n = rows * (long long)num_class;
  if (n == 0) return SSNB_OK;
  va_fuse_kernel<<<blocks(n, 256), 256, 0, s>>>(major, f, n, out);
  SSNB_LAUNCH_CHECK("va_fuse_kernel");
  if (normalize) return launch_softmax(out, rows, num_class, (float)temperature, s);
  return SSNB_OK;
}

size_t ssnb_video_metrics_workspace_bytes(int n_videos, int num_class) {
  if (vm_check(n_videos, num_class, 0, 1)) return 0;
  return vm_layout(n_videos, num_class).total;
}

int ssnb_video_metrics(const void* scores, int scores_f64, int n_videos, int num_class, const int32_t* label_video, const int32_t* label,
                       int64_t n_labels, const int32_t* class_label, int top_k, int32_t* hits, int32_t* label_count, int32_t* top_k_idx,
                       double* top_k_accuracy, double* ap, double* mean_ap, int32_t* confusion, double* mean_class_accuracy,
                       void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("video_metrics: " + m); return (int)SSNB_EINVAL; };
  if (const char* bad = vm_check(n_videos, num_class, n_labels, top_k)) return fail(bad);
  if (!scores || (n_labels && (!label_video || !label)) || !hits || !label_count || !top_k_accuracy || !ap || !mean_ap ||
      !mean_class_accuracy || !workspace)
    return fail("NULL input, output or workspace pointer");
  if (workspace_bytes < vm_layout(n_videos, num_class).total) return fail("workspace too small (ssnb_video_metrics_workspace_bytes)");
  if (scores_f64)
    return run_metrics((const double*)scores, n_videos, num_class, label_video, label, (int)n_labels, class_label, top_k, hits, label_count,
                       top_k_idx, top_k_accuracy, ap, mean_ap, confusion, mean_class_accuracy, (char*)workspace, s);
  return run_metrics((const float*)scores, n_videos, num_class, label_video, label, (int)n_labels, class_label, top_k, hits, label_count,
                     top_k_idx, top_k_accuracy, ap, mean_ap, confusion, mean_class_accuracy, (char*)workspace, s);
}

}  // extern "C"
