// Untrimmed video classification on the GPU: the ActivityNet toolkit's per-class average precision and video hit@k
// (anet_toolkit/Evaluation/eval_classification.py:124-249: wrapper_compute_average_precision,
// compute_average_precision_classification, compute_video_hit_at_k; interpolated_prec_rec of utils.py:14-23), every class and
// video in one call.  eval_kinetics.py is the same code.
//
//   cl_keys_kernel        every row keyed by its descending score, rows in reverse order
//   cub radix sort        64-bit, stable: the global ranking -- NaN first, then descending score (-0 == +0), equal scores the
//                         later row first: the toolkit's score.argsort()[::-1]
//   cl_split_kernel       the ranking's class and video keys (an invalid row gets K / V and sorts last)
//   cub radix sort x2     stable by class: each class's ranking; stable by video: each video's ranking
//   cl_class_pos_kernel   each class's range, and the rank position of every row in its class
//   cl_video_rank_kernel  each video's first rank, then the rank of every row within its video and the class keys of the
//                         video ranking
//   cub radix sort        stable by class of the video ranking: rows by (class, video, rank)
//   cl_gt_*               ground truth (video, label) keys sorted; the distinct pairs counted per class (npos) and per video
//   cl_mark_kernel        the first row of each (class, video) is a true positive when the pair is ground truth (the lock of
//                         eval_classification.py:190-203: a later row of the pair, or a row of a video without ground truth
//                         of the class, is a false positive); it is a hit of its video when it ranks below top_k there
//   cl_ap_kernel          one CTA per class: interp_ap_cta (interp_ap.cuh), the stage detection_ap.cu uses
//   cl_hit_kernel         one CTA: hit@k and the average hit@k over the videos with ground truth
#include <cub/cub.cuh>

#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "interp_ap.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

constexpr int kMaxClass = 1024, kThreads = 256, kHitThreads = 1024;

struct ClParams {
  int V, K, top_k, rows;
  int n_gt;
};

int key_bits(int n) { int b = 1; while ((1LL << b) <= n) ++b; return b; }   // keys 0..n

int blocks(long long n, int t) { return (int)((n + t - 1) / t); }

__global__ void cl_keys_kernel(const double* __restrict__ score, ClParams p, unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.rows) return;
  keys[p.rows - 1 - r] = score_key64(score[r]);          // reversed: a stable sort leaves ties in descending row order
  vals[p.rows - 1 - r] = r;
}

__device__ __forceinline__ bool valid_row(int v, int c, const ClParams& p) { return v >= 0 && v < p.V && c >= 0 && c < p.K; }

__global__ void cl_split_kernel(const int32_t* __restrict__ video, const int32_t* __restrict__ label, const int* __restrict__ ranked,
                                ClParams p, uint32_t* __restrict__ ckeys, int* __restrict__ cvals, uint32_t* __restrict__ vkeys,
                                int* __restrict__ vvals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows) return;
  const int r = ranked[i], v = video[r], c = label[r];
  const bool ok = valid_row(v, c, p);
  ckeys[i] = ok ? (uint32_t)c : (uint32_t)p.K;
  vkeys[i] = ok ? (uint32_t)v : (uint32_t)p.V;
  cvals[i] = r;
  vvals[i] = r;
}

// class ranges of the class ranking (cls_begin / cls_end zeroed before) and every row's position in it
__global__ void cl_class_pos_kernel(const uint32_t* __restrict__ ckeys, const int* __restrict__ rows, ClParams p, int* __restrict__ cls_begin,
                                    int* __restrict__ cls_end, int* __restrict__ pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows) return;
  const uint32_t c = ckeys[i];
  if (c >= (uint32_t)p.K) return;
  if (i == 0 || ckeys[i - 1] != c) cls_begin[c] = i;
  if (i == p.rows - 1 || ckeys[i + 1] != c) cls_end[c] = i + 1;
  pos[rows[i]] = i;
}

__global__ void cl_video_begin_kernel(const uint32_t* __restrict__ vkeys, ClParams p, int* __restrict__ vid_begin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows) return;
  const uint32_t v = vkeys[i];
  if (v < (uint32_t)p.V && (i == 0 || vkeys[i - 1] != v)) vid_begin[v] = i;
}

__global__ void cl_video_rank_kernel(const uint32_t* __restrict__ vkeys, const int* __restrict__ rows, const int32_t* __restrict__ label,
                                     const int* __restrict__ vid_begin, ClParams p, int* __restrict__ vrank, uint32_t* __restrict__ ckeys,
                                     int* __restrict__ cvals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows) return;
  const uint32_t v = vkeys[i];
  const int r = rows[i];
  cvals[i] = r;
  if (v >= (uint32_t)p.V) { ckeys[i] = (uint32_t)p.K; return; }
  vrank[r] = i - vid_begin[v];
  ckeys[i] = (uint32_t)label[r];
}

__global__ void cl_gt_keys_kernel(const int32_t* __restrict__ gt_video, const int32_t* __restrict__ gt_label, ClParams p,
                                  uint32_t* __restrict__ keys) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n_gt) return;
  const int v = gt_video[g], c = gt_label[g];
  keys[g] = valid_row(v, c, p) ? (uint32_t)c * (uint32_t)p.V + (uint32_t)v : 0xffffffffu;
}

// drop_duplicates (eval_classification.py:86): each distinct (video, label) counts once, for npos and for the video's labels
__global__ void cl_gt_count_kernel(const uint32_t* __restrict__ keys, ClParams p, int* __restrict__ npos, int* __restrict__ gt_labels) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n_gt) return;
  const uint32_t k = keys[g];
  if (k == 0xffffffffu || (g > 0 && keys[g - 1] == k)) return;
  atomicAdd(&npos[k / (uint32_t)p.V], 1);
  atomicAdd(&gt_labels[k % (uint32_t)p.V], 1);
}

__device__ __forceinline__ bool is_gt(const uint32_t* __restrict__ keys, int n, uint32_t k) {
  int lo = 0, hi = n;                                     // lower bound
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo < n && keys[lo] == k;
}

// rows in (class, video, rank) order: the first of each (class, video) is the highest-ranked prediction of the pair
__global__ void cl_mark_kernel(const uint32_t* __restrict__ ckeys, const int* __restrict__ rows, const int32_t* __restrict__ video,
                               const uint32_t* __restrict__ gt_keys, const int* __restrict__ pos, const int* __restrict__ vrank, ClParams p,
                               unsigned char* __restrict__ tp_ranked, int32_t* __restrict__ hits, uint8_t* __restrict__ tp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows) return;
  const uint32_t c = ckeys[i];
  if (c >= (uint32_t)p.K) return;
  const int r = rows[i], v = video[r];
  if (i > 0 && ckeys[i - 1] == c && video[rows[i - 1]] == v) return;
  if (!is_gt(gt_keys, p.n_gt, c * (uint32_t)p.V + (uint32_t)v)) return;
  tp_ranked[pos[r]] = 1;
  if (tp) tp[r] = 1;
  if (vrank[r] < p.top_k) atomicAdd(&hits[v], 1);
}

__global__ void cl_ap_kernel(const unsigned char* __restrict__ tp_ranked, const int* __restrict__ cls_begin, const int* __restrict__ cls_end,
                             const int* __restrict__ npos, double* __restrict__ ap) {
  const int c = blockIdx.x;
  const int b = cls_begin[c], n = cls_end[c] - b, np = npos[c];
  const double r = interp_ap_cta(tp_ranked + b, n, np);
  if (threadIdx.x == 0) ap[c] = r;
}

// eval_classification.py:231-249 over the videos with ground truth: the fraction hits / labels (one IEEE division, np.mean of
// the 0 / 1 list), ceil of it for hit@k.  The hit count is exact; the fractions are summed per thread in video order and then
// by a block reduction, a fixed order (repeatable to the bit).  No video with ground truth: NaN, as np.mean of nothing.
__global__ void __launch_bounds__(kHitThreads) cl_hit_kernel(const int32_t* __restrict__ hits, const int32_t* __restrict__ gt_labels, ClParams p,
                                                             double* __restrict__ hit_at_k, double* __restrict__ avg_hit_at_k) {
  using IRed = cub::BlockReduce<int, kHitThreads>;
  using DRed = cub::BlockReduce<double, kHitThreads>;
  __shared__ union {
    typename IRed::TempStorage ir;
    typename DRed::TempStorage dr;
  } tmp;
  int n = 0, n_hit = 0;
  double acc = 0.0;
  for (int v = threadIdx.x; v < p.V; v += kHitThreads) {
    const int g = gt_labels[v];
    if (g == 0) continue;
    const int h = hits[v];
    ++n;
    n_hit += h > 0;
    acc = __dadd_rn(acc, __ddiv_rn((double)h, (double)g));
  }
  const int videos = IRed(tmp.ir).Sum(n);
  __syncthreads();
  const int hit = IRed(tmp.ir).Sum(n_hit);
  __syncthreads();
  const double sum = DRed(tmp.dr).Sum(acc);
  if (threadIdx.x == 0) {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    hit_at_k[0] = videos ? __ddiv_rn((double)hit, (double)videos) : nan;
    avg_hit_at_k[0] = videos ? __ddiv_rn(sum, (double)videos) : nan;
  }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct ClLayout {
  size_t k64a, k64b, ra, rb, cka, ckb, cva, cvb, vka, vkb, vva, vvb, gka, gkb, pos, vrank, vid_begin, cls_begin, cls_end, npos, gt_labels,
      hits, tp_ranked, cub, total;
};

size_t cl_cub_bytes(long long rows, long long n_gt, int V, int K) {
  size_t a = 0, b = 0, c = 0, d = 0;
  cub::DoubleBuffer<unsigned long long> k64(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> k32(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  if (rows > 0) {
    cub::DeviceRadixSort::SortPairs(nullptr, a, k64, v, (int)rows, 0, 64);
    cub::DeviceRadixSort::SortPairs(nullptr, b, k32, v, (int)rows, 0, key_bits(K));
    cub::DeviceRadixSort::SortPairs(nullptr, c, k32, v, (int)rows, 0, key_bits(V));
  }
  if (n_gt > 0) cub::DeviceRadixSort::SortKeys(nullptr, d, k32, (int)n_gt, 0, 32);
  return std::max(std::max(a, b), std::max(std::max(c, d), (size_t)1));
}

ClLayout cl_layout(long long rows, long long n_gt, int V, int K) {
  ClLayout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.k64a = take(8 * rows); L.k64b = take(8 * rows); L.ra = take(4 * rows); L.rb = take(4 * rows);
  L.cka = take(4 * rows); L.ckb = take(4 * rows); L.cva = take(4 * rows); L.cvb = take(4 * rows);
  L.vka = take(4 * rows); L.vkb = take(4 * rows); L.vva = take(4 * rows); L.vvb = take(4 * rows);
  L.gka = take(4 * n_gt); L.gkb = take(4 * n_gt);
  L.pos = take(4 * rows); L.vrank = take(4 * rows); L.vid_begin = take(4LL * V);
  // cls_begin .. tp_ranked are consecutive: one memset clears them
  L.cls_begin = take(4LL * K); L.cls_end = take(4LL * K); L.npos = take(4LL * K); L.gt_labels = take(4LL * V); L.hits = take(4LL * V);
  L.tp_ranked = take(rows);
  L.cub = take(cl_cub_bytes(rows, n_gt, V, K));
  L.total = o;
  return L;
}

const char* cl_check(long long rows, long long n_gt, int V, int K) {
  if (V < 1) return "no video";
  if (K < 1 || K > kMaxClass) return "num_class must be in 1..1024";
  if (rows < 0 || rows > INT_MAX - 1) return "rows outside 0..INT_MAX-1";
  if (n_gt < 0 || n_gt > INT_MAX - 1) return "n_gt outside 0..INT_MAX-1";
  if ((long long)K * V >= INT_MAX) return "num_class * n_videos must be below INT_MAX";
  return nullptr;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_classification_ap_workspace_bytes(int64_t rows, int64_t n_gt, int n_videos, int num_class) {
  if (cl_check(rows, n_gt, n_videos, num_class)) return 0;
  return cl_layout(rows, n_gt, n_videos, num_class).total;
}

int ssnb_classification_ap(const int32_t* video, const int32_t* label, const double* score, int64_t rows, const int32_t* gt_video,
                           const int32_t* gt_label, int64_t n_gt, int n_videos, int num_class, int top_k, double* ap, double* hit_at_k,
                           double* avg_hit_at_k, int32_t* hits, int32_t* gt_labels, uint8_t* tp, void* workspace, size_t workspace_bytes,
                           void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("classification_ap: " + m); return (int)SSNB_EINVAL; };
  if (const char* bad = cl_check(rows, n_gt, n_videos, num_class)) return fail(bad);
  if (top_k < 1) return fail("top_k must be >= 1");
  if ((rows > 0 && (!video || !label || !score)) || (n_gt > 0 && (!gt_video || !gt_label)) || !ap || !hit_at_k || !avg_hit_at_k || !workspace)
    return fail("NULL input, output or workspace pointer");
  ClParams p{};
  p.V = n_videos; p.K = num_class; p.top_k = top_k; p.rows = (int)rows; p.n_gt = (int)n_gt;
  const ClLayout L = cl_layout(rows, n_gt, p.V, p.K);
  if (workspace_bytes < L.total) return fail("workspace too small (ssnb_classification_ap_workspace_bytes)");
  char* ws = (char*)workspace;
  int* cls_begin = (int*)(ws + L.cls_begin);
  int* cls_end = (int*)(ws + L.cls_end);
  int* npos = (int*)(ws + L.npos);
  unsigned char* tp_ranked = (unsigned char*)(ws + L.tp_ranked);
  if (cudaMemsetAsync(ws + L.cls_begin, 0, L.cub - L.cls_begin, s) != cudaSuccess ||
      (tp && rows > 0 && cudaMemsetAsync(tp, 0, (size_t)rows, s) != cudaSuccess)) {
    cudaGetLastError(); set_thread_error("classification_ap: memset failed"); return SSNB_ECUDA; }
  int32_t* hits_ws = (int32_t*)(ws + L.hits);
  int32_t* gtl_ws = (int32_t*)(ws + L.gt_labels);
  auto sort_failed = [](const char* what) {
    cudaGetLastError(); set_thread_error(std::string("classification_ap: ") + what + " sort failed"); return (int)SSNB_ECUDA; };
  cub::DoubleBuffer<uint32_t> gk((uint32_t*)(ws + L.gka), (uint32_t*)(ws + L.gkb));
  if (n_gt > 0) {
    cl_gt_keys_kernel<<<blocks(n_gt, kThreads), kThreads, 0, s>>>(gt_video, gt_label, p, gk.Current());
    SSNB_LAUNCH_CHECK("cl_gt_keys_kernel");
    size_t cub_bytes = cl_cub_bytes(rows, n_gt, p.V, p.K);
    if (cub::DeviceRadixSort::SortKeys(ws + L.cub, cub_bytes, gk, p.n_gt, 0, 32, s) != cudaSuccess) return sort_failed("ground-truth");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cl_gt_count_kernel<<<blocks(n_gt, kThreads), kThreads, 0, s>>>(gk.Current(), p, npos, gtl_ws);
    SSNB_LAUNCH_CHECK("cl_gt_count_kernel");
  }
  if (rows > 0) {
    cub::DoubleBuffer<unsigned long long> kb((unsigned long long*)(ws + L.k64a), (unsigned long long*)(ws + L.k64b));
    cub::DoubleBuffer<int> rb((int*)(ws + L.ra), (int*)(ws + L.rb));
    cl_keys_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(score, p, kb.Current(), rb.Current());
    SSNB_LAUNCH_CHECK("cl_keys_kernel");
    size_t cub_bytes = cl_cub_bytes(rows, n_gt, p.V, p.K);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, rb, p.rows, 0, 64, s) != cudaSuccess) return sort_failed("score");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cub::DoubleBuffer<uint32_t> ck((uint32_t*)(ws + L.cka), (uint32_t*)(ws + L.ckb)), vk((uint32_t*)(ws + L.vka), (uint32_t*)(ws + L.vkb));
    cub::DoubleBuffer<int> cv((int*)(ws + L.cva), (int*)(ws + L.cvb)), vv((int*)(ws + L.vva), (int*)(ws + L.vvb));
    cl_split_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(video, label, rb.Current(), p, ck.Current(), cv.Current(), vk.Current(),
                                                               vv.Current());
    SSNB_LAUNCH_CHECK("cl_split_kernel");
    cub_bytes = cl_cub_bytes(rows, n_gt, p.V, p.K);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, ck, cv, p.rows, 0, key_bits(p.K), s) != cudaSuccess) return sort_failed("class");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cub_bytes = cl_cub_bytes(rows, n_gt, p.V, p.K);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, vk, vv, p.rows, 0, key_bits(p.V), s) != cudaSuccess) return sort_failed("video");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    int* pos = (int*)(ws + L.pos);
    int* vrank = (int*)(ws + L.vrank);
    cl_class_pos_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(ck.Current(), cv.Current(), p, cls_begin, cls_end, pos);
    SSNB_LAUNCH_CHECK("cl_class_pos_kernel");
    cl_video_begin_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(vk.Current(), p, (int*)(ws + L.vid_begin));
    SSNB_LAUNCH_CHECK("cl_video_begin_kernel");
    // the class ranking has been read: its buffers take the (class, video, rank) sort
    cl_video_rank_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(vk.Current(), vv.Current(), label, (int*)(ws + L.vid_begin), p, vrank,
                                                                    ck.Current(), cv.Current());
    SSNB_LAUNCH_CHECK("cl_video_rank_kernel");
    cub_bytes = cl_cub_bytes(rows, n_gt, p.V, p.K);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, ck, cv, p.rows, 0, key_bits(p.K), s) != cudaSuccess)
      return sort_failed("(class, video)");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cl_mark_kernel<<<blocks(rows, kThreads), kThreads, 0, s>>>(ck.Current(), cv.Current(), video, gk.Current(), pos, vrank, p, tp_ranked,
                                                              hits_ws, tp);
    SSNB_LAUNCH_CHECK("cl_mark_kernel");
  }
  cl_ap_kernel<<<p.K, kApSumThreads, 0, s>>>(tp_ranked, cls_begin, cls_end, npos, ap);
  SSNB_LAUNCH_CHECK("cl_ap_kernel");
  cl_hit_kernel<<<1, kHitThreads, 0, s>>>(hits_ws, gtl_ws, p, hit_at_k, avg_hit_at_k);
  SSNB_LAUNCH_CHECK("cl_hit_kernel");
  if ((hits && cudaMemcpyAsync(hits, hits_ws, 4LL * p.V, cudaMemcpyDeviceToDevice, s) != cudaSuccess) ||
      (gt_labels && cudaMemcpyAsync(gt_labels, gtl_ws, 4LL * p.V, cudaMemcpyDeviceToDevice, s) != cudaSuccess)) {
    cudaGetLastError(); set_thread_error("classification_ap: trace copy failed"); return SSNB_ECUDA; }
  return SSNB_OK;
}

}  // extern "C"
