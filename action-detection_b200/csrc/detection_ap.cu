// Detection AP on the GPU: what eval_detection_results.py:199-237 hands to a process pool, one
// compute_average_precision_detection (anet_toolkit/Evaluation/eval_detection.py:160-235; segment_iou and
// interpolated_prec_rec of utils.py:14-51) per (class, tIoU threshold) job, for every class and threshold in one call.
// The greedy matching is sequential only within one (class, threshold, video): a prediction can lock only ground truth of its
// own video, so the videos of a class are matched in parallel and the ranks tie them back together.
//
// Two prediction sources share every stage after the class ranking: ssnb_detection_ap reads ssnb_detect_batch's fp32
// survivor slots (SlotSource), ssnb_detection_ap_rows the double rows of an ActivityNet results file in file order
// (RowSource).  A slot's key (class, fp32 score key) fits one 64-bit word and is ranked in one sort; a row's double score key
// and its class do not, so rows are ranked in two stable LSD passes, score then class, as classification_ap.cu ranks its rows.
//
//   ap_keys_kernel        slots: one CTA per video, every survivor slot keyed (class, descending score), slots in reverse order
//   cub radix sort        class-wide ranking: NaN first, equal scores the later (video, kept position) first (stable sort of
//                         the reversed slots)
//   ap_row_keys_kernel    rows: every row keyed by its descending double score, rows in reverse order; cub radix sort (64 bits)
//   ap_row_class_kernel   rows: the class of each ranked row (K for a row outside the videos or classes); cub radix sort by
//                         class, stable: each class's ranking, equal scores the later row first
//   ap_class_ranges_kernel  each class's range of the ranking
//   ap_bounds_kernel      (class, video) keys of the ranked predictions, rank trace
//   cub radix sort        by (class, video), stable: every (class, video) list in rank order
//   ap_cv_bounds_kernel   each (class, video) range
//   ap_npos_kernel        ground-truth instances per class (all videos, with or without detections)
//   ap_match_kernel       one warp per (class, video), lanes over the video's ground truth: for each prediction in rank order
//                         and each threshold, the unlocked ground truth of the highest tIoU that is not below it (the walk of
//                         eval_detection.py:209-223), tp / fp flags at the prediction's rank
//   ap_sum_kernel         one CTA per (class, threshold): cumulative tp, precision / recall as numpy divides them, suffix
//                         maximum of precision and the interpolated sum, walked from the last tile to the first (interp_ap.cuh)
#include <cub/cub.cuh>

#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "interp_ap.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

constexpr int kMaxClass = 1024, kMaxThr = 64, kKeyThreads = 128, kMatchWarps = 8;

struct ApParams {
  int V, K, n_thr, n_slots;                                   // n_slots: survivor slots, or rows
  long long n_gt;
  double thr[kMaxThr];
};

int class_bits(int K) { int b = 1; while ((1LL << b) <= K) ++b; return b; }   // keys 0..K

// the last video whose slots start at or before i
__device__ __forceinline__ int video_of_slot(const int64_t* __restrict__ slot0, int V, long long i) {
  int lo = 0, hi = V - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (slot0[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// where a prediction's video and segment are read: item i is a survivor slot or a row
struct SlotSource {
  const float* __restrict__ dets;
  const int64_t* __restrict__ slot0;
  __device__ __forceinline__ int video(int i, const ApParams& p) const { return video_of_slot(slot0, p.V, i); }
  __device__ __forceinline__ double t0(int i) const { return (double)dets[(long long)i * 5]; }
  __device__ __forceinline__ double t1(int i) const { return (double)dets[(long long)i * 5 + 1]; }
};

struct RowSource {
  const int32_t* __restrict__ videos;
  const double* __restrict__ seg;
  __device__ __forceinline__ int video(int i, const ApParams&) const { return videos[i]; }
  __device__ __forceinline__ double t0(int i) const { return seg[2LL * i]; }
  __device__ __forceinline__ double t1(int i) const { return seg[2LL * i + 1]; }
};

// the class of a ranked key: the high word of a slot's (class, score) key, or a row's class key
__device__ __forceinline__ unsigned long long key_class(unsigned long long k) { return k >> 32; }
__device__ __forceinline__ unsigned long long key_class(uint32_t k) { return k; }

// survivor j of class c in video v sits at slot slot0[v] + counts[v, 0..c-1] + j; it goes to input position
// n_slots - 1 - slot with key (c, score_key(score)).  The video's slots past its survivors get the last key.
__global__ void __launch_bounds__(kKeyThreads) ap_keys_kernel(const float* __restrict__ dets, const int32_t* __restrict__ counts,
                                                               const int64_t* __restrict__ slot0, ApParams p, unsigned long long* __restrict__ keys,
                                                               int* __restrict__ vals) {
  __shared__ int pre[kMaxClass + 1];
  const int v = blockIdx.x;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int c = 0; c < p.K; ++c) { pre[c] = acc; acc += counts[v * p.K + c]; }
    pre[p.K] = acc;
  }
  __syncthreads();
  const long long s0 = slot0[v], s1 = slot0[v + 1];
  for (int c = 0; c < p.K; ++c) {
    const int n = pre[c + 1] - pre[c];
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const long long slot = s0 + pre[c] + j, at = p.n_slots - 1 - slot;
      keys[at] = ((unsigned long long)c << 32) | score_key(dets[slot * 5 + 2]);
      vals[at] = (int)slot;
    }
  }
  for (long long slot = s0 + pre[p.K] + threadIdx.x; slot < s1; slot += blockDim.x) {
    keys[p.n_slots - 1 - slot] = ~0ull;
    vals[p.n_slots - 1 - slot] = -1;
  }
}

// row r goes to input position rows - 1 - r with its descending double score key: a stable sort ranks equal scores (NaN
// among them) the later row first
__global__ void ap_row_keys_kernel(const double* __restrict__ score, ApParams p, unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_slots) return;
  keys[p.n_slots - 1 - r] = score_key64(score[r]);
  vals[p.n_slots - 1 - r] = r;
}

// the class key of score-ranked row i for the stable class pass; a row outside the videos or classes gets K, past every class
__global__ void ap_row_class_kernel(const int32_t* __restrict__ video, const int32_t* __restrict__ label, const int* __restrict__ ranked,
                                    ApParams p, uint32_t* __restrict__ ckeys, int* __restrict__ cvals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_slots) return;
  const int r = ranked[i], v = video[r], c = label[r];
  ckeys[i] = (v >= 0 && v < p.V && c >= 0 && c < p.K) ? (uint32_t)c : (uint32_t)p.K;
  cvals[i] = r;
}

// class ranges of the ranking (cls_begin / cls_end zeroed before)
template <typename Key>
__global__ void ap_class_ranges_kernel(const Key* __restrict__ keys, ApParams p, int* __restrict__ cls_begin, int* __restrict__ cls_end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_slots) return;
  const unsigned long long c = key_class(keys[i]);
  if (c >= (unsigned long long)p.K) return;
  if (i == 0 || key_class(keys[i - 1]) != c) cls_begin[c] = i;
  if (i == p.n_slots - 1 || key_class(keys[i + 1]) != c) cls_end[c] = i + 1;
}

// ranked prediction i: its (class, video) key for the (class, video) sort, and its rank within the class
template <typename Key, typename Src>
__global__ void ap_bounds_kernel(const Key* __restrict__ keys, const int* __restrict__ items, Src src, ApParams p,
                                 const int* __restrict__ cls_begin, uint32_t* __restrict__ cv_keys, int* __restrict__ cv_vals,
                                 int32_t* __restrict__ rank) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_slots) return;
  const unsigned long long c = key_class(keys[i]);
  cv_vals[i] = i;
  if (c >= (unsigned long long)p.K) { cv_keys[i] = 0xffffffffu; return; }
  const int item = items[i];
  cv_keys[i] = (uint32_t)(c * p.V + src.video(item, p));
  if (rank) rank[item] = i - cls_begin[c];
}

__global__ void ap_cv_bounds_kernel(const uint32_t* __restrict__ cv_keys, ApParams p, int* __restrict__ cv_begin, int* __restrict__ cv_end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_slots) return;
  const uint32_t k = cv_keys[i];
  if (k >= (uint32_t)p.K * (uint32_t)p.V) return;
  if (i == 0 || cv_keys[i - 1] != k) cv_begin[k] = i;
  if (i == p.n_slots - 1 || cv_keys[i + 1] != k) cv_end[k] = i + 1;
}

__global__ void ap_npos_kernel(const int32_t* __restrict__ gt_cls, ApParams p, int* __restrict__ npos) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n_gt) return;
  const int c = gt_cls[g];
  if (c >= 0 && c < p.K) atomicAdd(&npos[c], 1);
}

// np.maximum / np.minimum / clip(0) in double: NaN propagates
__device__ __forceinline__ double np_max(double a, double b) { return (a != a || b != b) ? a + b : fmax(a, b); }
__device__ __forceinline__ double np_min(double a, double b) { return (a != a || b != b) ? a + b : fmin(a, b); }

// candidate (tIoU, ground-truth row) a walks before b in tiou_arr.argsort()[::-1]: NaN first, then larger tIoU, equal tIoU
// (and NaN against NaN) the larger row first; g < 0 is no candidate
__device__ __forceinline__ bool walks_first(double ta, int ga, double tb, int gb) {
  if (ga < 0 || gb < 0) return gb < 0 && ga >= 0;
  const bool na = ta != ta, nb = tb != tb;
  if (na || nb) return na && (!nb || ga > gb);
  return ta > tb || (ta == tb && ga > gb);
}

// one warp per (class, video).  For prediction (t0, t1) in rank order and threshold k, the walk over tiou_sorted_idx stops at
// the first entry that is < thr (fp) or unlocked (tp, locked); entries are in walks_first order and every entry after one that
// is < thr is < thr as well, so the prediction is a tp exactly when an unlocked ground truth with tIoU NaN or >= thr exists,
// and it locks the first such one in walk order.
template <typename Src>
__global__ void __launch_bounds__(32 * kMatchWarps) ap_match_kernel(Src src, const int* __restrict__ ranked_items,
                                                                     const int* __restrict__ cv_vals, const int* __restrict__ cv_begin,
                                                                     const int* __restrict__ cv_end, const int64_t* __restrict__ gt_offsets,
                                                                     const int32_t* __restrict__ gt_cls, const double* __restrict__ gt_seg, ApParams p,
                                                                     unsigned char* __restrict__ lock, unsigned char* __restrict__ tp_ranked,
                                                                     uint8_t* __restrict__ tp_trace) {
  const long long w = (long long)blockIdx.x * kMatchWarps + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)p.K * p.V) return;
  const int c = (int)(w / p.V), v = (int)(w % p.V);
  const int b = cv_begin[w], e = cv_end[w];
  if (b >= e) return;
  const long long g0 = gt_offsets[v], g1 = gt_offsets[v + 1];
  for (int i = b; i < e; ++i) {
    const int pos = cv_vals[i], item = ranked_items[pos];
    const double p0 = src.t0(item), p1 = src.t1(item);
    for (int k = 0; k < p.n_thr; ++k) {
      const double thr = p.thr[k];
      double best_t = 0.0;
      int best_g = -1;
      for (int g = (int)g0 + lane; g < (int)g1; g += 32) {
        if (gt_cls[g] != c || lock[(long long)k * p.n_gt + g]) continue;
        const double q0 = gt_seg[2LL * g], q1 = gt_seg[2LL * g + 1];
        const double inter = np_max(np_min(p1, q1) - np_max(p0, q0), 0.0);
        const double uni = (q1 - q0) + (p1 - p0) - inter;
        const double tiou = inter / uni;
        if (tiou < thr) continue;                             // NaN is not < thr: it walks first and matches
        if (walks_first(tiou, g, best_t, best_g)) { best_t = tiou; best_g = g; }
      }
      for (int off = 16; off > 0; off >>= 1) {
        const double ot = __shfl_xor_sync(0xffffffffu, best_t, off);
        const int og = __shfl_xor_sync(0xffffffffu, best_g, off);
        if (walks_first(ot, og, best_t, best_g)) { best_t = ot; best_g = og; }
      }
      if (lane == 0) {
        if (best_g >= 0) lock[(long long)k * p.n_gt + best_g] = 1;
        tp_ranked[(long long)k * p.n_slots + pos] = best_g >= 0;
        if (tp_trace) tp_trace[(long long)k * p.n_slots + item] = best_g >= 0;
      }
      __syncwarp();                                           // the lock is visible before the next prediction reads it
    }
  }
}

// one CTA per (class, threshold): interp_ap_cta over the class's ranked flags of threshold k
__global__ void ap_sum_kernel(const unsigned char* __restrict__ tp_ranked, const int* __restrict__ cls_begin,
                              const int* __restrict__ cls_end, const int* __restrict__ npos_arr, ApParams p, double* __restrict__ ap) {
  const int c = blockIdx.x / p.n_thr, k = blockIdx.x % p.n_thr;
  const int b = cls_begin[c], n = cls_end[c] - b, npos = npos_arr[c];
  const double r = interp_ap_cta(tp_ranked + (long long)k * p.n_slots + b, n, npos);
  if (threadIdx.x == 0) ap[c * p.n_thr + k] = r;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct ApLayout {
  size_t keys0, keys1, vals0, vals1, cvk0, cvk1, cvv0, cvv1, cls_begin, cls_end, cv_begin, cv_end, npos, tp, lock, cub, total;
};

// rows: the first pass sorts 64-bit score keys and the class pass 32-bit class keys; slots: one (class, score) pass
size_t ap_cub_bytes(int n_slots, int K, bool rows) {
  size_t a = 0, b = 0;
  cub::DoubleBuffer<unsigned long long> k64(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> k32(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k64, v, n_slots, 0, rows ? 64 : 32 + class_bits(K));
  cub::DeviceRadixSort::SortPairs(nullptr, b, k32, v, n_slots, 0, 32);
  return a > b ? a : b;
}

// The slot ranking sorts (keys, vals) and the (class, video) sort (cvk, cvv).  The row ranking's score pass sorts (keys, vals)
// and its class pass (cvk, cvv); the (class, video) sort then reuses the dead score-pass buffers, keys as 32-bit keys.
ApLayout ap_layout(int V, int K, long long n_slots, long long n_gt, int n_thr, bool rows) {
  ApLayout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.keys0 = take(8 * n_slots); L.keys1 = take(8 * n_slots); L.vals0 = take(4 * n_slots); L.vals1 = take(4 * n_slots);
  L.cvk0 = take(4 * n_slots); L.cvk1 = take(4 * n_slots); L.cvv0 = take(4 * n_slots); L.cvv1 = take(4 * n_slots);
  L.cls_begin = take(4LL * K); L.cls_end = take(4LL * K);
  L.cv_begin = take(4LL * K * V); L.cv_end = take(4LL * K * V);
  L.npos = take(4LL * K);
  L.tp = take((size_t)n_thr * n_slots);
  L.lock = take((size_t)n_thr * n_gt);
  L.cub = take(std::max<size_t>(ap_cub_bytes((int)n_slots, K, rows), 1));
  L.total = o;
  return L;
}

const char* ap_check(int V, int K, long long n_slots, long long n_gt, int n_thr) {
  if (V < 1) return "no video";
  if (K < 1 || K > kMaxClass) return "num_class must be in 1..1024";
  if (n_slots < 0 || n_slots > INT_MAX - 1) return "n_slots outside 0..INT_MAX-1";
  if (n_gt < 0 || n_gt > INT_MAX) return "n_gt outside 0..INT_MAX";
  if (n_thr < 1 || n_thr > kMaxThr) return "1..64 thresholds";
  if ((long long)K * V >= INT_MAX) return "num_class * n_videos must be below INT_MAX";
  return nullptr;
}

int blocks(long long n, int t) { return (int)((n + t - 1) / t); }

const char* ap_params(ApParams& p, int V, int K, long long n, long long n_gt, const double* thresholds, int n_thr) {
  p.V = V; p.K = K; p.n_thr = n_thr; p.n_slots = (int)n; p.n_gt = n_gt;
  for (int k = 0; k < n_thr; ++k) {
    if (std::isnan(thresholds[k])) return "NaN threshold";
    p.thr[k] = thresholds[k];
  }
  return nullptr;
}

// zero the ranges, npos and the locks, then count each class's ground truth
int ap_begin(const ApParams& p, const ApLayout& L, char* ws, const int32_t* gt_cls, const char* who, cudaStream_t s) {
  // cls_begin .. npos are consecutive regions: one memset
  if (cudaMemsetAsync(ws + L.cls_begin, 0, L.tp - L.cls_begin, s) != cudaSuccess ||
      (p.n_gt > 0 && cudaMemsetAsync(ws + L.lock, 0, (size_t)p.n_thr * p.n_gt, s) != cudaSuccess)) {
    cudaGetLastError(); set_thread_error(std::string(who) + ": memset failed"); return SSNB_ECUDA; }
  if (p.n_gt > 0) {
    ap_npos_kernel<<<blocks(p.n_gt, 256), 256, 0, s>>>(gt_cls, p, (int*)(ws + L.npos));
    SSNB_LAUNCH_CHECK("ap_npos_kernel");
  }
  return SSNB_OK;
}

// from the class-wide ranking (keys: each position's class key, items: its slot or row) to the tp flags: class ranges, rank
// trace, the stable (class, video) sort in (ckb, cvb), each (class, video) range, the matching
template <typename Key, typename Src>
int ap_match(const Key* keys, const int* items, Src src, const ApParams& p, const ApLayout& L, char* ws, cub::DoubleBuffer<uint32_t>& ckb,
             cub::DoubleBuffer<int>& cvb, const int64_t* gt_offsets, const int32_t* gt_cls, const double* gt_seg, int32_t* rank, uint8_t* tp,
             bool rows, const char* who, cudaStream_t s) {
  int* cls_begin = (int*)(ws + L.cls_begin);
  int* cv_begin = (int*)(ws + L.cv_begin);
  int* cv_end = (int*)(ws + L.cv_end);
  ap_class_ranges_kernel<<<blocks(p.n_slots, 256), 256, 0, s>>>(keys, p, cls_begin, (int*)(ws + L.cls_end));
  SSNB_LAUNCH_CHECK("ap_class_ranges_kernel");
  ap_bounds_kernel<<<blocks(p.n_slots, 256), 256, 0, s>>>(keys, items, src, p, cls_begin, ckb.Current(), cvb.Current(), rank);
  SSNB_LAUNCH_CHECK("ap_bounds_kernel");
  size_t cub_bytes = ap_cub_bytes(p.n_slots, p.K, rows);
  if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, ckb, cvb, p.n_slots, 0, 32, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error(std::string(who) + ": (class, video) sort failed"); return SSNB_ECUDA; }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  ap_cv_bounds_kernel<<<blocks(p.n_slots, 256), 256, 0, s>>>(ckb.Current(), p, cv_begin, cv_end);
  SSNB_LAUNCH_CHECK("ap_cv_bounds_kernel");
  ap_match_kernel<<<blocks((long long)p.K * p.V, kMatchWarps), 32 * kMatchWarps, 0, s>>>(
      src, items, cvb.Current(), cv_begin, cv_end, gt_offsets, gt_cls, gt_seg, p, (unsigned char*)(ws + L.lock), (unsigned char*)(ws + L.tp), tp);
  SSNB_LAUNCH_CHECK("ap_match_kernel");
  return SSNB_OK;
}

// one CTA per (class, threshold)
int ap_end(const ApParams& p, const ApLayout& L, char* ws, double* ap, cudaStream_t s) {
  ap_sum_kernel<<<p.K * p.n_thr, kApSumThreads, 0, s>>>((unsigned char*)(ws + L.tp), (int*)(ws + L.cls_begin), (int*)(ws + L.cls_end),
                                                        (int*)(ws + L.npos), p, ap);
  SSNB_LAUNCH_CHECK("ap_sum_kernel");
  return SSNB_OK;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_detection_ap_workspace_bytes(int n_videos, int num_class, int64_t n_slots, int64_t n_gt, int n_thresholds) {
  if (ap_check(n_videos, num_class, n_slots, n_gt, n_thresholds)) return 0;
  return ap_layout(n_videos, num_class, n_slots, n_gt, n_thresholds, false).total;
}

int ssnb_detection_ap(const float* dets, const int32_t* counts, const int64_t* det_slot0, int n_videos, int num_class, int64_t n_slots,
                      const int64_t* gt_offsets, const int32_t* gt_cls, const double* gt_seg, int64_t n_gt, const double* thresholds,
                      int n_thresholds, double* ap, int32_t* rank, uint8_t* tp, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("detection_ap: " + m); return (int)SSNB_EINVAL; };
  if (const char* bad = ap_check(n_videos, num_class, n_slots, n_gt, n_thresholds)) return fail(bad);
  if (!thresholds) return fail("NULL thresholds");
  if (!counts || !det_slot0 || !gt_offsets || !ap || !workspace || (n_slots > 0 && !dets) || (n_gt > 0 && (!gt_cls || !gt_seg)))
    return fail("NULL input, output or workspace pointer");
  ApParams p{};
  if (const char* bad = ap_params(p, n_videos, num_class, n_slots, n_gt, thresholds, n_thresholds)) return fail(bad);
  const ApLayout L = ap_layout(p.V, p.K, n_slots, n_gt, p.n_thr, false);
  if (workspace_bytes < L.total) return fail("workspace too small (ssnb_detection_ap_workspace_bytes)");
  char* ws = (char*)workspace;
  if (int rc = ap_begin(p, L, ws, gt_cls, "detection_ap", s)) return rc;
  if (n_slots > 0) {
    ap_keys_kernel<<<p.V, kKeyThreads, 0, s>>>(dets, counts, det_slot0, p, (unsigned long long*)(ws + L.keys0), (int*)(ws + L.vals0));
    SSNB_LAUNCH_CHECK("ap_keys_kernel");
    cub::DoubleBuffer<unsigned long long> kb((unsigned long long*)(ws + L.keys0), (unsigned long long*)(ws + L.keys1));
    cub::DoubleBuffer<int> vb((int*)(ws + L.vals0), (int*)(ws + L.vals1));
    size_t cub_bytes = ap_cub_bytes(p.n_slots, p.K, false);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, p.n_slots, 0, 32 + class_bits(p.K), s) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("detection_ap: class sort failed"); return SSNB_ECUDA; }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cub::DoubleBuffer<uint32_t> ckb((uint32_t*)(ws + L.cvk0), (uint32_t*)(ws + L.cvk1));
    cub::DoubleBuffer<int> cvb((int*)(ws + L.cvv0), (int*)(ws + L.cvv1));
    if (int rc = ap_match(kb.Current(), vb.Current(), SlotSource{dets, det_slot0}, p, L, ws, ckb, cvb, gt_offsets, gt_cls, gt_seg, rank, tp,
                          false, "detection_ap", s))
      return rc;
  }
  return ap_end(p, L, ws, ap, s);
}

size_t ssnb_detection_ap_rows_workspace_bytes(int64_t rows, int n_videos, int num_class, int64_t n_gt, int n_thresholds) {
  if (ap_check(n_videos, num_class, rows, n_gt, n_thresholds)) return 0;
  return ap_layout(n_videos, num_class, rows, n_gt, n_thresholds, true).total;
}

int ssnb_detection_ap_rows(const int32_t* video, const int32_t* label, const double* seg, const double* score, int64_t rows, int n_videos,
                           int num_class, const int64_t* gt_offsets, const int32_t* gt_cls, const double* gt_seg, int64_t n_gt,
                           const double* thresholds, int n_thresholds, double* ap, int32_t* rank, uint8_t* tp, void* workspace,
                           size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("detection_ap_rows: " + m); return (int)SSNB_EINVAL; };
  if (const char* bad = ap_check(n_videos, num_class, rows, n_gt, n_thresholds)) return fail(bad);
  if (!thresholds) return fail("NULL thresholds");
  if (!gt_offsets || !ap || !workspace || (rows > 0 && (!video || !label || !seg || !score)) || (n_gt > 0 && (!gt_cls || !gt_seg)))
    return fail("NULL input, output or workspace pointer");
  ApParams p{};
  if (const char* bad = ap_params(p, n_videos, num_class, rows, n_gt, thresholds, n_thresholds)) return fail(bad);
  const ApLayout L = ap_layout(p.V, p.K, rows, n_gt, p.n_thr, true);
  if (workspace_bytes < L.total) return fail("workspace too small (ssnb_detection_ap_rows_workspace_bytes)");
  char* ws = (char*)workspace;
  if (int rc = ap_begin(p, L, ws, gt_cls, "detection_ap_rows", s)) return rc;
  if (rows > 0) {
    auto sort_failed = [](const char* what) {
      cudaGetLastError(); set_thread_error(std::string("detection_ap_rows: ") + what + " sort failed"); return (int)SSNB_ECUDA; };
    ap_row_keys_kernel<<<blocks(rows, 256), 256, 0, s>>>(score, p, (unsigned long long*)(ws + L.keys0), (int*)(ws + L.vals0));
    SSNB_LAUNCH_CHECK("ap_row_keys_kernel");
    cub::DoubleBuffer<unsigned long long> kb((unsigned long long*)(ws + L.keys0), (unsigned long long*)(ws + L.keys1));
    cub::DoubleBuffer<int> vb((int*)(ws + L.vals0), (int*)(ws + L.vals1));
    size_t cub_bytes = ap_cub_bytes(p.n_slots, p.K, true);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, p.n_slots, 0, 64, s) != cudaSuccess) return sort_failed("score");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cub::DoubleBuffer<uint32_t> ck((uint32_t*)(ws + L.cvk0), (uint32_t*)(ws + L.cvk1));
    cub::DoubleBuffer<int> cv((int*)(ws + L.cvv0), (int*)(ws + L.cvv1));
    ap_row_class_kernel<<<blocks(rows, 256), 256, 0, s>>>(video, label, vb.Current(), p, ck.Current(), cv.Current());
    SSNB_LAUNCH_CHECK("ap_row_class_kernel");
    cub_bytes = ap_cub_bytes(p.n_slots, p.K, true);
    if (cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, ck, cv, p.n_slots, 0, class_bits(p.K), s) != cudaSuccess)
      return sort_failed("class");
    g_launches.fetch_add(1, std::memory_order_relaxed);
    // the score pass's buffers are dead: they take the (class, video) sort
    cub::DoubleBuffer<uint32_t> ckb((uint32_t*)(ws + L.keys0), (uint32_t*)(ws + L.keys1));
    cub::DoubleBuffer<int> cvb((int*)(ws + L.vals0), (int*)(ws + L.vals1));
    if (int rc = ap_match(ck.Current(), cv.Current(), RowSource{video, seg}, p, L, ws, ckb, cvb, gt_offsets, gt_cls, gt_seg, rank, tp,
                          true, "detection_ap_rows", s))
      return rc;
  }
  return ap_end(p, L, ws, ap, s);
}

}  // extern "C"
