// ActivityNet proposal evaluation on the GPU: average recall against the average number of proposals per video (AR-AN) of
// anet_toolkit/Evaluation/eval_proposal.py:158-273 (average_recall_vs_avg_nr_proposals; segment_iou of utils.py:25-75), every
// video and every tIoU threshold in one call.
//
//   ar_keys_kernel       one CTA per (video, chunk): the descending-score key of every proposal of a video with ground truth,
//                        written in reversed row order, and the video's segment of the sort
//   cub segmented sort   per video, stable and ascending on the key: NaN first, then descending score (-0 == +0), ties in
//                        descending row order -- the toolkit's score.argsort()[::-1]
//   ar_budget_kernel     one CTA: P_all, the ratio, nr_v = min(int(P_v * ratio), P_v), total_nr, pcn_j, proposals_per_video
//   ar_first_hit_kernel  one warp per ground-truth instance, walking its video's first nr_v ranked proposals 32 at a time:
//                        per threshold the first rank with tIoU >= t (INT_MAX: none); it stops once every threshold has one
//   ar_count_kernel      per (threshold, curve point) the instances with first_hit < n_vj, integer atomics (exact, any order)
//   ar_finalise_kernel   recall, its mean over the thresholds (a sequential sum in threshold order, then / T) in double
// The instance is recalled at (t, j) when one of the first n_vj ranked proposals has tIoU >= t, i.e. when its first hit is
// below n_vj, so one walk per instance answers all 100 curve points.  Every double operation is the toolkit's, rounded on its
// own in its order (no FMA contraction), so the curve is bitwise the toolkit's.
#include <cub/cub.cuh>

#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

constexpr int kMaxThr = 64, kPoints = 100, kKeyThreads = 256, kKeyChunksY = 64, kBudgetThreads = 1024, kHitWarps = 4,
              kCountThreads = 256, kCountChunk = 32;

struct ArParams {
  int V_all, V, n_thr;
  long long n_gt;
  double max_avg;                 // <= 0: the default, P_all / V
  double thr[kMaxThr];
};

// np.maximum / np.minimum / clip(0) in double: NaN propagates
__device__ __forceinline__ double np_max(double a, double b) { return (a != a || b != b) ? a + b : fmax(a, b); }
__device__ __forceinline__ double np_min(double a, double b) { return (a != a || b != b) ? a + b : fmin(a, b); }

// utils.py:41-50, segment_iou(proposal, ground truth): a 0 / 0 union is NaN and matches no threshold
__device__ __forceinline__ double segment_iou(double p0, double p1, double g0, double g1) {
  const double inter = np_max(__dsub_rn(np_min(p1, g1), np_max(p0, g0)), 0.0);
  const double uni = __dsub_rn(__dadd_rn(__dsub_rn(g1, g0), __dsub_rn(p1, p0)), inter);
  return __ddiv_rn(inter, uni);
}

// min(int(n * x), n) with the comparison first, so that a huge product does not overflow the conversion
__device__ __forceinline__ int scaled_count(int n, double x) {
  const double y = __dmul_rn((double)n, x);
  return y >= (double)n ? n : (int)y;
}

__global__ void __launch_bounds__(kKeyThreads) ar_keys_kernel(const double* __restrict__ scores, const int64_t* __restrict__ first,
                                                              const int32_t* __restrict__ count, const int64_t* __restrict__ gt_off,
                                                              unsigned long long* __restrict__ keys, int* __restrict__ vals,
                                                              int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int v = blockIdx.x;
  const long long f = first[v];
  const int n = gt_off[v + 1] > gt_off[v] ? count[v] : 0;      // videos without ground truth are not ranked
  if (blockIdx.y == 0 && threadIdx.x == 0) { seg_begin[v] = (int)f; seg_end[v] = (int)(f + n); }
  for (long long r = (long long)blockIdx.y * kKeyThreads + threadIdx.x; r < n; r += (long long)gridDim.y * kKeyThreads) {
    const long long at = f + n - 1 - r;                         // reversed: a stable sort leaves ties in descending row order
    keys[at] = score_key64(scores[f + r]);
    vals[at] = (int)(f + r);
  }
}

__global__ void __launch_bounds__(kBudgetThreads) ar_budget_kernel(const int32_t* __restrict__ count, const int64_t* __restrict__ gt_off,
                                                                   ArParams p, int32_t* __restrict__ nr, int64_t* __restrict__ total_nr,
                                                                   double* __restrict__ pcn, double* __restrict__ ppv) {
  using Red = cub::BlockReduce<long long, kBudgetThreads>;
  __shared__ typename Red::TempStorage tmp;
  __shared__ long long s_p_all, s_total;
  long long acc = 0;
  for (int v = threadIdx.x; v < p.V_all; v += kBudgetThreads) acc += count[v];
  const long long p_all = Red(tmp).Sum(acc);
  if (threadIdx.x == 0) s_p_all = p_all;
  __syncthreads();
  // :188-191, left to right in double
  const double V = (double)p.V;
  const double max_avg = p.max_avg > 0.0 ? p.max_avg : __ddiv_rn((double)s_p_all, V);
  const double ratio = __ddiv_rn(__dmul_rn(max_avg, V), (double)s_p_all);
  acc = 0;
  for (int v = threadIdx.x; v < p.V_all; v += kBudgetThreads) {
    const int n = count[v];
    const int k = (gt_off[v + 1] > gt_off[v] && n > 0) ? scaled_count(n, ratio) : 0;   // :229-230
    nr[v] = k;
    acc += k;
  }
  __syncthreads();
  const long long tot = Red(tmp).Sum(acc);
  if (threadIdx.x == 0) { s_total = tot; total_nr[0] = tot; }
  __syncthreads();
  if (threadIdx.x < kPoints) {
    const long long t = s_total;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    const int j = threadIdx.x + 1;
    // :243 np.arange(1, 101) / 100.0 * (max_avg * float(V) / total_nr); :271 pcn * (float(total_nr) / V)
    const double c = __dmul_rn(__ddiv_rn((double)j, 100.0), __ddiv_rn(__dmul_rn(max_avg, V), (double)t));
    pcn[threadIdx.x] = t ? c : nan;
    ppv[threadIdx.x] = t ? __dmul_rn(c, __ddiv_rn((double)t, V)) : nan;
  }
}

// lane l keeps the first hit of threshold l (h0) and l + 32 (h1)
__global__ void __launch_bounds__(32 * kHitWarps) ar_first_hit_kernel(const double2* __restrict__ boxes, const int* __restrict__ ranked,
                                                                      const int64_t* __restrict__ first, const int32_t* __restrict__ count,
                                                                      const int32_t* __restrict__ nr, const double2* __restrict__ gt,
                                                                      const int64_t* __restrict__ gt_off, ArParams p,
                                                                      int32_t* __restrict__ first_hit, int32_t* __restrict__ gt_cols) {
  const int v = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long g0 = gt_off[v], g1 = gt_off[v + 1];
  if (g0 == g1) return;
  const int n_p = count[v];
  const long long f = first[v];
  const int cols = n_p > 0 ? nr[v] : 1;                          // no proposal: one phantom column of tIoU 0.0 (:208-218)
  for (long long g = g0 + warp; g < g1; g += kHitWarps) {
    const double2 q = gt[g];
    int h0 = INT_MAX, h1 = INT_MAX;
    if (n_p == 0) {
      if (lane < p.n_thr && 0.0 >= p.thr[lane]) h0 = 0;
      if (lane + 32 < p.n_thr && 0.0 >= p.thr[lane + 32]) h1 = 0;
    } else {
      for (int c0 = 0; c0 < cols; c0 += 32) {
        const int r = c0 + lane;
        double tiou = 0.0;
        const bool on = r < cols;
        if (on) {
          const double2 b = boxes[ranked[f + r]];
          tiou = segment_iou(b.x, b.y, q.x, q.y);
        }
        for (int t = 0; t < p.n_thr; ++t) {
          const unsigned m = __ballot_sync(0xffffffffu, on && tiou >= p.thr[t]);
          if (m && lane == (t & 31)) {
            const int hit = c0 + __ffs(m) - 1;
            if (t < 32) h0 = min(h0, hit); else h1 = min(h1, hit);
          }
        }
        const bool open = (lane < p.n_thr && h0 == INT_MAX) || (lane + 32 < p.n_thr && h1 == INT_MAX);
        if (!__any_sync(0xffffffffu, open)) break;
      }
    }
    if (lane < p.n_thr) first_hit[g * p.n_thr + lane] = h0;
    if (lane + 32 < p.n_thr) first_hit[g * p.n_thr + lane + 32] = h1;
    if (lane == 0) gt_cols[g] = cols;
  }
}

// :258-265 for kCountChunk instances per CTA: instance g is matched at (t, j) when first_hit[g, t] < min(int(P'_v * pcn_j), P'_v)
__global__ void __launch_bounds__(kCountThreads) ar_count_kernel(const int32_t* __restrict__ first_hit, const int32_t* __restrict__ gt_cols,
                                                                 const double* __restrict__ pcn, ArParams p,
                                                                 unsigned long long* __restrict__ matches) {
  __shared__ int s_hit[kCountChunk * kMaxThr];
  __shared__ int s_cols[kCountChunk];
  const long long g0 = (long long)blockIdx.x * kCountChunk;
  const int m = (int)(p.n_gt - g0 < kCountChunk ? p.n_gt - g0 : kCountChunk);
  for (int i = threadIdx.x; i < m * p.n_thr; i += kCountThreads) s_hit[i] = first_hit[g0 * p.n_thr + i];
  if (threadIdx.x < m) s_cols[threadIdx.x] = gt_cols[g0 + threadIdx.x];
  __syncthreads();
  for (int tj = threadIdx.x; tj < p.n_thr * kPoints; tj += kCountThreads) {
    const int t = tj / kPoints;
    const double x = pcn[tj % kPoints];
    unsigned long long c = 0;
    for (int i = 0; i < m; ++i) c += s_hit[i * p.n_thr + t] < scaled_count(s_cols[i], x);
    if (c) atomicAdd(&matches[tj], c);
  }
}

__global__ void ar_finalise_kernel(const unsigned long long* __restrict__ matches, const int64_t* __restrict__ total_nr, ArParams p,
                                   double* __restrict__ recall, double* __restrict__ avg_recall) {
  const int j = threadIdx.x;
  if (j >= kPoints) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const bool ok = total_nr[0] != 0;
  double acc = 0.0;
  for (int t = 0; t < p.n_thr; ++t) {
    const double r = __ddiv_rn((double)matches[t * kPoints + j], (double)p.n_gt);     // :265 matches.sum(0) / positives.sum()
    recall[t * kPoints + j] = ok ? r : nan;
    acc = __dadd_rn(acc, r);
  }
  avg_recall[j] = ok ? __ddiv_rn(acc, (double)p.n_thr) : nan;                          // :268 recall.mean(axis=0)
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct ArLayout { size_t keys0, keys1, vals0, vals1, seg_begin, seg_end, nr, first_hit, gt_cols, pcn, matches, cub, total; };

size_t ar_cub_bytes(long long rows, int V_all) {
  size_t b = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b, k, v, (int)rows, V_all, (const int*)nullptr, (const int*)nullptr, 0, 64);
  return b;
}

ArLayout ar_layout(int V_all, long long rows, long long n_gt, int n_thr) {
  ArLayout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.keys0 = take(8 * rows); L.keys1 = take(8 * rows); L.vals0 = take(4 * rows); L.vals1 = take(4 * rows);
  L.seg_begin = take(4LL * V_all); L.seg_end = take(4LL * V_all); L.nr = take(4LL * V_all);
  L.first_hit = take(4 * n_gt * n_thr); L.gt_cols = take(4 * n_gt);
  L.pcn = take(8 * kPoints); L.matches = take(8LL * kPoints * n_thr);
  L.cub = take(std::max<size_t>(rows > 0 ? ar_cub_bytes(rows, V_all) : 0, 1));
  L.total = o;
  return L;
}

bool ascending(const int64_t* off, int V) {
  if (off[0] != 0) return false;
  for (int v = 0; v < V; ++v)
    if (off[v + 1] < off[v]) return false;
  return true;
}

// the host-side checks shared by the call and the workspace query; V = videos with ground truth
const char* ar_check(int V_all, long long rows, const int64_t* gt_off, int n_thr, int* V) {
  if (V_all < 1) return "no video";
  if (rows < 0 || rows > INT_MAX) return "rows outside 0..INT_MAX";
  if (n_thr < 1 || n_thr > kMaxThr) return "1..64 thresholds";
  if (!gt_off || !ascending(gt_off, V_all)) return "gt_offsets must start at 0 and ascend";
  if (gt_off[V_all] > INT_MAX / kMaxThr) return "too many ground-truth instances";
  int n = 0;
  for (int v = 0; v < V_all; ++v) n += gt_off[v + 1] > gt_off[v];
  if (n == 0) return "no ground truth";
  *V = n;
  return nullptr;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_proposal_ar_workspace_bytes(int n_videos, int64_t rows, const int64_t* gt_offsets, int n_thresholds) {
  int V = 0;
  if (ar_check(n_videos, rows, gt_offsets, n_thresholds, &V)) return 0;
  return ar_layout(n_videos, rows, gt_offsets[n_videos], n_thresholds).total;
}

int ssnb_proposal_ar(const double* boxes, const double* scores, int64_t rows, const int64_t* first, const int32_t* count, int n_videos,
                     const double* gt_seg, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, const double* thresholds,
                     int n_thresholds, double max_avg, double* recall, double* avg_recall, double* proposals_per_video,
                     int64_t* total_nr, int32_t* nr, int32_t* first_hit, void* workspace, size_t workspace_bytes, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("proposal_ar: " + m); return (int)SSNB_EINVAL; };
  ArParams p{};
  if (const char* bad = ar_check(n_videos, rows, gt_offsets, n_thresholds, &p.V)) return fail(bad);
  if (!thresholds) return fail("NULL thresholds");
  for (int t = 0; t < n_thresholds; ++t) {
    if (std::isnan(thresholds[t])) return fail("NaN threshold");
    p.thr[t] = thresholds[t];
  }
  if (!std::isfinite(max_avg)) return fail("max_avg must be finite");
  if ((rows > 0 && (!boxes || !scores)) || !first || !count || !gt_seg || !gt_offsets_dev || !recall || !avg_recall ||
      !proposals_per_video || !total_nr || !workspace)
    return fail("NULL input, output or workspace pointer");
  p.V_all = n_videos; p.n_thr = n_thresholds; p.n_gt = gt_offsets[n_videos]; p.max_avg = max_avg;
  const ArLayout L = ar_layout(n_videos, rows, p.n_gt, n_thresholds);
  if (workspace_bytes < L.total) return fail("workspace too small (ssnb_proposal_ar_workspace_bytes)");
  char* ws = (char*)workspace;
  if (!nr) nr = (int32_t*)(ws + L.nr);
  if (!first_hit) first_hit = (int32_t*)(ws + L.first_hit);
  unsigned long long* matches = (unsigned long long*)(ws + L.matches);
  double* pcn = (double*)(ws + L.pcn);
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(matches, 0, 8 * kPoints * (size_t)n_thresholds, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("proposal_ar: memset failed"); return SSNB_ECUDA; }
  cub::DoubleBuffer<unsigned long long> kb((unsigned long long*)(ws + L.keys0), (unsigned long long*)(ws + L.keys1));
  cub::DoubleBuffer<int> vb((int*)(ws + L.vals0), (int*)(ws + L.vals1));
  if (rows > 0) {
    const long long y = (rows / n_videos + kKeyThreads - 1) / kKeyThreads;
    const dim3 grid((unsigned)n_videos, (unsigned)(y < 1 ? 1 : y > kKeyChunksY ? kKeyChunksY : y));
    ar_keys_kernel<<<grid, kKeyThreads, 0, s>>>(scores, first, count, gt_offsets_dev, kb.Current(), vb.Current(), (int*)(ws + L.seg_begin),
                                                (int*)(ws + L.seg_end));
    SSNB_LAUNCH_CHECK("ar_keys_kernel");
    size_t cub_bytes = ar_cub_bytes(rows, n_videos);
    if (cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, (int)rows, n_videos, (const int*)(ws + L.seg_begin),
                                                 (const int*)(ws + L.seg_end), 0, 64, s) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("proposal_ar: ranking sort failed"); return SSNB_ECUDA; }
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  ar_budget_kernel<<<1, kBudgetThreads, 0, s>>>(count, gt_offsets_dev, p, nr, total_nr, pcn, proposals_per_video);
  SSNB_LAUNCH_CHECK("ar_budget_kernel");
  ar_first_hit_kernel<<<n_videos, 32 * kHitWarps, 0, s>>>((const double2*)boxes, vb.Current(), first, count, nr, (const double2*)gt_seg,
                                                          gt_offsets_dev, p, first_hit, (int32_t*)(ws + L.gt_cols));
  SSNB_LAUNCH_CHECK("ar_first_hit_kernel");
  ar_count_kernel<<<(unsigned)((p.n_gt + kCountChunk - 1) / kCountChunk), kCountThreads, 0, s>>>(first_hit, (int32_t*)(ws + L.gt_cols), pcn, p,
                                                                                                 matches);
  SSNB_LAUNCH_CHECK("ar_count_kernel");
  ar_finalise_kernel<<<1, 128, 0, s>>>(matches, total_nr, p, recall, avg_recall);
  SSNB_LAUNCH_CHECK("ar_finalise_kernel");
  return SSNB_OK;
}

}  // extern "C"
