// Proposal labelling on the GPU: the stage between "boxes" and "the SSN data set's tensors" of the reference, for many ragged
// videos per call.
//   gen_bottom_up_proposals.py:158-193 / gen_sliding_window_proposals.py:44-60   recall report, name_proposal, dump_window_list
//   ops/detection_metrics.py:7-83      temporal_iou, overlap_over_b, temporal_recall, name_proposal, get_temporal_proposal_recall
//   ops/sequence_funcs.py:37-54        gen_exponential_sw_proposal
//   ops/io.py:44-47,109-127            seconds / normalised -> frames
//   ssn_dataset.py:29-55,81-131,382-428   SSNVideoRecord validity, pools, regression targets and their statistics, get_test_data
//
//   name_proposals_kernel   one CTA per (video, 256-proposal chunk), one thread per proposal; the video's ground truth goes
//                           through shared memory 256 rows at a time; the per-ground-truth maximum tIoU is kept per CTA in
//                           shared memory and merged with a 64-bit atomicMax on the bit pattern (exact: non-negative doubles
//                           order like their bits, and a maximum does not depend on the order it is taken in)
//   recall_kernel           one CTA per video: hits per threshold from those maxima, integer atomics for the totals
//   sw_count_scan_kernel    one CTA: per (video, level) window count by bisection on the reference's own validity predicate
//                           (the valid windows of a level are a prefix), exclusive scan over the videos
//   sw_fill_kernel          the boxes, level-major, start ascending
//   frames_kernel           seconds / normalised -> frame integers, validity, clipped end, coverage
//   targets_kernel          one CTA per video: pool tags, regression targets, per-video pool counts and partial sums;
//   stats_*_kernel          reg_stats as a fixed-order two-stage reduction in double (per video, then over the videos)
//   test_props_kernel       rel_prop, proposal ticks, scaling, every operation rounded on its own in the order written
// All arithmetic that the reference does in Python floats is done with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn so
// that no FMA is contracted across it; min / max are Python's (the second argument wins only when strictly smaller / larger,
// so a NaN coordinate lands where the reference's does).
#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int kThreads = 256, kMaxThr = 32, kMaxLevel = 32, kMaxChunksY = 64;

__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }

// ops/detection_metrics.py:7-20 (and ops/utils.py:40-53): temporal_iou(A, B)
__device__ __forceinline__ double temporal_iou(double a0, double a1, double b0, double b1) {
  const double i0 = py_max(a0, b0), i1 = py_min(a1, b1);
  if (i0 >= i1) return 0.0;
  return __ddiv_rn(__dsub_rn(i1, i0), __dsub_rn(py_max(a1, b1), py_min(a0, b0)));
}

// ---- name_proposal + per-ground-truth maximum tIoU ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) name_proposals_kernel(const double2* __restrict__ boxes, const int64_t* __restrict__ first,
                                                                  const int32_t* __restrict__ count, const double2* __restrict__ gt,
                                                                  const int32_t* __restrict__ gt_label, const int64_t* __restrict__ gt_off,
                                                                  double thresh, int32_t* __restrict__ label, double* __restrict__ max_overlap,
                                                                  double* __restrict__ overlap_self, unsigned long long* __restrict__ gt_best) {
  __shared__ double2 s_gt[kThreads];
  __shared__ int s_lab[kThreads];
  __shared__ unsigned long long s_best[kThreads];
  const int v = blockIdx.x, tid = threadIdx.x;
  const int n = count[v];
  const long long f = first[v], g0 = gt_off[v];
  const long long G = gt_off[v + 1] - g0;
  for (long long c0 = (long long)blockIdx.y * kThreads; c0 < n; c0 += (long long)gridDim.y * kThreads) {
    const bool on = c0 + tid < n;
    const double2 es = on ? boxes[f + c0 + tid] : make_double2(0.0, 0.0);
    int lab = 0;
    double mo = 0.0, ms = 0.0;
    for (long long j0 = 0; j0 < G; j0 += kThreads) {
      const int m = (int)(G - j0 < kThreads ? G - j0 : kThreads);
      __syncthreads();
      if (tid < m) {
        s_gt[tid] = gt[g0 + j0 + tid];
        s_lab[tid] = gt_label[g0 + j0 + tid];
        s_best[tid] = 0ULL;
      }
      __syncthreads();
      if (on) {
        for (int j = 0; j < m; ++j) {
          const double2 gs = s_gt[j];
          const double i0 = py_max(gs.x, es.x), i1 = py_min(gs.y, es.y);
          if (i0 >= i1) continue;                      // both overlaps are 0: never selected (0 > max_overlap is false)
          const double inter = __dsub_rn(i1, i0);
          const double ov = __ddiv_rn(inter, __dsub_rn(py_max(gs.y, es.y), py_min(gs.x, es.x)));
          if (ov > thresh && ov > mo) {                // ground-truth order: the first of equal overlaps stays; NaN never wins
            lab = s_lab[j] + 1;
            mo = ov;
            ms = __ddiv_rn(inter, __dsub_rn(es.y, es.x));   // overlap_over_b(gs, es)
          }
          if (ov > 0.0) {                              // NaN is above no threshold (temporal_recall: tIoU > th)
            const unsigned long long bits = (unsigned long long)__double_as_longlong(ov);
            if (bits > *(volatile unsigned long long*)&s_best[j]) atomicMax(&s_best[j], bits);
          }
        }
      }
      __syncthreads();
      if (tid < m && s_best[tid]) atomicMax(&gt_best[g0 + j0 + tid], s_best[tid]);
    }
    if (on) {
      label[f + c0 + tid] = lab;
      max_overlap[f + c0 + tid] = mo;
      overlap_self[f + c0 + tid] = ms;
    }
  }
}

// ---- temporal_recall / get_temporal_proposal_recall --------------------------------------------------------------------------
struct RecallParams { int n_thr; double thr[kMaxThr]; };

__global__ void __launch_bounds__(kThreads) recall_kernel(const double* __restrict__ gt_best, const int64_t* __restrict__ gt_off, RecallParams p,
                                                          int32_t* __restrict__ hits, long long* __restrict__ totals) {
  __shared__ int s_hit[kMaxThr];
  const int v = blockIdx.x, tid = threadIdx.x;
  if (tid < p.n_thr) s_hit[tid] = 0;
  __syncthreads();
  const long long g0 = gt_off[v], G = gt_off[v + 1] - g0;
  for (long long j = tid; j < G; j += kThreads) {
    const double b = gt_best[g0 + j];
    for (int t = 0; t < p.n_thr; ++t)
      if (b > p.thr[t]) atomicAdd(&s_hit[t], 1);
  }
  __syncthreads();
  if (tid < p.n_thr) {
    const int h = s_hit[tid];
    hits[(long long)v * p.n_thr + tid] = h;
    if (h == G) atomicAdd((unsigned long long*)&totals[tid], 1ULL);                 // videos with every instance recalled
    if (h) atomicAdd((unsigned long long*)&totals[p.n_thr + tid], (unsigned long long)h);
  }
  if (tid == 0 && G) atomicAdd((unsigned long long*)&totals[2 * p.n_thr], (unsigned long long)G);
}

// ---- gen_exponential_sw_proposal ---------------------------------------------------------------------------------------------
struct SwParams { int L; double t_span[kMaxLevel]; double step[kMaxLevel]; };

// valid_proposal (ops/sequence_funcs.py:49-51) of window k of a level
__device__ __forceinline__ bool sw_valid(double duration, double step, double t_span, int k) {
  const double s = __dmul_rn((double)k, step);
  return __dsub_rn(py_min(duration, __dadd_rn(s, t_span)), s) >= 1.0;
}

// np.arange(0, duration, step) has ceil(duration / step) elements; the valid ones are a prefix (min(duration, end) - start
// does not grow with the start), found by bisection on the predicate itself
__device__ int sw_level_count(double duration, double step, double t_span) {
  if (!(duration > 0.0) || isinf(duration)) return 0;
  const double nk = ceil(__ddiv_rn(duration, step));
  int lo = 0, hi = nk < (double)INT_MAX ? (int)nk : INT_MAX;
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (sw_valid(duration, step, t_span, mid)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

constexpr int kScanThreads = 1024;
__global__ void __launch_bounds__(kScanThreads) sw_count_scan_kernel(const double* __restrict__ durations, int V, SwParams p,
                                                                     int32_t* __restrict__ level_count, int32_t* __restrict__ count,
                                                                     int64_t* __restrict__ first, int64_t* __restrict__ total) {
  __shared__ long long s_sum[kScanThreads];
  const int tid = threadIdx.x, per = (V + kScanThreads - 1) / kScanThreads;
  const int v0 = tid * per, v1 = v0 + per < V ? v0 + per : V;
  long long acc = 0;
  for (int v = v0; v < v1; ++v) {
    const double d = durations[v];
    long long n = 0;
    for (int l = 0; l < p.L; ++l) {
      const int c = sw_level_count(d, p.step[l], p.t_span[l]);
      level_count[(long long)v * p.L + l] = c;
      n += c;
    }
    if (n > INT_MAX) n = INT_MAX;
    count[v] = (int)n;
    acc += n;
  }
  s_sum[tid] = acc;
  __syncthreads();
  if (tid == 0) {
    long long run = 0;
    for (int i = 0; i < kScanThreads; ++i) { const long long t = s_sum[i]; s_sum[i] = run; run += t; }
    total[0] = run;
  }
  __syncthreads();
  long long run = s_sum[tid];
  for (int v = v0; v < v1; ++v) { first[v] = run; run += count[v]; }
}

__global__ void __launch_bounds__(kThreads) sw_fill_kernel(SwParams p, const int32_t* __restrict__ level_count, const int32_t* __restrict__ count,
                                                           const int64_t* __restrict__ first, long long capacity, double2* __restrict__ boxes) {
  __shared__ int s_pre[kMaxLevel + 1];
  const int v = blockIdx.x;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int l = 0; l < p.L; ++l) { s_pre[l] = acc; acc += level_count[(long long)v * p.L + l]; }
    s_pre[p.L] = acc;
  }
  __syncthreads();
  const int n = count[v];
  const long long f = first[v];
  for (long long r = (long long)blockIdx.y * kThreads + threadIdx.x; r < n; r += (long long)gridDim.y * kThreads) {
    int l = 0;
    while (l + 1 < p.L && r >= s_pre[l + 1]) ++l;
    const double s = __dmul_rn((double)(r - s_pre[l]), p.step[l]);
    if (f + r < capacity) boxes[f + r] = make_double2(s, __dadd_rn(s, p.t_span[l]));
  }
}

// ---- seconds / normalised -> frames, SSNVideoRecord validity -----------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) frames_kernel(const double2* __restrict__ boxes, const int64_t* __restrict__ first,
                                                          const int32_t* __restrict__ count, const double* __restrict__ durations,
                                                          const int32_t* __restrict__ frame_cnt, int mode, int64_t* __restrict__ frames,
                                                          int64_t* __restrict__ valid, double* __restrict__ coverage, uint8_t* __restrict__ keep) {
  const int v = blockIdx.x;
  const int n = count[v];
  const long long f = first[v], fc = frame_cnt[v];
  // dump_window_list: real_fps = float(frame_cnt) / float(duration); process_proposal_list: float(x) * frame_cnt
  const double mul = mode == SSNB_PROPFRAMES_SECONDS ? __ddiv_rn((double)fc, durations[v]) : (double)fc;
  for (long long r = (long long)blockIdx.y * kThreads + threadIdx.x; r < n; r += (long long)gridDim.y * kThreads) {
    const double2 b = boxes[f + r];
    long long s, e;
    if (mode == SSNB_PROPFRAMES_AS_GIVEN) { s = __double2ll_rz(b.x); e = __double2ll_rz(b.y); }
    else { s = __double2ll_rz(__dmul_rn(b.x, mul)); e = __double2ll_rz(__dmul_rn(b.y, mul)); }
    frames[2 * (f + r)] = s;
    frames[2 * (f + r) + 1] = e;
    if (valid) { valid[2 * (f + r)] = s; valid[2 * (f + r) + 1] = e < fc ? e : fc; }
    if (coverage) coverage[f + r] = __ddiv_rn((double)(e - s), (double)fc);      // the unclipped end (ssn_dataset.py:21)
    if (keep) keep[f + r] = (e > s && s < fc) ? 1 : 0;
  }
}

// ---- pools, regression targets, reg_stats ------------------------------------------------------------------------------------
// sum of one double per thread in a fixed order: the tree over thread indices
__device__ double block_sum(double x, double* s) {
  __syncthreads();
  s[threadIdx.x] = x;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + w]);
    __syncthreads();
  }
  return s[0];
}

struct TargetParams {
  double fg_thresh, incomplete_iou_thresh, bg_iou_thresh, bg_coverage_thresh, incomplete_overlap_thresh;
  int exclude_empty;
};

__global__ void __launch_bounds__(kThreads) targets_kernel(const int64_t* __restrict__ frames, const double* __restrict__ best_iou,
                                                           const double* __restrict__ overlap_self, const double* __restrict__ coverage,
                                                           const int64_t* __restrict__ first, const int32_t* __restrict__ count,
                                                           const int64_t* __restrict__ gt_frames, const int64_t* __restrict__ gt_off, TargetParams p,
                                                           uint8_t* __restrict__ tags, double* __restrict__ reg, int32_t* __restrict__ pool_counts,
                                                           double* __restrict__ partial) {
  __shared__ double s_red[kThreads];
  const int v = blockIdx.x, tid = threadIdx.x;
  const int n = count[v];
  const long long f = first[v], g0 = gt_off[v], G = gt_off[v + 1] - g0;
  const bool used = !(p.exclude_empty && G == 0);
  int n_fg = 0, n_inc = 0, n_bg = 0;
  double s_loc = 0.0, s_size = 0.0;
  for (long long r = tid; r < n; r += kThreads) {
    const long long i = f + r;
    uint8_t tag = 0;
    double loc = 0.0, size = 0.0;
    if (used) {
      const double iou = best_iou[i], os = overlap_self[i];
      const bool fg = iou > p.fg_thresh;                                                     // get_fg (:104)
      const bool inc = iou < p.incomplete_iou_thresh && os > p.incomplete_overlap_thresh;    // get_negatives (:121-124)
      const bool bg = !inc && iou < p.bg_iou_thresh && coverage[i] > p.bg_coverage_thresh;   // (:127-130)
      tag = (fg ? SSNB_TAG_FG : 0) | (inc ? SSNB_TAG_INCOMPLETE : 0) | (bg ? SSNB_TAG_BACKGROUND : 0);
      n_fg += fg; n_inc += inc; n_bg += bg;
      if (fg && G > 0) {                                                                     // compute_regression_targets (:29-55)
        const long long ps = frames[2 * i], pe = frames[2 * i + 1];
        double best = -1.0;
        long long bs = 0, be = 0;
        for (long long j = 0; j < G; ++j) {                                                  // np.argmax: the first maximum
          const long long gs = gt_frames[2 * (g0 + j)], ge = gt_frames[2 * (g0 + j) + 1];
          const double ov = temporal_iou((double)ps, (double)pe, (double)gs, (double)ge);
          if (ov > best) { best = ov; bs = gs; be = ge; }
        }
        const double pc = __ddiv_rn((double)(ps + pe), 2.0), gc = __ddiv_rn((double)(bs + be), 2.0);
        const double psz = (double)(pe - ps + 1), gsz = (double)(be - bs + 1);
        loc = __ddiv_rn(__dsub_rn(gc, pc), psz);
        size = log(__ddiv_rn(gsz, psz));
        s_loc = __dadd_rn(s_loc, loc);
        s_size = __dadd_rn(s_size, size);
      }
    }
    tags[i] = tag;
    reg[2 * i] = loc;
    reg[2 * i + 1] = size;
  }
  // integers are exact in double far beyond any row count
  const double t_fg = block_sum((double)n_fg, s_red), t_inc = block_sum((double)n_inc, s_red), t_bg = block_sum((double)n_bg, s_red);
  const double t_loc = block_sum(s_loc, s_red), t_size = block_sum(s_size, s_red);
  if (tid == 0) {
    pool_counts[4 * v] = (int)t_fg;
    pool_counts[4 * v + 1] = (int)t_inc;
    pool_counts[4 * v + 2] = (int)t_bg;
    pool_counts[4 * v + 3] = used ? (int)G : 0;
    partial[3 * v] = t_fg;
    partial[3 * v + 1] = t_loc;
    partial[3 * v + 2] = t_size;
  }
}

// over the videos in a fixed order: pool totals (exact integers) and the mean of the fg targets
__global__ void __launch_bounds__(kThreads) stats_mean_kernel(const double* __restrict__ partial, const int32_t* __restrict__ pool_counts,
                                                              const int64_t* __restrict__ gt_off, int V, int exclude_empty,
                                                              int64_t* __restrict__ totals, double* __restrict__ stats) {
  __shared__ double s_red[kThreads];
  double a[3] = {0.0, 0.0, 0.0};
  long long c[5] = {0, 0, 0, 0, 0};
  for (int v = threadIdx.x; v < V; v += kThreads) {
    for (int k = 0; k < 3; ++k) a[k] = __dadd_rn(a[k], partial[3 * v + k]);
    for (int k = 0; k < 4; ++k) c[k] += pool_counts[4 * v + k];
    c[4] += !(exclude_empty && gt_off[v + 1] == gt_off[v]);
  }
  double t[3];
  for (int k = 0; k < 3; ++k) t[k] = block_sum(a[k], s_red);
  long long tc[5];
  for (int k = 0; k < 5; ++k) tc[k] = (long long)block_sum((double)c[k], s_red);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 5; ++k) totals[k] = tc[k];      // fg, incomplete, background, ground truth, videos
    stats[0] = __ddiv_rn(t[1], t[0]);                   // no fg proposal at all: 0 / 0 = NaN, numpy's mean of nothing
    stats[1] = __ddiv_rn(t[2], t[0]);
  }
}

__global__ void __launch_bounds__(kThreads) stats_var_kernel(const uint8_t* __restrict__ tags, const double* __restrict__ reg,
                                                             const int64_t* __restrict__ first, const int32_t* __restrict__ count,
                                                             const double* __restrict__ stats, double* __restrict__ partial2) {
  __shared__ double s_red[kThreads];
  const int v = blockIdx.x;
  const int n = count[v];
  const long long f = first[v];
  const double m0 = stats[0], m1 = stats[1];
  double a0 = 0.0, a1 = 0.0;
  for (long long r = threadIdx.x; r < n; r += kThreads) {
    if (!(tags[f + r] & SSNB_TAG_FG)) continue;
    const double d0 = __dsub_rn(reg[2 * (f + r)], m0), d1 = __dsub_rn(reg[2 * (f + r) + 1], m1);
    a0 = __dadd_rn(a0, __dmul_rn(d0, d0));
    a1 = __dadd_rn(a1, __dmul_rn(d1, d1));
  }
  const double t0 = block_sum(a0, s_red), t1 = block_sum(a1, s_red);
  if (threadIdx.x == 0) { partial2[2 * v] = t0; partial2[2 * v + 1] = t1; }
}

__global__ void __launch_bounds__(kThreads) stats_std_kernel(const double* __restrict__ partial2, int V, const int64_t* __restrict__ totals,
                                                             double* __restrict__ stats) {
  __shared__ double s_red[kThreads];
  double a0 = 0.0, a1 = 0.0;
  for (int v = threadIdx.x; v < V; v += kThreads) {
    a0 = __dadd_rn(a0, partial2[2 * v]);
    a1 = __dadd_rn(a1, partial2[2 * v + 1]);
  }
  const double t0 = block_sum(a0, s_red), t1 = block_sum(a1, s_red);
  if (threadIdx.x == 0) {
    const double n = (double)totals[0];
    stats[2] = sqrt(__ddiv_rn(t0, n));
    stats[3] = sqrt(__ddiv_rn(t1, n));
  }
}

// ---- get_test_data's proposal half -------------------------------------------------------------------------------------------
__device__ __forceinline__ void test_row(long long s, long long e, double fc, double nt, long long o, double* __restrict__ rel_prop,
                                         int64_t* __restrict__ ticks, double* __restrict__ scaling, int32_t* __restrict__ ticks32,
                                         float* __restrict__ scaling32) {
  const double r0 = __ddiv_rn((double)s, fc), r1 = __ddiv_rn((double)e, fc);          // :410
  const double dur = __dsub_rn(r1, r0);
  const double sd = __dmul_rn(dur, 0.5), ed = __dmul_rn(dur, 0.5);                    // starting_ratio, ending_ratio
  const double rs = py_max(0.0, __dsub_rn(r0, sd)), re = py_min(1.0, __dadd_rn(r1, ed));
  const double sc0 = __ddiv_rn(__dsub_rn(r0, rs), sd), sc1 = __ddiv_rn(__dsub_rn(re, r1), ed);
  const long long t[4] = {__double2ll_rz(__dmul_rn(rs, nt)), __double2ll_rz(__dmul_rn(r0, nt)), __double2ll_rz(__dmul_rn(r1, nt)),
                          __double2ll_rz(__dmul_rn(re, nt))};
  rel_prop[2 * o] = r0; rel_prop[2 * o + 1] = r1;
  scaling[2 * o] = sc0; scaling[2 * o + 1] = sc1;
  for (int k = 0; k < 4; ++k) ticks[4 * o + k] = t[k];
  if (ticks32) for (int k = 0; k < 4; ++k) ticks32[4 * o + k] = (int32_t)t[k];
  if (scaling32) { scaling32[2 * o] = (float)sc0; scaling32[2 * o + 1] = (float)sc1; }
}

__global__ void __launch_bounds__(kThreads) test_props_kernel(const int64_t* __restrict__ frames, const int64_t* __restrict__ first,
                                                              const int32_t* __restrict__ count, const int64_t* __restrict__ out_first,
                                                              const int32_t* __restrict__ frame_cnt, int new_length, int test_interval,
                                                              int32_t* __restrict__ num_ticks, double* __restrict__ rel_prop, int64_t* __restrict__ ticks,
                                                              double* __restrict__ scaling, int32_t* __restrict__ ticks32, float* __restrict__ scaling32) {
  const int v = blockIdx.x;
  const int n = count[v];
  const long long f = first[v], o = out_first[v], fc = frame_cnt[v];
  // len(np.arange(0, frame_cnt - new_length, test_interval))
  const long long span = fc - new_length;
  const long long nt = span > 0 ? (span + test_interval - 1) / test_interval : 0;
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    num_ticks[v] = (int)nt;
    if (n == 0) test_row(0, fc - 1, (double)fc, (double)nt, o, rel_prop, ticks, scaling, ticks32, scaling32);   // :402-403
  }
  for (long long r = (long long)blockIdx.y * kThreads + threadIdx.x; r < n; r += (long long)gridDim.y * kThreads)
    test_row(frames[2 * (f + r)], frames[2 * (f + r) + 1], (double)fc, (double)nt, o + r, rel_prop, ticks, scaling, ticks32, scaling32);
}

// CTAs per video of the row kernels: enough for max_count rows at one row per thread, capped (the kernels loop beyond)
dim3 row_grid(int V, int64_t max_count) {
  long long y = (max_count + kThreads - 1) / kThreads;
  return dim3((unsigned)V, (unsigned)(y < 1 ? 1 : y > kMaxChunksY ? kMaxChunksY : y));
}

bool ascending(const int64_t* off, int V) {
  if (off[0] != 0) return false;
  for (int v = 0; v < V; ++v)
    if (off[v + 1] < off[v]) return false;
  return true;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_name_proposals(const double* boxes, const int64_t* first, const int32_t* count, int n_videos, int64_t max_count, const double* gt,
                        const int32_t* gt_label, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, double thresh, int32_t* label,
                        double* max_overlap, double* overlap_self, double* gt_best, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("name_proposals: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 0 || max_count < 0) return fail("negative count");
  if (!gt_offsets || !ascending(gt_offsets, n_videos)) return fail("gt_offsets must start at 0 and ascend");
  const int64_t n_gt = gt_offsets[n_videos];
  if (n_videos == 0) return SSNB_OK;
  if (!boxes || !first || !count || !gt_offsets_dev || !label || !max_overlap || !overlap_self || !gt_best) return fail("null argument");
  if (n_gt > 0 && (!gt || !gt_label)) return fail("null ground truth");
  if (thresh != thresh) return fail("thresh is NaN");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_gt > 0 && cudaMemsetAsync(gt_best, 0, sizeof(double) * (size_t)n_gt, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("name_proposals: memset failed"); return SSNB_ECUDA; }
  name_proposals_kernel<<<row_grid(n_videos, max_count), kThreads, 0, s>>>((const double2*)boxes, first, count, (const double2*)gt, gt_label,
                                                                           gt_offsets_dev, thresh, label, max_overlap, overlap_self,
                                                                           (unsigned long long*)gt_best);
  SSNB_LAUNCH_CHECK("name_proposals_kernel");
  return SSNB_OK;
}

int ssnb_proposal_recall(const double* gt_best, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, int n_videos, const double* thresholds,
                         int n_thresholds, int32_t* hits, int64_t* totals, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("proposal_recall: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 0) return fail("negative count");
  if (n_thresholds < 1 || n_thresholds > kMaxThr || !thresholds) return fail("1..32 thresholds");
  if (!gt_offsets || !ascending(gt_offsets, n_videos)) return fail("gt_offsets must start at 0 and ascend");
  if (!totals) return fail("null argument");
  if (n_videos > 0 && (!hits || !gt_offsets_dev || (gt_offsets[n_videos] > 0 && !gt_best))) return fail("null argument");
  RecallParams p;
  p.n_thr = n_thresholds;
  for (int t = 0; t < n_thresholds; ++t) p.thr[t] = thresholds[t];
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(totals, 0, sizeof(int64_t) * (2 * n_thresholds + 1), s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("proposal_recall: memset failed"); return SSNB_ECUDA; }
  if (n_videos == 0) return SSNB_OK;
  recall_kernel<<<n_videos, kThreads, 0, s>>>(gt_best, gt_offsets_dev, p, hits, (long long*)totals);
  SSNB_LAUNCH_CHECK("recall_kernel");
  return SSNB_OK;
}

int ssnb_sliding_windows(const double* durations, int n_videos, const double* t_spans, const double* steps, int n_levels, int64_t max_count,
                         int64_t capacity, double* boxes, int64_t* first, int32_t* count, int32_t* level_count, int64_t* total, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("sliding_windows: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 0 || max_count < 0 || capacity < 0) return fail("negative count");
  if (n_levels < 1 || n_levels > kMaxLevel || !t_spans || !steps) return fail("1..32 levels");
  SwParams p;
  p.L = n_levels;
  for (int l = 0; l < n_levels; ++l) {
    if (!(t_spans[l] >= 1.0) || !(steps[l] >= 1.0) || t_spans[l] > 1e15 || steps[l] > 1e15 || steps[l] != floor(steps[l]))
      return fail("t_span >= 1 and an integer step >= 1 per level");
    p.t_span[l] = t_spans[l];
    p.step[l] = steps[l];
  }
  if (!total) return fail("null argument");
  if (n_videos > 0 && (!durations || !first || !count || !level_count || (capacity > 0 && !boxes))) return fail("null argument");
  cudaStream_t s = (cudaStream_t)stream;
  sw_count_scan_kernel<<<1, kScanThreads, 0, s>>>(durations, n_videos, p, level_count, count, first, total);
  SSNB_LAUNCH_CHECK("sw_count_scan_kernel");
  if (n_videos == 0 || capacity == 0) return SSNB_OK;
  sw_fill_kernel<<<row_grid(n_videos, max_count), kThreads, 0, s>>>(p, level_count, count, first, capacity, (double2*)boxes);
  SSNB_LAUNCH_CHECK("sw_fill_kernel");
  return SSNB_OK;
}

int ssnb_proposal_frames(const double* boxes, const int64_t* first, const int32_t* count, int n_videos, int64_t max_count, const double* durations,
                         const int32_t* frame_cnt, int mode, int64_t* frames, int64_t* valid, double* coverage, uint8_t* keep, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("proposal_frames: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 0 || max_count < 0) return fail("negative count");
  if (mode != SSNB_PROPFRAMES_SECONDS && mode != SSNB_PROPFRAMES_NORMALISED && mode != SSNB_PROPFRAMES_AS_GIVEN) return fail("unknown mode");
  if (n_videos == 0) return SSNB_OK;
  if (!boxes || !first || !count || !frame_cnt || !frames) return fail("null argument");
  if (mode == SSNB_PROPFRAMES_SECONDS && !durations) return fail("seconds need durations");
  cudaStream_t s = (cudaStream_t)stream;
  frames_kernel<<<row_grid(n_videos, max_count), kThreads, 0, s>>>((const double2*)boxes, first, count, durations, frame_cnt, mode, frames, valid,
                                                                   coverage, keep);
  SSNB_LAUNCH_CHECK("frames_kernel");
  return SSNB_OK;
}

size_t ssnb_proposal_targets_workspace_bytes(int n_videos) { return n_videos < 0 ? 0 : sizeof(double) * 5 * (size_t)(n_videos > 0 ? n_videos : 1); }

int ssnb_proposal_targets(const ssnb_proposal_targets_cfg* cfg, const int64_t* frames, const double* best_iou, const double* overlap_self,
                          const double* coverage, const int64_t* first, const int32_t* count, int n_videos, const int64_t* gt_frames,
                          const int64_t* gt_offsets, const int64_t* gt_offsets_dev, uint8_t* tags, double* reg, int32_t* pool_counts,
                          int64_t* totals, double* stats, void* workspace, size_t workspace_bytes, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("proposal_targets: " + m); return (int)SSNB_EINVAL; };
  if (!cfg) return fail("null cfg");
  if (n_videos < 0) return fail("negative count");
  if (!gt_offsets || !ascending(gt_offsets, n_videos)) return fail("gt_offsets must start at 0 and ascend");
  if (!totals || !stats) return fail("null argument");
  if (n_videos > 0 && (!frames || !best_iou || !overlap_self || !coverage || !first || !count || !gt_offsets_dev || !tags || !reg || !pool_counts))
    return fail("null argument");
  if (gt_offsets[n_videos] > 0 && !gt_frames) return fail("null ground truth");
  if (!workspace || workspace_bytes < ssnb_proposal_targets_workspace_bytes(n_videos)) return fail("workspace too small");
  const TargetParams p = {cfg->fg_thresh, cfg->incomplete_iou_thresh, cfg->bg_iou_thresh, cfg->bg_coverage_thresh,
                          cfg->incomplete_overlap_thresh, cfg->exclude_empty};
  double* partial = (double*)workspace;
  double* partial2 = partial + 3 * (size_t)n_videos;
  cudaStream_t s = (cudaStream_t)stream;
  if (n_videos > 0) {
    targets_kernel<<<n_videos, kThreads, 0, s>>>(frames, best_iou, overlap_self, coverage, first, count, gt_frames, gt_offsets_dev, p, tags, reg,
                                                 pool_counts, partial);
    SSNB_LAUNCH_CHECK("targets_kernel");
  }
  stats_mean_kernel<<<1, kThreads, 0, s>>>(partial, pool_counts, gt_offsets_dev, n_videos, p.exclude_empty, totals, stats);
  SSNB_LAUNCH_CHECK("stats_mean_kernel");
  if (n_videos > 0) {
    stats_var_kernel<<<n_videos, kThreads, 0, s>>>(tags, reg, first, count, stats, partial2);
    SSNB_LAUNCH_CHECK("stats_var_kernel");
  }
  stats_std_kernel<<<1, kThreads, 0, s>>>(partial2, n_videos, totals, stats);
  SSNB_LAUNCH_CHECK("stats_std_kernel");
  return SSNB_OK;
}

int ssnb_test_proposals(const int64_t* frames, const int64_t* first, const int32_t* count, const int64_t* out_first, int n_videos,
                        int64_t max_count, const int32_t* frame_cnt, int new_length, int test_interval, int32_t* num_ticks, double* rel_prop,
                        int64_t* ticks, double* scaling, int32_t* ticks32, float* scaling32, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("test_proposals: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 0 || max_count < 0) return fail("negative count");
  if (new_length < 1 || test_interval < 1) return fail("new_length and test_interval must be >= 1");
  if (n_videos == 0) return SSNB_OK;
  if (!frames || !first || !count || !out_first || !frame_cnt || !num_ticks || !rel_prop || !ticks || !scaling) return fail("null argument");
  cudaStream_t s = (cudaStream_t)stream;
  test_props_kernel<<<row_grid(n_videos, max_count), kThreads, 0, s>>>(frames, first, count, out_first, frame_cnt, new_length, test_interval,
                                                                       num_ticks, rel_prop, ticks, scaling, ticks32, scaling32);
  SSNB_LAUNCH_CHECK("test_props_kernel");
  return SSNB_OK;
}

}  // extern "C"
