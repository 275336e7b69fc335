// Detection post-processing on the GPU (SURVEY section 8 f3): what eval_detection_results.py:91-183 does per video with
// numpy -- combined scores softmax(act)[:, 1:] * exp(comp) (:104, ops/utils.py:38-40), class-wise temporal NMS
// (ops/utils.py:56-82) and location regression (:147-160) -- as two kernels: one thread per proposal row for the scores,
// one CTA per class for sort + greedy NMS + regression.  Semantics kept: scores sorted descending, a box survives when its
// IoU with every kept box is <= thresh, IoU = inter / (dur_i + dur_j - inter) with a possibly NEGATIVE inter (disjoint boxes
// are never suppressed) and the division carried out in double like numpy's `.astype(float)`.
//
// ssnb_detect_batch does the same for many ragged videos in one call, in all three branches of gen_detection_results:
//   batch_desc_kernel     one CTA: per video its rows, its candidate pairs and its slot range (a block scan of the slots)
//   batch_scores_kernel   one thread per proposal row: the branch's combined scores
//   candidates_kernel     one thread per candidate (proposal, class) pair: descending radix key, pairs in reverse order
//   cub segmented radix sort per video by score (stable, so equal scores keep the reverse order: larger index first)
//   select_kernel         the first S_v sorted pairs of each video (top_k: min(top_k, N K); else all), keyed by class
//   cub segmented radix sort per video by class (stable: every class keeps the score order)
//   runs_kernel           where each (video, class) run of the sorted list starts and ends
//   batch_nms_kernel      one CTA per (video, class): nms_regress_list over the run, the one loop nms_regress_kernel runs
//   compact_kernel        one CTA per video: the survivors class by class from the video's first slot on
#include <cub/cub.cuh>

#include <cfloat>
#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

// combined[i, c] = softmax(act[i, :])[c + 1] * exp(comp[i, c])
__global__ void combined_scores_kernel(const float* __restrict__ act, const float* __restrict__ comp, int N, int K, float* __restrict__ combined) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* a = act + (long long)i * (K + 1);
  float m = a[0];
  for (int j = 1; j <= K; ++j) m = fmaxf(m, a[j]);
  float sum = 0.f;
  for (int j = 0; j <= K; ++j) sum += expf(a[j] - m);
  for (int c = 0; c < K; ++c) combined[(long long)i * K + c] = (expf(a[c + 1] - m) / sum) * expf(comp[(long long)i * K + c]);
}

// (score, index) a precedes b in the sorted list: NaN first (numpy's argsort()[::-1] puts NaN first), then larger score, ties
// and NaN against NaN: larger index first (a stable ascending argsort reversed); the padding (index < 0) after everything
__device__ __forceinline__ bool nms_precedes(float ka, int ia, float kb, int ib) {
  if (ia < 0 || ib < 0) return ib < 0 && ia >= 0;
  const bool na = ka != ka, nb = kb != kb;
  if (na || nb) return na && (!nb || ia > ib);
  return ka > kb || (ka == kb && ia > ib);
}

// greedy temporal NMS (ops/utils.py:56-82) over one list already in ranking order, and the regression of its survivors
// (eval_detection_results.py:162-174, fp32 like the numpy arrays), run by every thread of the CTA.  key / idx / t1 / t2 are
// the sorted scores, proposal rows and boxes, alive[i] = 1 for each entry (global or shared memory, all written before a
// barrier).  Survivor o goes to out[5 o .. 5 o + 4]; (loc, dur) of row s are reg[s * reg_stride + reg_off + {0, 1}], or
// zeros when reg is NULL.  *n_kept (shared) ends at the number kept, visible to thread 0.
__device__ __forceinline__ void nms_regress_list(int N, const float* key, const int* idx, const float* t1, const float* t2,
                                                 unsigned char* alive, const float* __restrict__ reg, long long reg_stride, int reg_off,
                                                 double thresh, int regress, float* __restrict__ out, int* n_kept) {
  if (threadIdx.x == 0) *n_kept = 0;
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    if (!alive[i]) continue;                                // uniform: written before the last barrier
    const float a1 = t1[i], a2 = t2[i], da = a2 - a1;
    if (threadIdx.x == 0) {
      const int s = idx[i], o = (*n_kept)++;
      float* q = out + (long long)o * 5;
      const float loc = reg ? reg[(long long)s * reg_stride + reg_off] : 0.f, dur = reg ? reg[(long long)s * reg_stride + reg_off + 1] : 0.f;
      float b1 = a1, b2 = a2;
      if (regress) {
        const float center = (a1 + a2) / 2, duration = a2 - a1;
        const float nc = center + duration * loc, nd = duration * expf(dur);
        b1 = fminf(fmaxf(nc - nd / 2, 0.f), 1.f); b2 = fminf(fmaxf(nc + nd / 2, 0.f), 1.f);
      }
      q[0] = b1; q[1] = b2; q[2] = key[i]; q[3] = loc; q[4] = dur;
    }
    for (int j = i + 1 + threadIdx.x; j < N; j += blockDim.x) {
      if (!alive[j]) continue;
      const float inter = fminf(a2, t2[j]) - fmaxf(a1, t1[j]);
      const float den = da + (t2[j] - t1[j]) - inter;
      const double iou = (double)inter / (double)den;
      if (!(iou <= thresh)) alive[j] = 0;           // np.where(IoU <= thresh): NaN is dropped as well
    }
    __syncthreads();
  }
}

// one CTA per class: bitonic sort of (score, index) in nms_precedes order, greedy NMS over the sorted list, regression of the
// survivors, written in kept order
__global__ void __launch_bounds__(256) nms_regress_kernel(const float* __restrict__ props, const float* __restrict__ combined,
                                                          const float* __restrict__ reg, int N, int K, int P, double thresh, int regress,
                                                          float* __restrict__ out, int* __restrict__ count) {
  extern __shared__ unsigned char sm_raw[];
  float* key = reinterpret_cast<float*>(sm_raw);          // [P]
  int* idx = reinterpret_cast<int*>(key + P);              // [P]
  float* t1 = reinterpret_cast<float*>(idx + P);           // [P] sorted order
  float* t2 = t1 + P;
  unsigned char* alive = reinterpret_cast<unsigned char*>(t2 + P);
  __shared__ int n_kept;
  const int c = blockIdx.x;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    key[i] = i < N ? combined[(long long)i * K + c] : -INFINITY;
    idx[i] = i < N ? i : -1;
  }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const bool desc = (i & k) == 0;                   // this run sorted descending
          const float ka = key[i], kb = key[l];
          const int ia = idx[i], ib = idx[l];
          const bool a_first = nms_precedes(ka, ia, kb, ib);
          if (a_first != desc) { key[i] = kb; key[l] = ka; idx[i] = ib; idx[l] = ia; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < N; i += blockDim.x) {       // the padding sorts after the N proposals: s >= 0 here
    const int s = idx[i];
    t1[i] = s >= 0 ? props[2 * s] : 0.f; t2[i] = s >= 0 ? props[2 * s + 1] : 0.f;
    alive[i] = s >= 0;
  }
  nms_regress_list(N, key, idx, t1, t2, alive, reg, 2LL * K, 2 * c, thresh, regress, out + (long long)c * N * 5, &n_kept);
  if (threadIdx.x == 0) count[c] = n_kept;
}


// ---- many videos: ssnb_detect_batch ----------------------------------------------------------------------------------------
constexpr int kDescThreads = 256, kBatchNmsThreads = 256;

struct BatchDesc {
  int row0, n;          // the video's proposal rows
  int cand0, n_cand;    // its candidate pairs in the score sort: N K (all, top_k) or N n_sel (cls)
  int slot0, n_slot;    // its slots: N K, min(top_k, N K) or N n_sel
};

struct BatchParams {
  int V, K, mode, top_k, n_sel, sbf;
};

// the last video whose range starts at or before i (empty videos share a start with the next one and are skipped)
template <int BatchDesc::*start>
__device__ __forceinline__ int video_at(const BatchDesc* __restrict__ d, int V, long long i) {
  int lo = 0, hi = V - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (d[mid].*start <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// one CTA: per video its rows, candidates and slots; the slot starts are an exclusive scan of the slot counts
__global__ void __launch_bounds__(kDescThreads) batch_desc_kernel(const int64_t* __restrict__ offsets, BatchParams p, BatchDesc* __restrict__ desc,
                                                                   int* __restrict__ cand_begin, int* __restrict__ cand_end, int* __restrict__ slot_begin,
                                                                   int* __restrict__ slot_end) {
  using Scan = cub::BlockScan<int, kDescThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int base = 0; base < p.V; base += kDescThreads) {
    const int v = base + threadIdx.x;
    BatchDesc d{};
    if (v < p.V) {
      d.row0 = (int)offsets[v];
      d.n = (int)(offsets[v + 1] - offsets[v]);
      const int per = p.mode == SSNB_DET_CLS ? p.n_sel : p.K;
      d.cand0 = d.row0 * per;
      d.n_cand = d.n * per;
      d.n_slot = p.mode == SSNB_DET_TOPK ? min(p.top_k, d.n_cand) : d.n_cand;
    }
    int x, tot;
    Scan(tmp).ExclusiveSum(d.n_slot, x, tot);
    __syncthreads();
    if (v < p.V) {
      d.slot0 = carry + x;
      desc[v] = d;
      cand_begin[v] = d.cand0; cand_end[v] = d.cand0 + d.n_cand;
      slot_begin[v] = d.slot0; slot_end[v] = d.slot0 + d.n_slot;
    }
    carry += tot;
  }
}

// the branch's combined scores of one proposal row (fp32, as numpy computes them on the fp32 arrays):
//   all, cls + softmax_before_filter: softmax(act)[:, 1:] * exp(comp)  (the expressions of combined_scores_kernel)
//   top_k:                            softmax(act[:, 1:]) * exp(comp)
//   cls without it:                   act[:, 1:] * exp(comp)
__global__ void batch_scores_kernel(const float* __restrict__ act, const float* __restrict__ comp, int N, BatchParams p, float* __restrict__ combined) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int K = p.K;
  const float* a = act + (long long)i * (K + 1);
  const float* cp = comp + (long long)i * K;
  float* out = combined + (long long)i * K;
  if (p.mode == SSNB_DET_CLS && !p.sbf) {
    for (int c = 0; c < K; ++c) out[c] = a[c + 1] * expf(cp[c]);
    return;
  }
  const int j0 = p.mode == SSNB_DET_TOPK ? 1 : 0;
  float m = a[j0];
  for (int j = j0 + 1; j <= K; ++j) m = fmaxf(m, a[j]);
  float sum = 0.f;
  for (int j = j0; j <= K; ++j) sum += expf(a[j] - m);
  for (int c = 0; c < K; ++c) out[c] = (expf(a[c + 1] - m) / sum) * expf(cp[c]);
}

// candidate i of video v is pair q = n_cand - 1 - (i - cand0): reversed, so that the stable sort puts equal scores larger
// index first.  q = p K + c (all, top_k) or p n_sel + j (cls, class cls_sel[v, j]); the value is the pair's global row * K + c,
// -1 (last key) for a selected class outside [0, K)
__global__ void candidates_kernel(const BatchDesc* __restrict__ desc, BatchParams p, int n_cand, const float* __restrict__ combined,
                                  const int32_t* __restrict__ cls_sel, uint32_t* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cand) return;
  const int v = video_at<&BatchDesc::cand0>(desc, p.V, i);
  const BatchDesc d = desc[v];
  const int q = d.n_cand - 1 - (i - d.cand0);
  int row, c;
  if (p.mode == SSNB_DET_CLS) {
    row = d.row0 + q / p.n_sel;
    c = cls_sel[(long long)v * p.n_sel + q % p.n_sel];
  } else {
    row = d.row0 + q / p.K;
    c = q % p.K;
  }
  if (c < 0 || c >= p.K) { keys[i] = 0xffffffffu; vals[i] = -1; return; }
  const int f = row * p.K + c;
  keys[i] = score_key(combined[f]);
  vals[i] = f;
}

// slot i of video v takes the (i - slot0)-th pair of the video's score order, keyed by its class (K: none)
__global__ void select_kernel(const BatchDesc* __restrict__ desc, BatchParams p, int n_slots, const int* __restrict__ sorted,
                              uint32_t* __restrict__ cls_key, int* __restrict__ vals, int32_t* __restrict__ sel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_slots) return;
  const BatchDesc d = desc[video_at<&BatchDesc::slot0>(desc, p.V, i)];
  const int f = sorted[d.cand0 + (i - d.slot0)];
  cls_key[i] = f >= 0 ? (uint32_t)(f % p.K) : (uint32_t)p.K;
  vals[i] = f;
  if (sel) sel[i] = f;
}

// run_begin / run_end [V, K] (zeroed before): the class runs of every video's class-sorted slots, relative to its slot0
__global__ void runs_kernel(const BatchDesc* __restrict__ desc, BatchParams p, int n_slots, const uint32_t* __restrict__ cls_key,
                            int* __restrict__ run_begin, int* __restrict__ run_end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_slots) return;
  const int v = video_at<&BatchDesc::slot0>(desc, p.V, i);
  const BatchDesc d = desc[v];
  const uint32_t c = cls_key[i];
  if (c >= (uint32_t)p.K) return;
  const int j = i - d.slot0;
  if (j == 0 || cls_key[i - 1] != c) run_begin[v * p.K + c] = j;
  if (j == d.n_slot - 1 || cls_key[i + 1] != c) run_end[v * p.K + c] = j + 1;
}

// one CTA per (video, class): the run's scores and boxes in ranking order, then the NMS / regression loop
__global__ void __launch_bounds__(kBatchNmsThreads) batch_nms_kernel(const BatchDesc* __restrict__ desc, BatchParams p, const int* __restrict__ run_begin,
                                                                      const int* __restrict__ run_end, const int* __restrict__ sorted,
                                                                      const float* __restrict__ combined, const float* __restrict__ props,
                                                                      const float* __restrict__ reg, double thresh, int regress, float* key, int* idx,
                                                                      float* t1, float* t2, unsigned char* alive, float* __restrict__ tmp,
                                                                      int32_t* __restrict__ counts) {
  __shared__ int n_kept;
  const int vc = blockIdx.x, v = vc / p.K, c = vc % p.K;
  const int rb = run_begin[vc], n = run_end[vc] - rb;
  if (n <= 0) { if (threadIdx.x == 0) counts[vc] = 0; return; }
  const long long b = (long long)desc[v].slot0 + rb;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int f = sorted[b + i], s = f / p.K;
    key[b + i] = combined[f]; idx[b + i] = s;
    t1[b + i] = props[2LL * s]; t2[b + i] = props[2LL * s + 1];
    alive[b + i] = 1;
  }
  __syncthreads();
  nms_regress_list(n, key + b, idx + b, t1 + b, t2 + b, alive + b, reg, 2LL * p.K, 2 * c, thresh, regress, tmp + b * 5, &n_kept);
  if (threadIdx.x == 0) counts[vc] = n_kept;
}

// one CTA per video: class c's survivors (at its run start in tmp) go to slot0 + counts of the classes before it
__global__ void compact_kernel(const BatchDesc* __restrict__ desc, BatchParams p, const int* __restrict__ run_begin, const int32_t* __restrict__ counts,
                               const float* __restrict__ tmp, float* __restrict__ dets) {
  const int v = blockIdx.x;
  const long long s0 = desc[v].slot0;
  long long o = s0;
  for (int c = 0; c < p.K; ++c) {
    const int n = counts[v * p.K + c];
    const float* src = tmp + (s0 + run_begin[v * p.K + c]) * 5;
    for (int e = threadIdx.x; e < 5 * n; e += blockDim.x) dets[o * 5 + e] = src[e];
    o += n;
  }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct BatchLayout {
  size_t desc, cand_begin, cand_end, slot_begin, slot_end, combined, keys0, keys1, vals0, vals1, ckey0, ckey1, cval0, cval1, run_begin,
      run_end, key, idx, t1, t2, alive, tmp, cub, total;
};

int class_bits(int K) { int b = 1; while ((1LL << b) <= K) ++b; return b; }   // keys 0..K

size_t batch_cub_bytes(int n_cand, int n_slots, int V, int K) {
  size_t a = 0, b = 0;
  cub::DoubleBuffer<uint32_t> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, a, k, v, n_cand, V, (const int*)nullptr, (const int*)nullptr, 0, 32);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b, k, v, n_slots, V, (const int*)nullptr, (const int*)nullptr, 0, class_bits(K));
  return a > b ? a : b;
}

BatchLayout batch_layout(int V, int K, long long N, long long n_cand, long long n_slots) {
  BatchLayout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.desc = take(sizeof(BatchDesc) * V);
  L.cand_begin = take(4LL * V); L.cand_end = take(4LL * V); L.slot_begin = take(4LL * V); L.slot_end = take(4LL * V);
  L.combined = take(4 * N * K);
  L.keys0 = take(4 * n_cand); L.keys1 = take(4 * n_cand); L.vals0 = take(4 * n_cand); L.vals1 = take(4 * n_cand);
  L.ckey0 = take(4 * n_slots); L.ckey1 = take(4 * n_slots); L.cval0 = take(4 * n_slots); L.cval1 = take(4 * n_slots);
  L.run_begin = take(4LL * V * K); L.run_end = take(4LL * V * K);
  L.key = take(4 * n_slots); L.idx = take(4 * n_slots); L.t1 = take(4 * n_slots); L.t2 = take(4 * n_slots); L.alive = take(n_slots);
  L.tmp = take(20 * n_slots);
  L.cub = take(std::max<size_t>(batch_cub_bytes((int)n_cand, (int)n_slots, V, K), 1));
  L.total = o;
  return L;
}

// host-side validation and sizes; "" when the arguments are accepted
struct BatchSizes { long long N, n_cand, n_slots; };
const char* batch_check(const ssnb_detect_batch_cfg* cfg, int K, const int64_t* offsets, int V, BatchSizes* z) {
  if (!cfg || !offsets || V < 1) return "NULL config / offsets or no video";
  if (K < 1) return "num_class must be >= 1";
  if (cfg->mode != SSNB_DET_ALL && cfg->mode != SSNB_DET_TOPK && cfg->mode != SSNB_DET_CLS) return "unknown mode";
  if (cfg->mode == SSNB_DET_TOPK && cfg->top_k < 1) return "top_k must be >= 1";
  if (cfg->mode == SSNB_DET_CLS && (cfg->n_sel < 1 || cfg->n_sel > K)) return "n_sel must be in 1..num_class";
  if (std::isnan(cfg->nms_thresh)) return "nms_thresh is NaN";
  if (offsets[0] != 0) return "offsets[0] must be 0";
  long long slots = 0;
  const long long per = cfg->mode == SSNB_DET_CLS ? cfg->n_sel : K;
  for (int v = 0; v < V; ++v) {
    if (offsets[v + 1] < offsets[v]) return "offsets must not decrease";
    const long long n = offsets[v + 1] - offsets[v];
    slots += cfg->mode == SSNB_DET_TOPK ? std::min<long long>(cfg->top_k, n * K) : n * per;
    if (offsets[v + 1] * (long long)K > INT_MAX) return "more than INT_MAX (proposal, class) pairs in one call: split the batch";
  }
  z->N = offsets[V]; z->n_cand = offsets[V] * per; z->n_slots = slots;
  return nullptr;
}

int blocks(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_detect_postprocess(const float* rel_props, const float* act_scores, const float* comp_scores, const float* reg_scores, int n_props,
                            int num_class, double nms_thresh, int regress, float* detections, int* counts, float* combined_ws, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  // act_scores == NULL: combined_ws already holds the [N, K] scores to rank by (plain class-wise temporal NMS)
  if (!rel_props || (act_scores && !comp_scores) || !reg_scores || !detections || !counts || !combined_ws || n_props < 0 || num_class <= 0) {
    set_thread_error("detect_postprocess: bad argument"); return SSNB_EINVAL; }
  if (n_props == 0) { if (cudaMemsetAsync(counts, 0, num_class * sizeof(int), s) != cudaSuccess) return SSNB_ECUDA; return SSNB_OK; }
  int P = 1;
  while (P < n_props) P <<= 1;
  if (P > 8192) { set_thread_error("detect_postprocess: at most 8192 proposals per video"); return SSNB_ENOSUPPORT; }
  if (act_scores) {
    combined_scores_kernel<<<(n_props + 127) / 128, 128, 0, s>>>(act_scores, comp_scores, n_props, num_class, combined_ws);
    SSNB_LAUNCH_CHECK("combined_scores_kernel");
  }
  const size_t smem = (size_t)P * 17;          // key, idx, t1, t2 (4 B each) + alive (1 B)
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !attr_set[dev]) {
    if (cudaFuncSetAttribute(nms_regress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 17) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("detect_postprocess: cannot raise the dynamic shared memory limit"); return SSNB_ECUDA; }
    attr_set[dev] = true;
  }
  nms_regress_kernel<<<num_class, 256, smem, s>>>(rel_props, combined_ws, reg_scores, n_props, num_class, P, nms_thresh, regress, detections, counts);
  SSNB_LAUNCH_CHECK("nms_regress_kernel");
  return SSNB_OK;
}


size_t ssnb_detect_batch_workspace_bytes(const ssnb_detect_batch_cfg* cfg, int num_class, const int64_t* offsets, int n_videos) {
  BatchSizes z;
  if (batch_check(cfg, num_class, offsets, n_videos, &z)) return 0;
  return batch_layout(n_videos, num_class, z.N, z.n_cand, z.n_slots).total;
}

int ssnb_detect_batch(const ssnb_detect_batch_cfg* cfg, const float* rel_props, const float* act, const float* comp, const float* reg,
                      int num_class, const int64_t* offsets, const int64_t* offsets_dev, int n_videos, const int32_t* cls_sel,
                      float* dets, int32_t* counts, float* combined, int32_t* sel, void* workspace, size_t workspace_bytes,
                      void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  BatchSizes z;
  if (const char* bad = batch_check(cfg, num_class, offsets, n_videos, &z)) {
    set_thread_error(std::string("detect_batch: ") + bad); return SSNB_EINVAL; }
  if (!rel_props || !act || !comp || !offsets_dev || !dets || !counts || !workspace || (cfg->mode == SSNB_DET_CLS && !cls_sel)) {
    set_thread_error("detect_batch: NULL input, output or workspace pointer (reg may be NULL; cls_sel is needed in cls mode)");
    return SSNB_EINVAL; }
  const int V = n_videos, K = num_class;
  const BatchLayout L = batch_layout(V, K, z.N, z.n_cand, z.n_slots);
  if (workspace_bytes < L.total) { set_thread_error("detect_batch: workspace too small (ssnb_detect_batch_workspace_bytes)"); return SSNB_EINVAL; }
  BatchParams p{V, K, cfg->mode, cfg->top_k, cfg->n_sel, cfg->softmax_before_filter != 0};
  char* ws = (char*)workspace;
  BatchDesc* desc = (BatchDesc*)(ws + L.desc);
  int* cand_begin = (int*)(ws + L.cand_begin);
  int* cand_end = (int*)(ws + L.cand_end);
  int* slot_begin = (int*)(ws + L.slot_begin);
  int* slot_end = (int*)(ws + L.slot_end);
  int* run_begin = (int*)(ws + L.run_begin);
  int* run_end = (int*)(ws + L.run_end);
  float* comb = combined ? combined : (float*)(ws + L.combined);
  const int n_cand = (int)z.n_cand, n_slots = (int)z.n_slots;

  batch_desc_kernel<<<1, kDescThreads, 0, s>>>(offsets_dev, p, desc, cand_begin, cand_end, slot_begin, slot_end);
  SSNB_LAUNCH_CHECK("batch_desc_kernel");
  if (cudaMemsetAsync(run_begin, 0, 4LL * V * K, s) != cudaSuccess || cudaMemsetAsync(run_end, 0, 4LL * V * K, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("detect_batch: memset failed"); return SSNB_ECUDA; }
  if (z.N > 0) {
    batch_scores_kernel<<<blocks(z.N, 128), 128, 0, s>>>(act, comp, (int)z.N, p, comb);
    SSNB_LAUNCH_CHECK("batch_scores_kernel");
  }
  if (n_slots > 0) {
    candidates_kernel<<<blocks(n_cand, 256), 256, 0, s>>>(desc, p, n_cand, comb, cls_sel, (uint32_t*)(ws + L.keys0), (int*)(ws + L.vals0));
    SSNB_LAUNCH_CHECK("candidates_kernel");
    cub::DoubleBuffer<uint32_t> kb((uint32_t*)(ws + L.keys0), (uint32_t*)(ws + L.keys1));
    cub::DoubleBuffer<int> vb((int*)(ws + L.vals0), (int*)(ws + L.vals1));
    size_t cub_bytes = batch_cub_bytes(n_cand, n_slots, V, K);
    if (cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, n_cand, V, (const int*)cand_begin, (const int*)cand_end, 0, 32,
                                                 s) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("detect_batch: score sort failed"); return SSNB_ECUDA; }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    select_kernel<<<blocks(n_slots, 256), 256, 0, s>>>(desc, p, n_slots, vb.Current(), (uint32_t*)(ws + L.ckey0), (int*)(ws + L.cval0), sel);
    SSNB_LAUNCH_CHECK("select_kernel");
    cub::DoubleBuffer<uint32_t> ckb((uint32_t*)(ws + L.ckey0), (uint32_t*)(ws + L.ckey1));
    cub::DoubleBuffer<int> cvb((int*)(ws + L.cval0), (int*)(ws + L.cval1));
    cub_bytes = batch_cub_bytes(n_cand, n_slots, V, K);
    if (cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, ckb, cvb, n_slots, V, (const int*)slot_begin, (const int*)slot_end, 0,
                                                 class_bits(K), s) != cudaSuccess) {
      cudaGetLastError(); set_thread_error("detect_batch: class sort failed"); return SSNB_ECUDA; }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    runs_kernel<<<blocks(n_slots, 256), 256, 0, s>>>(desc, p, n_slots, ckb.Current(), run_begin, run_end);
    SSNB_LAUNCH_CHECK("runs_kernel");
    float* tmp = (float*)(ws + L.tmp);
    batch_nms_kernel<<<V * K, kBatchNmsThreads, 0, s>>>(desc, p, run_begin, run_end, cvb.Current(), comb, rel_props, reg, cfg->nms_thresh,
                                                         cfg->regress != 0, (float*)(ws + L.key), (int*)(ws + L.idx), (float*)(ws + L.t1),
                                                         (float*)(ws + L.t2), (unsigned char*)(ws + L.alive), tmp, counts);
    SSNB_LAUNCH_CHECK("batch_nms_kernel");
    compact_kernel<<<V, 128, 0, s>>>(desc, p, run_begin, counts, tmp, dets);
    SSNB_LAUNCH_CHECK("compact_kernel");
  } else if (cudaMemsetAsync(counts, 0, 4LL * V * K, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("detect_batch: memset failed"); return SSNB_ECUDA;
  }
  return SSNB_OK;
}

}  // extern "C"
