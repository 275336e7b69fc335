// TAG bottom-up proposals on the GPU: what gen_bottom_up_proposals.py:116-142 (gen_prop) does per video with
// ops/sequence_funcs.py -- softmax of the merged score, Gaussian smoothing of the foreground column, labels at every
// threshold, the watershed-style box search at every tolerance, frame-inclusive temporal NMS, seconds -- for many ragged
// videos in one call, with no per-video launch and no host synchronisation.
//
//   softmax_column_kernel   one thread per tick: softmax(f_score)[:, cls+1] and the raw column f_score[:, cls+1]
//   smooth_label_kernel     one thread per tick: scipy's gaussian_filter (double, 'reflect', scipy's tap order) and the
//                           threshold bitmask of the tick
//   edges_kernel            one CTA per (video, threshold): the run starts `up`, ends `down` and cs = cumsum(1 - label) there
//   search_kernel           one CTA per (video, threshold): per tolerance, a max tree over signal[up] and a min tree over
//                           signal[down]; every forward / backward search is one O(log U) tree walk instead of the
//                           reference's O(U) scan, and writes its box to the slot the reference's loop order gives it
//   score_kernel            per box: sum(frm_scores[a:b]) left to right in fp32, as Python's sum over np.float32 does
//   cub segmented radix sort by descending score (stable: ties keep the search order; every NaN score ranks ahead of
//                           +inf, NaN-scored boxes in search order, as the reference's argsort()[::-1] puts NaN first)
//   nms_kernel              one CTA per video: drops identical copies (same start, end and score bits, adjacent after the
//                           sort), greedy NMS, seconds and the minimum-length filter
#include <cub/cub.cuh>

#include <cfloat>
#include <climits>
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "rank_key.cuh"

namespace ssnb {
namespace {

constexpr int kMaxThr = 32, kMaxTol = 32, kMaxRadius = 63;
constexpr int kEdgeThreads = 256, kSearchThreads = 256, kScoreThreads = 128, kScoreSplit = 4, kNmsThreads = 512;

struct VideoDesc {
  long long tick0;      // first row of the video in f_score
  long long slot0;      // first box slot: n_thr * n_tol * (tick0 + v)
  long long edge0;      // first edge entry: n_thr * (tick0 + v); threshold k's edges start (T + 1) * k later
  double duration;
  int T, pad_;
};

struct Params {
  int V, K, cls, n_thr, n_tol, radius;
  float thr[kMaxThr];             // thresholds rounded to fp32: numpy 2 compares an fp32 array with a Python float in fp32
  double tol[kMaxTol];
  double w[kMaxRadius + 1];       // Gaussian tap j (symmetric), scipy's normalised double weights
  double nms_thresh, minimum_len;
};

// the first video whose ticks contain tick i
__device__ __forceinline__ int video_of(const VideoDesc* d, int V, long long i) {
  int lo = 0, hi = V - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (d[mid].tick0 <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void softmax_column_kernel(const float* __restrict__ f, long long N, Params p, float* __restrict__ col, float* __restrict__ ss) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* r = f + i * p.K;
  float m = r[0];
  for (int k = 1; k < p.K; ++k) m = fmaxf(m, r[k]);
  float sum = 0.f;
  for (int k = 0; k < p.K; ++k) sum += expf(r[k] - m);
  col[i] = r[p.cls + 1];
  ss[i] = expf(r[p.cls + 1] - m) / sum;
}

// one thread per video: where its ticks, box slots and edge entries start
__global__ void desc_kernel(const int64_t* __restrict__ offsets, const double* __restrict__ durations, Params p, VideoDesc* __restrict__ desc) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= p.V) return;
  VideoDesc d;
  d.tick0 = offsets[v];
  d.T = (int)(offsets[v + 1] - offsets[v]);
  d.pad_ = 0;
  d.duration = durations[v];
  d.slot0 = (long long)p.n_thr * p.n_tol * (d.tick0 + v);
  d.edge0 = (long long)p.n_thr * (d.tick0 + v);
  desc[v] = d;
}

// scipy's 'reflect' (d c b a | a b c d | d c b a), periodic with period 2T for reaches longer than the video
__device__ __forceinline__ int reflect(int i, int T) {
  int m = i % (2 * T);
  if (m < 0) m += 2 * T;
  return m < T ? m : 2 * T - 1 - m;
}

// NI_Correlate1D's symmetric loop: w0 * x[i], then += (x[i-j] + x[i+j]) * w_j from j = radius down to 1, in double
// without contraction, rounded to fp32; radius 0 (sigma = 0) returns the softmax column unchanged
__global__ void smooth_label_kernel(const float* __restrict__ ss, const VideoDesc* __restrict__ desc, long long N, Params p,
                                    uint32_t* __restrict__ lab, float* __restrict__ smoothed) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const VideoDesc d = desc[video_of(desc, p.V, i)];
  const float* x = ss + d.tick0;
  const int t = (int)(i - d.tick0), T = d.T;
  double acc = __dmul_rn((double)x[t], p.w[0]);
  for (int j = p.radius; j > 0; --j)
    acc = __dadd_rn(acc, __dmul_rn(__dadd_rn((double)x[reflect(t - j, T)], (double)x[reflect(t + j, T)]), p.w[j]));
  const float v = __double2float_rn(acc);
  uint32_t bits = 0;
  for (int k = 0; k < p.n_thr; ++k) bits |= (v > p.thr[k] ? 1u : 0u) << k;
  lab[i] = bits;
  if (smoothed) smoothed[i] = v;
}

// diff = [label[0], label[1:] - label[:-1], -label[-1]]: up = rising edges, down = falling edges (length T + 1).
// cs at up[k]: background ticks before it; cs at down[k]: cs[down[k]], or cs[T-1] when down[k] == T.
__global__ void __launch_bounds__(kEdgeThreads) edges_kernel(const uint32_t* __restrict__ lab, const VideoDesc* __restrict__ desc, Params p,
                                                             int* __restrict__ up, int* __restrict__ down, int* __restrict__ csu,
                                                             int* __restrict__ csd, int* __restrict__ nruns) {
  using Scan = cub::BlockScan<int, kEdgeThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int v = blockIdx.x / p.n_thr, k = blockIdx.x % p.n_thr;
  const VideoDesc d = desc[v];
  const int T = d.T;
  const long long e0 = d.edge0 + (long long)(T + 1) * k;
  const uint32_t* L = lab + d.tick0;
  int n_up = 0, n_dn = 0, fg = 0;                  // running totals before this tile
  for (int base = 0; base <= T; base += kEdgeThreads) {
    const int i = base + threadIdx.x;
    const int cur = i < T ? (L[i] >> k) & 1 : 0, prev = (i > 0 && i <= T) ? (L[i - 1] >> k) & 1 : 0;
    const int is_up = cur & !prev, is_dn = !cur & prev;
    int x_up, x_dn, x_fg, t_up, t_dn, t_fg;
    Scan(tmp).ExclusiveSum(is_up, x_up, t_up);
    __syncthreads();
    Scan(tmp).ExclusiveSum(is_dn, x_dn, t_dn);
    __syncthreads();
    Scan(tmp).ExclusiveSum(cur, x_fg, t_fg);
    __syncthreads();
    const int fg_before = fg + x_fg;
    if (is_up) { up[e0 + n_up + x_up] = i; csu[e0 + n_up + x_up] = i - fg_before; }
    if (is_dn) { down[e0 + n_dn + x_dn] = i; csd[e0 + n_dn + x_dn] = i < T ? i + 1 - fg_before : T - fg_before; }
    n_up += t_up; n_dn += t_dn; fg += t_fg;
  }
  if (threadIdx.x == 0) nruns[blockIdx.x] = n_up;
}

// signal[i] = cs[i] - t*i in double, product and difference rounded separately (numpy's `cs - t * offset`)
__device__ __forceinline__ double signal(int cs, int i, double t) { return __dsub_rn((double)cs, __dmul_rn(t, (double)i)); }

__device__ __forceinline__ unsigned long long pack_box(int start, int end, int whole_prefix) {
  return (unsigned long long)(unsigned)start | ((unsigned long long)((unsigned)end | ((unsigned)whole_prefix << 31)) << 32);
}

// build_box_by_search (sequence_funcs.py:101-136) for one (video, threshold), every tolerance in turn.  Box slots:
// the video's box range, then 2 * n_tol * U per earlier threshold, then per tolerance the U forward boxes (x ascending)
// and the U backward boxes (x descending) -- the order the reference appends them in.
__global__ void __launch_bounds__(kSearchThreads) search_kernel(const VideoDesc* __restrict__ desc, Params p, const int* __restrict__ up,
                                                                const int* __restrict__ down, const int* __restrict__ csu,
                                                                const int* __restrict__ csd, const int* __restrict__ nruns,
                                                                double* __restrict__ trees, unsigned long long* __restrict__ vals,
                                                                int* __restrict__ seg_begin, int* __restrict__ seg_end, int* __restrict__ raw_counts) {
  const int v = blockIdx.x / p.n_thr, k = blockIdx.x % p.n_thr;
  const VideoDesc d = desc[v];
  const int T = d.T;
  long long before = 0, total = 0;
  for (int q = 0; q < p.n_thr; ++q) {
    const int u = nruns[v * p.n_thr + q];
    if (q < k) before += u;
    total += u;
  }
  if (k == 0 && threadIdx.x == 0) {
    seg_begin[v] = (int)d.slot0;
    seg_end[v] = (int)(d.slot0 + 2 * p.n_tol * total);
    if (raw_counts) raw_counts[v] = (int)(2 * p.n_tol * total);
  }
  const int U = nruns[v * p.n_thr + k];
  if (U == 0) return;
  const long long e0 = d.edge0 + (long long)(T + 1) * k;
  const int* UP = up + e0;
  const int* DN = down + e0;
  const int* CU = csu + e0;
  const int* CD = csd + e0;
  int P = 1;
  while (P < U) P <<= 1;
  double* tmax = trees + 4 * e0;                  // [2P] each, root at 1, leaves at P + y (P <= T + 1)
  double* tmin = tmax + 2 * (long long)(T + 1);
  unsigned long long* out = vals + d.slot0 + 2 * p.n_tol * before;
  for (int ti = 0; ti < p.n_tol; ++ti) {
    const double t = p.tol[ti];
    for (int y = threadIdx.x; y < P; y += blockDim.x) {
      tmax[P + y] = y < U ? signal(CU[y], UP[y], t) : -INFINITY;
      tmin[P + y] = y < U ? (DN[y] < T ? signal(CD[y], DN[y], t) : __dsub_rn(signal(CD[y], T - 1, t), t)) : INFINITY;
    }
    __syncthreads();
    for (int lvl = P >> 1; lvl >= 1; lvl >>= 1) {
      for (int n = lvl + threadIdx.x; n < 2 * lvl; n += blockDim.x) {
        tmax[n] = fmax(tmax[2 * n], tmax[2 * n + 1]);
        tmin[n] = fmin(tmin[2 * n], tmin[2 * n + 1]);
      }
      __syncthreads();
    }
    unsigned long long* o = out + 2LL * U * ti;
    for (int x = threadIdx.x; x < U; x += blockDim.x) {
      // forward: the first y > x with signal[up[y]] > signal[up[x]]
      const double s = tmax[P + x];
      int n = P + x;
      bool hit = false;
      while (n > 1) {
        if (!(n & 1) && tmax[n + 1] > s) { n += 1; hit = true; break; }
        n >>= 1;
      }
      if (hit)
        while (n < P) { n = 2 * n; if (!(tmax[n] > s)) n += 1; }
      o[x] = pack_box(UP[x], (hit ? DN[n - P - 1] : DN[U - 1]) + 1, 0);
      // backward: the last y < x with signal[down[y]] < s_x
      const double sb = tmin[P + x];
      n = P + x;
      hit = false;
      while (n > 1) {
        if ((n & 1) && tmin[n - 1] < sb) { n -= 1; hit = true; break; }
        n >>= 1;
      }
      if (hit)
        while (n < P) { n = 2 * n + 1; if (!(tmin[n] < sb)) n -= 1; }
      // no such y: (up[0], down[x]+1) scored over [0, down[x]+2) (sequence_funcs.py:134)
      o[U + (U - 1 - x)] = hit ? pack_box(UP[n - P + 1], DN[x] + 1, 0) : pack_box(UP[0], DN[x] + 1, 1);
    }
    __syncthreads();
  }
}

// score_key / key_score (rank_key.cuh): NaN-scored boxes rank first, as in the reference's argsort()[::-1], and among
// themselves keep the search order

__global__ void __launch_bounds__(kScoreThreads) score_kernel(const float* __restrict__ col, const VideoDesc* __restrict__ desc,
                                                              const int* __restrict__ seg_end, unsigned long long* __restrict__ vals,
                                                              uint32_t* __restrict__ keys, int* __restrict__ raw_frames, float* __restrict__ raw_scores) {
  const int v = blockIdx.x / kScoreSplit, part = blockIdx.x % kScoreSplit;
  const VideoDesc d = desc[v];
  const long long n = seg_end[v] - d.slot0;
  const float* x = col + d.tick0;
  for (long long b = (long long)part * blockDim.x + threadIdx.x; b < n; b += (long long)kScoreSplit * blockDim.x) {
    const long long slot = d.slot0 + b;
    const unsigned long long val = vals[slot];
    const int start = (int)(val & 0xffffffffu), end = (int)((val >> 32) & 0x7fffffffu);
    const bool whole_prefix = (val >> 63) != 0;
    const int a = whole_prefix ? 0 : start, e = min(whole_prefix ? end + 1 : end, d.T);
    float sum = 0.f;                              // Python's sum: 0 + x[a] + x[a+1] + ... in fp32, left to right
    for (int i = a; i < e; ++i) sum += x[i];
    keys[slot] = score_key(sum);
    vals[slot] = val & ~(1ull << 63);
    if (raw_frames) { raw_frames[2 * slot] = start; raw_frames[2 * slot + 1] = end; }
    if (raw_scores) raw_scores[slot] = sum;
  }
}

// temporal_nms_fallback (sequence_funcs.py:71-97) over one video's sorted boxes, then gen_prop's seconds and length filter
// (:138-141).  Identical copies (same start, end and score) are adjacent after the stable sort unless a distinct box with
// the same score sits between them; they are dropped first, which only saves work: with thresh < 1 the first copy
// suppresses the others (IoU = 1).
__global__ void __launch_bounds__(kNmsThreads) nms_kernel(const VideoDesc* __restrict__ desc, Params p, const int* __restrict__ seg_end,
                                                          const uint32_t* __restrict__ keys, const unsigned long long* __restrict__ vals,
                                                          uint32_t* __restrict__ ukeys, int2* __restrict__ ubox, unsigned char* __restrict__ alive,
                                                          int* __restrict__ frames, float* __restrict__ scores, double* __restrict__ seconds,
                                                          int* __restrict__ counts) {
  using Scan = cub::BlockScan<int, kNmsThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_out;
  const int v = blockIdx.x;
  const VideoDesc d = desc[v];
  const long long n = seg_end[v] - d.slot0;
  const uint32_t* K = keys + d.slot0;
  const unsigned long long* B = vals + d.slot0;
  uint32_t* UK = ukeys + d.slot0;
  int2* UB = ubox + d.slot0;
  unsigned char* A = alive + d.slot0;
  int D = 0;
  for (long long base = 0; base < n; base += kNmsThreads) {
    const long long i = base + threadIdx.x;
    const int keep = i < n && (i == 0 || K[i] != K[i - 1] || B[i] != B[i - 1]);
    int x, tot;
    Scan(tmp).ExclusiveSum(keep, x, tot);
    __syncthreads();
    if (keep) {
      const unsigned long long b = B[i];
      UK[D + x] = K[i];
      UB[D + x] = make_int2((int)(b & 0xffffffffu), (int)(b >> 32));
      A[D + x] = 1;
    }
    D += tot;
  }
  if (threadIdx.x == 0) s_out = 0;
  __syncthreads();
  const double T = (double)d.T;
  for (int i = 0; i < D; ++i) {
    if (!A[i]) continue;                          // uniform: its last write happened before the last barrier
    const int2 bi = UB[i];
    if (threadIdx.x == 0) {
      const double t0 = __dmul_rn(__ddiv_rn((double)bi.x, T), d.duration), t1 = __dmul_rn(__ddiv_rn((double)bi.y, T), d.duration);
      if (__dsub_rn(t1, t0) > p.minimum_len) {
        const long long o = d.slot0 + s_out++;
        frames[2 * o] = bi.x; frames[2 * o + 1] = bi.y;
        scores[o] = key_score(UK[i]);
        seconds[2 * o] = t0; seconds[2 * o + 1] = t1;
      }
    }
    const long long di = (long long)bi.y - bi.x + 1;
    for (int j = i + 1 + threadIdx.x; j < D; j += blockDim.x) {
      if (!A[j]) continue;
      const int2 bj = UB[j];
      const long long inter = (long long)min(bi.y, bj.y) - max(bi.x, bj.x) + 1;
      if (inter <= 0) continue;                   // IoU <= 0 <= thresh: never suppressed
      const double iou = __ddiv_rn((double)inter, (double)(di + ((long long)bj.y - bj.x + 1) - inter));
      if (!(iou <= p.nms_thresh)) A[j] = 0;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[v] = s_out;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace regions, in order
struct Layout {
  size_t desc, col, ss, lab, nruns, seg_begin, seg_end, up, down, csu, csd, trees, keys0, keys1, vals0, vals1, alive, cub, total;
};

size_t cub_sort_bytes(long long n_slots, int V) {
  size_t bytes = 0;
  cub::DoubleBuffer<uint32_t> k(nullptr, nullptr);
  cub::DoubleBuffer<unsigned long long> v(nullptr, nullptr);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, bytes, k, v, (int)n_slots, V, (const int*)nullptr, (const int*)nullptr, 0, 32);
  return bytes;
}

Layout layout(int V, long long N, int n_thr, int n_tol) {
  const long long S = N + V, slots = (long long)n_thr * n_tol * S, edges = (long long)n_thr * S;
  Layout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
  L.desc = take(sizeof(VideoDesc) * V);
  L.col = take(4 * N); L.ss = take(4 * N); L.lab = take(4 * N);
  L.nruns = take(4LL * V * n_thr); L.seg_begin = take(4LL * V); L.seg_end = take(4LL * V);
  L.up = take(4 * edges); L.down = take(4 * edges); L.csu = take(4 * edges); L.csd = take(4 * edges);
  L.trees = take(8 * 4 * edges);
  L.keys0 = take(4 * slots); L.keys1 = take(4 * slots); L.vals0 = take(8 * slots); L.vals1 = take(8 * slots);
  L.alive = take(slots);
  L.cub = take(cub_sort_bytes(slots, V) > 0 ? cub_sort_bytes(slots, V) : 1);   // 256 B: the sort needs none with DoubleBuffers
  L.total = o;
  return L;
}

// numpy's float64 sum of n <= 128 values: eight interleaved partial sums combined pairwise, then the remainder
double numpy_sum(const double* a, int n) {
  if (n < 8) { double r = 0.; for (int i = 0; i < n; ++i) r += a[i]; return r; }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] += a[i + j];
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += a[i];
  return res;
}

int fail(const char* msg) { set_thread_error(std::string("tag_proposals: ") + msg); return SSNB_EINVAL; }

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_tag_proposals_workspace_bytes(int n_videos, int64_t total_ticks, int n_thresholds, int n_tolerances) {
  if (n_videos < 0 || total_ticks < 0 || n_thresholds < 1 || n_thresholds > kMaxThr || n_tolerances < 1 || n_tolerances > kMaxTol) return 0;
  if ((long long)n_thresholds * n_tolerances * (total_ticks + n_videos) > INT_MAX) return 0;
  return layout(n_videos, total_ticks, n_thresholds, n_tolerances).total;
}

int ssnb_tag_proposals(const ssnb_tag_proposals_cfg* cfg, const float* f_score, int num_cols, const int64_t* offsets,
                       const int64_t* offsets_dev, int n_videos, const double* durations_dev, int32_t* frames, float* scores, double* seconds, int32_t* counts, float* smoothed,
                       uint32_t* labels, int32_t* raw_frames, float* raw_scores, int32_t* raw_counts, void* workspace,
                       size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!cfg || !offsets || n_videos < 0) return fail("NULL config / offsets or n_videos < 0");
  if (n_videos == 0) return SSNB_OK;
  const int V = n_videos, n_thr = cfg->n_thresholds, n_tol = cfg->n_tolerances;
  if (n_thr < 1 || n_thr > kMaxThr || !cfg->thresholds) return fail("1..32 thresholds");
  if (n_tol < 1 || n_tol > kMaxTol || !cfg->tolerances) return fail("1..32 tolerances");
  if (cfg->cls < 0 || num_cols <= cfg->cls + 1) return fail("the score needs more than cls + 1 columns");
  if (!(cfg->nms_thresh >= 0.0 && cfg->nms_thresh < 1.0)) return fail("nms_thresh outside [0, 1)");
  if (std::isnan(cfg->minimum_len)) return fail("minimum_len is NaN");
  if (!(cfg->sigma >= 0.0) || !std::isfinite(cfg->sigma)) return fail("sigma must be finite and >= 0 (0: no smoothing)");
  const int radius = cfg->sigma > 1e-15 ? (int)(4.0 * cfg->sigma + 0.5) : 0;   // scipy skips sigma <= 1e-15 (truncate 4.0)
  if (radius > kMaxRadius) return fail("sigma too large (Gaussian radius above 63)");
  if (offsets[0] != 0) return fail("offsets[0] must be 0");
  for (int v = 0; v < V; ++v)
    if (offsets[v + 1] <= offsets[v] || offsets[v + 1] - offsets[v] > INT_MAX - 2) return fail("offsets must increase strictly (every video needs >= 1 tick)");
  const long long N = offsets[V];
  if ((long long)n_thr * n_tol * (N + V) > INT_MAX) return fail("too many box slots in one call: split the batch");
  if (!f_score || !offsets_dev || !durations_dev || !frames || !scores || !seconds || !counts || !workspace)
    return fail("NULL score, device offsets / durations, output or workspace pointer");
  const Layout L = layout(V, N, n_thr, n_tol);
  if (workspace_bytes < L.total) return fail("workspace too small (ssnb_tag_proposals_workspace_bytes)");

  Params p{};
  p.V = V; p.K = num_cols; p.cls = cfg->cls; p.n_thr = n_thr; p.n_tol = n_tol; p.radius = radius;
  for (int k = 0; k < n_thr; ++k) {
    if (std::isnan(cfg->thresholds[k])) return fail("NaN threshold");
    p.thr[k] = (float)cfg->thresholds[k];
  }
  for (int k = 0; k < n_tol; ++k) {
    if (!std::isfinite(cfg->tolerances[k])) return fail("non-finite tolerance");
    p.tol[k] = cfg->tolerances[k];
  }
  // scipy.ndimage._filters._gaussian_kernel1d: exp(-0.5 / sigma^2 * x^2) over x = -radius..radius, over its numpy sum
  double phi[2 * kMaxRadius + 1];
  const double c = radius ? -0.5 / (cfg->sigma * cfg->sigma) : 0.0;
  for (int x = -radius; x <= radius; ++x) phi[x + radius] = std::exp(c * (double)((long long)x * x));
  const double norm = numpy_sum(phi, 2 * radius + 1);
  for (int j = 0; j <= radius; ++j) p.w[j] = phi[radius + j] / norm;
  p.nms_thresh = cfg->nms_thresh; p.minimum_len = cfg->minimum_len;

  char* ws = (char*)workspace;
  VideoDesc* ddesc = (VideoDesc*)(ws + L.desc);
  float* col = (float*)(ws + L.col);
  float* ss = (float*)(ws + L.ss);
  uint32_t* lab = (uint32_t*)(ws + L.lab);
  int* nruns = (int*)(ws + L.nruns);
  int* seg_begin = (int*)(ws + L.seg_begin);
  int* seg_end = (int*)(ws + L.seg_end);
  uint32_t* keys0 = (uint32_t*)(ws + L.keys0);
  uint32_t* keys1 = (uint32_t*)(ws + L.keys1);
  unsigned long long* vals0 = (unsigned long long*)(ws + L.vals0);
  unsigned long long* vals1 = (unsigned long long*)(ws + L.vals1);
  desc_kernel<<<(V + 127) / 128, 128, 0, s>>>(offsets_dev, durations_dev, p, ddesc);
  SSNB_LAUNCH_CHECK("desc_kernel");

  const int tick_blocks = (int)((N + 255) / 256);
  softmax_column_kernel<<<tick_blocks, 256, 0, s>>>(f_score, N, p, col, ss);
  SSNB_LAUNCH_CHECK("softmax_column_kernel");
  smooth_label_kernel<<<tick_blocks, 256, 0, s>>>(ss, ddesc, N, p, labels ? labels : lab, smoothed);
  SSNB_LAUNCH_CHECK("smooth_label_kernel");
  const uint32_t* lab_in = labels ? labels : lab;
  int* up = (int*)(ws + L.up);
  int* down = (int*)(ws + L.down);
  int* csu = (int*)(ws + L.csu);
  int* csd = (int*)(ws + L.csd);
  edges_kernel<<<V * n_thr, kEdgeThreads, 0, s>>>(lab_in, ddesc, p, up, down, csu, csd, nruns);
  SSNB_LAUNCH_CHECK("edges_kernel");
  search_kernel<<<V * n_thr, kSearchThreads, 0, s>>>(ddesc, p, up, down, csu, csd, nruns, (double*)(ws + L.trees), vals0, seg_begin,
                                                     seg_end, raw_counts);
  SSNB_LAUNCH_CHECK("search_kernel");
  score_kernel<<<V * kScoreSplit, kScoreThreads, 0, s>>>(col, ddesc, seg_end, vals0, keys0, raw_frames, raw_scores);
  SSNB_LAUNCH_CHECK("score_kernel");

  const long long slots = (long long)n_thr * n_tol * (N + V);
  cub::DoubleBuffer<uint32_t> kb(keys0, keys1);
  cub::DoubleBuffer<unsigned long long> vb(vals0, vals1);
  size_t cub_bytes = cub_sort_bytes(slots, V);
  if (cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kb, vb, (int)slots, V, (const int*)seg_begin,
                                               (const int*)seg_end, 0, 32, s) != cudaSuccess) {
    cudaGetLastError(); set_thread_error("tag_proposals: segmented sort failed"); return SSNB_ECUDA; }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  // the buffers the sort did not end in are free again: deduplicated keys and boxes go there
  uint32_t* ukeys = kb.Alternate();
  int2* ubox = (int2*)vb.Alternate();
  nms_kernel<<<V, kNmsThreads, 0, s>>>(ddesc, p, seg_end, kb.Current(), vb.Current(), ukeys, ubox, (unsigned char*)(ws + L.alive), frames,
                                       scores, seconds, counts);
  SSNB_LAUNCH_CHECK("nms_kernel");
  return SSNB_OK;
}

}  // extern "C"
