// Detection post-processing on the GPU (SURVEY section 8 f3): what eval_detection_results.py:91-183 does per video with
// numpy -- combined scores softmax(act)[:, 1:] * exp(comp) (:104, ops/utils.py:38-40), class-wise temporal NMS
// (ops/utils.py:56-82) and location regression (:147-160) -- as two kernels: one thread per proposal row for the scores,
// one CTA per class for sort + greedy NMS + regression.  Semantics kept: scores sorted descending, a box survives when its
// IoU with every kept box is <= thresh, IoU = inter / (dur_i + dur_j - inter) with a possibly NEGATIVE inter (disjoint boxes
// are never suppressed) and the division carried out in double like numpy's `.astype(float)`.
#include <cfloat>

#include "../../include/ssnb.h"
#include "common.cuh"

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
  if (threadIdx.x == 0) n_kept = 0;
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    if (!alive[i]) continue;                                // uniform: written before the last barrier
    const float a1 = t1[i], a2 = t2[i], da = a2 - a1;
    if (threadIdx.x == 0) {
      const int s = idx[i], o = n_kept++;
      float* q = out + ((long long)c * N + o) * 5;
      const float loc = reg[((long long)s * K + c) * 2], dur = reg[((long long)s * K + c) * 2 + 1];
      float b1 = a1, b2 = a2;
      if (regress) {                                        // eval_detection_results.py:147-160 (fp32 like the numpy arrays)
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
  if (threadIdx.x == 0) count[c] = n_kept;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_detect_workspace_bytes(int n_props, int num_class) { return (size_t)(n_props > 0 ? n_props : 0) * (num_class > 0 ? num_class : 0) * sizeof(float); }

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

}  // extern "C"
