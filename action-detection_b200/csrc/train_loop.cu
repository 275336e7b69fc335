// The rest of the training step between loss.backward() and optimizer.step() -- the gradient norm and clip of
// clip_grad_norm (torch 0.3) after the iter_size division -- and the loop's meters (loss and top-1 accuracy
// AverageMeters).  Reference: ssn_train.py:213-250,373-415; binary_train.py:170-197,288-321.  The clipped SGD step
// itself is heads.cu's sgd_groups_kernel<true>.
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int NORM_THREADS = 256;
constexpr int CLIP_THREADS = 256;
constexpr int CLIP_MAX_CTAS = 2048;
constexpr int METER_THREADS = 256;
constexpr int METER_MAX_ROWS = 65536;

struct Extras {
  int count;
  float* p[SSNB_MAX_EXTRA_GRADS];
  long long n[SSNB_MAX_EXTRA_GRADS];
};

Extras extras_of(const ssnb_extra_grads* e) {
  Extras x{};
  x.count = e ? e->count : 0;
  for (int i = 0; i < x.count; ++i) { x.p[i] = e->grad[i]; x.n[i] = (long long)e->numel[i]; }
  return x;
}

__device__ __forceinline__ double sq(float v) { const double d = (double)v; return d * d; }

// the sum of a block's per-thread values in a fixed order (warp butterflies, then the warps in index order): the result
// does not depend on timing
template <int THREADS>
__device__ double block_sum(double v) {
  __shared__ double s_warp[THREADS / 32];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < THREADS / 32; ++w) t += s_warp[w];
  return t;   // thread 0 only
}

// stage 1: every CTA of the fixed grid sums the squares of its grid-stride share of the flat buffer (times gm, the
// iter_size division) and of the extras in fp64
__global__ void __launch_bounds__(NORM_THREADS) grad_norm_partial_kernel(const float* __restrict__ g, long long n, float gm, Extras ex,
                                                                          double* __restrict__ partials) {
  const long long tid = (long long)blockIdx.x * NORM_THREADS + threadIdx.x;
  const long long stride = (long long)SSNB_GRAD_NORM_CTAS * NORM_THREADS;
  double acc = 0.0;
  long long head = 0;
  if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
    const long long n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (long long i = tid; i < n4; i += stride) {
      const float4 v = __ldg(g4 + i);
      acc += sq(v.x * gm); acc += sq(v.y * gm); acc += sq(v.z * gm); acc += sq(v.w * gm);
    }
    head = n4 << 2;
  }
  for (long long i = head + tid; i < n; i += stride) acc += sq(g[i] * gm);
  for (int e = 0; e < ex.count; ++e)
    for (long long i = tid; i < ex.n[e]; i += stride) acc += sq(ex.p[e][i]);
  const double t = block_sum<NORM_THREADS>(acc);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// stage 2: one CTA adds the partials in a fixed order
__global__ void __launch_bounds__(SSNB_GRAD_NORM_CTAS) grad_norm_final_kernel(const double* __restrict__ partials, float* __restrict__ norm) {
  const double t = block_sum<SSNB_GRAD_NORM_CTAS>(partials[threadIdx.x]);
  if (threadIdx.x == 0) *norm = (float)sqrt(t);
}

__global__ void __launch_bounds__(CLIP_THREADS) grad_clip_kernel(const float* __restrict__ norm, float max_norm, float* __restrict__ g,
                                                                  long long n, Extras ex) {
  const double c = (double)max_norm / ((double)*norm + 1e-6);
  if (!(c < 1.0)) return;
  const float cf = (float)c;
  const long long stride = (long long)gridDim.x * CLIP_THREADS;
  for (long long i = (long long)blockIdx.x * CLIP_THREADS + threadIdx.x; i < n; i += stride) g[i] *= cf;
  for (int e = 0; e < ex.count; ++e)
    for (long long i = (long long)blockIdx.x * CLIP_THREADS + threadIdx.x; i < ex.n[e]; i += stride) ex.p[e][i] *= cf;
}

// a beats b: higher, NaN above every number (torch.topk), and at equal scores the lower class index (caller order)
__device__ __forceinline__ bool beats(float a, int ia, float b, int ib) {
  if (isnan(a) || isnan(b)) return isnan(a) && (!isnan(b) || ia < ib);
  return a > b || (a == b && ia < ib);
}

// one CTA: a warp per activity row takes its top-1 class and its rank among the activity rows (even rank: fg, odd: bg);
// thread 0 then updates the meters in fp64 exactly as AverageMeter.update(val, n) does
__global__ void __launch_bounds__(METER_THREADS) train_meters_kernel(const float* __restrict__ scores, int rows, int cols,
                                                                      const long long* __restrict__ target,
                                                                      const long long* __restrict__ ptype, const float* __restrict__ losses,
                                                                      int n_losses, double loss_n, double* __restrict__ meters) {
  __shared__ unsigned s_cnt[4];    // activity rows, correct over all, fg, bg
  if (threadIdx.x < 4) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto is_act = [&](int r) { return ptype == nullptr || ptype[r] == 0 || ptype[r] == 2; };
  for (int r = warp; r < rows; r += METER_THREADS / 32) {
    if (!is_act(r)) continue;
    int rank = 0;
    for (int j = lane; j < r; j += 32) rank += is_act(j) ? 1 : 0;
    float best = 0.f;
    int bi = -1;
    for (int c = lane; c < cols; c += 32) {
      const float v = scores[(long long)r * cols + c];
      if (bi < 0 || beats(v, c, best, bi)) { best = v; bi = c; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      rank += __shfl_xor_sync(0xffffffffu, rank, o);
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || beats(ov, oi, best, bi))) { best = ov; bi = oi; }
    }
    if (lane == 0) {
      const unsigned ok = (long long)bi == target[r] ? 1u : 0u;
      atomicAdd(&s_cnt[0], 1u);
      atomicAdd(&s_cnt[1], ok);
      atomicAdd(&s_cnt[2 + (rank & 1)], ok);
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 0; i < n_losses; ++i) {
    meters[2 * i] += (double)losses[i] * loss_n;
    meters[2 * i + 1] += loss_n;
  }
  const unsigned m = s_cnt[0];
  const unsigned nn[3] = {m, m / 2, m / 2};
  for (int k = 0; k < 3; ++k) {
    if (nn[k] == 0) continue;
    // correct_k.float().sum(0).mul_(100.0 / batch_size): an fp32 product with the fp32 rounding of the Python double
    const float val = (float)s_cnt[1 + k] * (float)(100.0 / (double)nn[k]);
    double* mt = meters + 2 * (n_losses + k);
    mt[0] += (double)val * (double)nn[k];
    mt[1] += (double)nn[k];
  }
}

}  // namespace

int check_extra_grads(const ssnb_extra_grads* extra, const char* what) {
  if (!extra) return SSNB_OK;
  if (extra->count < 0 || extra->count > SSNB_MAX_EXTRA_GRADS) {
    set_thread_error(std::string(what) + ": 0..8 extra gradients"); return SSNB_EINVAL; }
  for (int i = 0; i < extra->count; ++i)
    if (extra->numel[i] < 0 || (extra->numel[i] > 0 && !extra->grad[i])) {
      set_thread_error(std::string(what) + ": extra gradient " + std::to_string(i) + " is NULL or has a negative size");
      return SSNB_EINVAL;
    }
  return SSNB_OK;
}

}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_grad_norm(const float* grad, size_t n, float grad_mult, const ssnb_extra_grads* extra, double* partials, float* norm,
                   void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!partials || !norm || (n > 0 && !grad)) { set_thread_error("grad_norm: null argument"); return SSNB_EINVAL; }
  if (int rc = check_extra_grads(extra, "grad_norm")) return rc;
  grad_norm_partial_kernel<<<SSNB_GRAD_NORM_CTAS, NORM_THREADS, 0, s>>>(grad, (long long)n, grad_mult, extras_of(extra), partials);
  SSNB_LAUNCH_CHECK("grad_norm_partial_kernel");
  grad_norm_final_kernel<<<1, SSNB_GRAD_NORM_CTAS, 0, s>>>(partials, norm);
  SSNB_LAUNCH_CHECK("grad_norm_final_kernel");
  return SSNB_OK;
}

int ssnb_grad_clip(const float* norm, float max_norm, float* grad, size_t n, const ssnb_extra_grads* extra, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!norm || (n > 0 && !grad) || !(max_norm >= 0.f)) { set_thread_error("grad_clip: null argument or max_norm not >= 0"); return SSNB_EINVAL; }
  if (int rc = check_extra_grads(extra, "grad_clip")) return rc;
  const Extras ex = extras_of(extra);
  long long most = (long long)n;
  for (int i = 0; i < ex.count; ++i) most = ex.n[i] > most ? ex.n[i] : most;
  if (most == 0) return SSNB_OK;
  const long long ctas = (most + CLIP_THREADS - 1) / CLIP_THREADS;
  grad_clip_kernel<<<(unsigned)(ctas < CLIP_MAX_CTAS ? ctas : CLIP_MAX_CTAS), CLIP_THREADS, 0, s>>>(norm, max_norm, grad, (long long)n, ex);
  SSNB_LAUNCH_CHECK("grad_clip_kernel");
  return SSNB_OK;
}

int ssnb_train_meters(const float* scores, int rows, int cols, const int64_t* target, const int64_t* prop_type,
                      const float* losses, int n_losses, double loss_n, double* meters, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (!scores || !target || !meters || (n_losses > 0 && !losses)) { set_thread_error("train_meters: null argument"); return SSNB_EINVAL; }
  if (rows < 1 || rows > METER_MAX_ROWS || cols < 1 || n_losses < 0 || n_losses > 8 || !(loss_n > 0.0)) {
    set_thread_error("train_meters: need 1..65536 rows, >= 1 column, 0..8 losses and loss_n > 0"); return SSNB_EINVAL; }
  train_meters_kernel<<<1, METER_THREADS, 0, s>>>(scores, rows, cols, (const long long*)target, (const long long*)prop_type, losses,
                                                   n_losses, loss_n, meters);
  SSNB_LAUNCH_CHECK("train_meters_kernel");
  return SSNB_OK;
}

}  // extern "C"
