// BinaryClassifier's head and loss: classifier_fc (binary_model.py:231) + torch.nn.CrossEntropyLoss (mean, binary_train.py:135,
// :162) + every gradient, in two launches.  Deterministic: each output is formed by one thread (or one warp's fixed shuffle
// tree) in a fixed order, and no floating-point atomics are used, so two calls give bitwise equal results.
#include <cmath>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int CE_THREADS = 256;
constexpr int CE_JB = 8;              // classes per thread in the weight-gradient role

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// launch 1, one CTA per row i.  Logit j is one warp's lane-strided fmaf dot product + xor-shuffle tree + bias: the order of
// linear_fwd_kernel, so the logits equal the module path's (_HeadLinear) bit for bit.  Warp 0 then forms the row's
// log-sum-exp in double, the row loss lse - z[t] and d(mean loss)/d(logit) = (softmax - onehot) * loss_scale / n.
__global__ void __launch_bounds__(CE_THREADS) ce_rows_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                              const float* __restrict__ b, const int64_t* __restrict__ target,
                                                              int D, int K, double gscale, float* __restrict__ logits,
                                                              float* __restrict__ dlogit, double* __restrict__ rowloss) {
  extern __shared__ float z[];                    // [K]
  const long long i = blockIdx.x;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, nw = CE_THREADS / 32;
  const float* xr = x + i * D;
  for (int j = warp; j < K; j += nw) {
    const float* wr = w + (long long)j * D;
    float s = 0.f;
    for (int d = lane; d < D; d += 32) s = fmaf(xr[d], wr[d], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      const float v = s + b[j];
      z[j] = v;
      logits[i * K + j] = v;
    }
  }
  __syncthreads();
  if (warp != 0) return;
  float mx = -INFINITY;
  for (int j = lane; j < K; j += 32) mx = fmaxf(mx, z[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  double se = 0.0;
  for (int j = lane; j < K; j += 32) se += exp((double)z[j] - (double)mx);
  const double lse = (double)mx + log(warp_sum(se));
  const long long t = target[i];
  const bool valid = t >= 0 && t < K;             // never used as an index otherwise
  for (int j = lane; j < K; j += 32) {
    const double p = exp((double)z[j] - lse);
    dlogit[i * K + j] = valid ? (float)((p - (j == t ? 1.0 : 0.0)) * gscale) : 0.f;
  }
  if (lane == 0) rowloss[i] = valid ? lse - (double)z[t] : (double)NAN;
}

// launch 2, three roles by block index, all reading the dlogit table of launch 1 (double accumulators, rows / classes ascending):
//   [0, nw)        dW[j][d] = sum_i dlogit[i][j] * x[i][d]   (a thread owns one d and CE_JB classes)
//   [nw, nw + nx)  dx[i][d] = sum_j dlogit[i][j] * W[j][d]   (a thread owns one (i, d))
//   nw + nx        db[j]    = sum_i dlogit[i][j], and loss = sum_i rowloss[i] / n
__global__ void __launch_bounds__(CE_THREADS) ce_grads_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ dlogit, const double* __restrict__ rowloss,
                                                               int n, int D, int K, int nw, int nx, float* __restrict__ dx,
                                                               float* __restrict__ dw, float* __restrict__ db, float* __restrict__ loss) {
  const int blk = blockIdx.x;
  if (blk < nw) {
    const int dblocks = (D + CE_THREADS - 1) / CE_THREADS;
    const int j0 = (blk / dblocks) * CE_JB;
    const int d = (blk % dblocks) * CE_THREADS + threadIdx.x;
    if (d >= D) return;
    const int nj = min(CE_JB, K - j0);
    double acc[CE_JB];
#pragma unroll
    for (int q = 0; q < CE_JB; ++q) acc[q] = 0.0;
    for (int i = 0; i < n; ++i) {
      const double xv = (double)x[(long long)i * D + d];
      const float* dl = dlogit + (long long)i * K + j0;
#pragma unroll
      for (int q = 0; q < CE_JB; ++q)
        if (q < nj) acc[q] = fma((double)dl[q], xv, acc[q]);
    }
#pragma unroll
    for (int q = 0; q < CE_JB; ++q)
      if (q < nj) dw[(long long)(j0 + q) * D + d] = (float)acc[q];
    return;
  }
  if (blk < nw + nx) {
    const long long e = (long long)(blk - nw) * CE_THREADS + threadIdx.x;
    if (e >= (long long)n * D) return;
    const long long i = e / D;
    const int d = (int)(e % D);
    const float* dl = dlogit + i * K;
    double acc = 0.0;
    for (int j = 0; j < K; ++j) acc = fma((double)dl[j], (double)w[(long long)j * D + d], acc);
    dx[e] = (float)acc;
    return;
  }
  for (int j = threadIdx.x; j < K; j += CE_THREADS) {
    double acc = 0.0;
    for (int i = 0; i < n; ++i) acc += (double)dlogit[(long long)i * K + j];
    db[j] = (float)acc;
  }
  if (threadIdx.x < 32) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 32) s += rowloss[i];
    s = warp_sum(s);
    if (threadIdx.x == 0) loss[0] = (float)(s / (double)n);
  }
}

size_t ce_align(size_t v) { return (v + 255) / 256 * 256; }

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

size_t ssnb_classifier_ce_workspace_bytes(int n, int num_class) {
  if (n <= 0 || num_class <= 0) return 0;
  return ce_align((size_t)n * num_class * sizeof(float)) + ce_align((size_t)n * sizeof(double));
}

int ssnb_classifier_ce_fwd_bwd(const float* x, const float* w, const float* b, const int64_t* target, int n, int in_dim,
                               int num_class, float loss_scale, float* logits, float* loss, float* dx, float* dw, float* db,
                               void* workspace, void* stream) {
  if (!x || !w || !b || !target || !logits || !loss || !dx || !dw || !db || !workspace) {
    set_thread_error("classifier_ce: null argument"); return SSNB_EINVAL; }
  if (n < 1 || in_dim < 1 || num_class < 1 || num_class > 4096) {
    set_thread_error("classifier_ce: need n >= 1, in_dim >= 1 and 1 <= num_class <= 4096"); return SSNB_EINVAL; }
  const long long nw = (long long)((num_class + CE_JB - 1) / CE_JB) * ((in_dim + CE_THREADS - 1) / CE_THREADS);
  const long long nx = ((long long)n * in_dim + CE_THREADS - 1) / CE_THREADS;
  if (nw + nx + 1 > 0x7fffffffLL) { set_thread_error("classifier_ce: problem too large for one grid"); return SSNB_EINVAL; }
  cudaStream_t s = (cudaStream_t)stream;
  float* dlogit = (float*)workspace;
  double* rowloss = (double*)((char*)workspace + ce_align((size_t)n * num_class * sizeof(float)));
  ce_rows_kernel<<<(unsigned)n, CE_THREADS, (size_t)num_class * sizeof(float), s>>>(
      x, w, b, target, in_dim, num_class, (double)loss_scale / (double)n, logits, dlogit, rowloss);
  SSNB_LAUNCH_CHECK("ce_rows_kernel");
  ce_grads_kernel<<<(unsigned)(nw + nx + 1), CE_THREADS, 0, s>>>(x, w, dlogit, rowloss, n, in_dim, num_class, (int)nw, (int)nx,
                                                                dx, dw, db, loss);
  SSNB_LAUNCH_CHECK("ce_grads_kernel");
  return SSNB_OK;
}

}  // extern "C"
