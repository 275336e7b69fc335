// Training-mode BatchNorm2d for the FIRST normalisation layer (bn_mode='partial': ssn_models.py:95-105,156-174 freezes every
// BatchNorm2d except conv1's), fp32 NHWC, fused with the ReLU that follows it:
//   forward   mu = mean_c(z), var = biased variance_c(z) over all F*H*W rows;  y = relu(gamma * (z - mu) / sqrt(var + eps) + beta)
//             running_mean / running_var <- (1 - m) * running + m * (mu | unbiased var)      (torch.nn.BatchNorm2d, momentum m)
//   backward  g = dy * (y > 0);  dbeta = sum g;  dgamma = sum g * xhat;
//             dz = gamma * invstd * (g - dbeta / M - xhat * dgamma / M)
// Column reductions are two-stage and deterministic: per-CTA partials, then one CTA reduces them in CTA order.  The
// variance is a true second pass over (z - mu) (sum of squares minus squared mean cancels badly for +-128 inputs).
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int BN_THREADS = 256;
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// MODE 0: sum z                      -> partial[cta][C]
// MODE 1: sum (z - mu)^2             -> partial[cta][C]            (stat[0..C) = mu)
// MODE 2: sum g, sum g * xhat        -> partial[cta][2C]           (stat = mu | invstd), g = dy * (y > 0)
template <int MODE>
__global__ void __launch_bounds__(BN_THREADS) bn_colreduce_kernel(const float* __restrict__ z, int zpitch, int zcoff, const float* __restrict__ dy,
                                                                  int dpitch, int dcoff, const float* __restrict__ y, int ypitch, int ycoff,
                                                                  const float* __restrict__ stat, long long rows, int C, long long rows_per_cta,
                                                                  float* __restrict__ partial) {
  extern __shared__ float red[];                  // [lanes][NOUT * C]
  constexpr int NOUT = MODE == 2 ? 2 : 1;
  const int G = C / 4, lanes = BN_THREADS / G;
  const int g = threadIdx.x % G, rl = threadIdx.x / G;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = (r0 + rows_per_cta < rows) ? r0 + rows_per_cta : rows;
  float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
  float mu[4] = {0.f, 0.f, 0.f, 0.f}, is[4] = {1.f, 1.f, 1.f, 1.f};
  if (MODE >= 1) { const float4 m = ld4(stat + g * 4); mu[0] = m.x; mu[1] = m.y; mu[2] = m.z; mu[3] = m.w; }
  if (MODE == 2) { const float4 s = ld4(stat + C + g * 4); is[0] = s.x; is[1] = s.y; is[2] = s.z; is[3] = s.w; }
  if (rl < lanes) {
    for (long long r = r0 + rl; r < r1; r += lanes) {
      const float4 zv = ld4(z + r * zpitch + zcoff + g * 4);
      const float zz[4] = {zv.x, zv.y, zv.z, zv.w};
      if (MODE == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) a0[j] += zz[j];
      } else if (MODE == 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float d = zz[j] - mu[j]; a0[j] = fmaf(d, d, a0[j]); }
      } else {
        const float4 dv = ld4(dy + r * dpitch + dcoff + g * 4), yv = ld4(y + r * ypitch + ycoff + g * 4);
        const float dd[4] = {dv.x, dv.y, dv.z, dv.w}, yy[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float gg = yy[j] > 0.f ? dd[j] : 0.f;
          a0[j] += gg;
          a1[j] = fmaf(gg, (zz[j] - mu[j]) * is[j], a1[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      red[rl * NOUT * C + g * 4 + j] = a0[j];
      if (NOUT == 2) red[rl * NOUT * C + C + g * 4 + j] = a1[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < NOUT * C; c += BN_THREADS) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += red[l * NOUT * C + c];
    partial[(long long)blockIdx.x * NOUT * C + c] = s;
  }
}

// stage 2 of the statistics: reduce the per-CTA partials in CTA order (double accumulation: up to ~600 partials of ~1e4 rows)
//   what = 0: mean          -> stat[c] = sum / M
//   what = 1: variance      -> stat[C + c] = 1 / sqrt(var + eps); running stats updated
__global__ void bn_stat_finish_kernel(const float* __restrict__ partial, int nparts, int C, double M, int what, float eps, float momentum,
                                      float* __restrict__ stat, float* __restrict__ running_mean, float* __restrict__ running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
  for (int i = 0; i < nparts; ++i) s += (double)partial[(long long)i * C + c];
  if (what == 0) {
    stat[c] = (float)(s / M);
  } else {
    const float var = (float)(s / M);
    stat[C + c] = 1.0f / sqrtf(var + eps);
    if (running_mean) running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * stat[c];
    if (running_var) running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)(s / (M > 1.0 ? M - 1.0 : 1.0));
  }
}

// backward stage 2: dbeta = sum g, dgamma = sum g * xhat; also kept in stat[2C..4C) for the apply pass
__global__ void bn_grad_finish_kernel(const float* __restrict__ partial, int nparts, int C, float* __restrict__ stat, float* __restrict__ dgamma,
                                      float* __restrict__ dbeta, const float* __restrict__ unscale, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sb = 0.0, sg = 0.0;
  for (int i = 0; i < nparts; ++i) { sb += (double)partial[(long long)i * 2 * C + c]; sg += (double)partial[(long long)i * 2 * C + C + c]; }
  stat[2 * C + c] = (float)sb;          // the apply pass works on the scaled gradient, like every kernel between entry and exit
  stat[3 * C + c] = (float)sg;
  const double u = unscale ? (double)__ldg(unscale) : 1.0;
  if (dbeta) dbeta[c] = (accumulate ? dbeta[c] : 0.f) + (float)(sb * u);
  if (dgamma) dgamma[c] = (accumulate ? dgamma[c] : 0.f) + (float)(sg * u);
}

// y = relu(gamma * xhat + beta)  (+ the value's fp16 hi / lo operand planes in EXACT_TC)
__global__ void bn_apply_relu_kernel(const float* __restrict__ z, int zpitch, int zcoff, const float* __restrict__ stat, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, long long rows, int C, float* __restrict__ y, int ypitch, int ycoff,
                                     __half* __restrict__ hi, long long lo_off) {
  const int G = C / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * G) return;
  const int g = (int)(i % G);
  const long long r = i / G;
  const float4 zv = ld4(z + r * zpitch + zcoff + g * 4), m = ld4(stat + g * 4), s = ld4(stat + C + g * 4), ga = ld4(gamma + g * 4), be = ld4(beta + g * 4);
  float4 o;
  o.x = relu((zv.x - m.x) * s.x * ga.x + be.x); o.y = relu((zv.y - m.y) * s.y * ga.y + be.y);
  o.z = relu((zv.z - m.z) * s.z * ga.z + be.z); o.w = relu((zv.w - m.w) * s.w * ga.w + be.w);
  *reinterpret_cast<float4*>(y + r * ypitch + ycoff + g * 4) = o;
  if (hi) store_planes4(hi + r * ypitch + ycoff + g * 4, lo_off, o);
}

// dz = gamma * invstd * (g - dbeta / M - xhat * dgamma / M)   (+ planes of dz * scale in EXACT_TC)
__global__ void bn_bwd_apply_kernel(const float* __restrict__ z, int zpitch, int zcoff, const float* __restrict__ dy, int dpitch, int dcoff,
                                    const float* __restrict__ y, int ypitch, int ycoff, const float* __restrict__ stat, const float* __restrict__ gamma,
                                    long long rows, int C, float inv_m, float* __restrict__ dz, int zgpitch, int zgcoff, __half* __restrict__ hi,
                                    long long lo_off, float scale, int* __restrict__ flag) {
  const int G = C / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * G) return;
  const int g = (int)(i % G);
  const long long r = i / G;
  const float4 zv = ld4(z + r * zpitch + zcoff + g * 4), dv = ld4(dy + r * dpitch + dcoff + g * 4), yv = ld4(y + r * ypitch + ycoff + g * 4);
  const float4 m = ld4(stat + g * 4), s = ld4(stat + C + g * 4), sb = ld4(stat + 2 * C + g * 4), sg = ld4(stat + 3 * C + g * 4), ga = ld4(gamma + g * 4);
  const float zz[4] = {zv.x, zv.y, zv.z, zv.w}, dd[4] = {dv.x, dv.y, dv.z, dv.w}, yy[4] = {yv.x, yv.y, yv.z, yv.w};
  const float mm[4] = {m.x, m.y, m.z, m.w}, ss[4] = {s.x, s.y, s.z, s.w}, bb[4] = {sb.x, sb.y, sb.z, sb.w}, gg[4] = {sg.x, sg.y, sg.z, sg.w};
  const float gm[4] = {ga.x, ga.y, ga.z, ga.w};
  float o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float gr = yy[j] > 0.f ? dd[j] : 0.f;
    const float xh = (zz[j] - mm[j]) * ss[j];
    o[j] = gm[j] * ss[j] * (gr - bb[j] * inv_m - xh * gg[j] * inv_m);
  }
  const float4 ov = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(dz + r * zgpitch + zgcoff + g * 4) = ov;
  if (hi) {
    const float4 sv = make_float4(o[0] * scale, o[1] * scale, o[2] * scale, o[3] * scale);
    const float am = fmaxf(fmaxf(fabsf(sv.x), fabsf(sv.y)), fmaxf(fabsf(sv.z), fabsf(sv.w)));
    if (flag && !(am <= HALF_MAX)) *flag = 1;
    store_planes4(hi + r * zgpitch + zgcoff + g * 4, lo_off, sv);
  }
}

inline int bn_ctas(long long rows, int max_ctas, long long* rpc) {
  int ctas = (int)((rows + 1023) / 1024);
  if (ctas > 592) ctas = 592;
  if (ctas > max_ctas) ctas = max_ctas;
  if (ctas < 1) ctas = 1;
  *rpc = (rows + ctas - 1) / ctas;
  return (int)((rows + *rpc - 1) / *rpc);
}

}  // namespace

// stat: 4*C floats (mean | invstd | sum g | sum g*xhat); partial: max_ctas * 2 * C floats
int launch_bn_train_fwd(View z, View y, View y_planes, int F, const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                        float* running_var, float* stat, float* partial, int max_ctas, cudaStream_t s) {
  const int C = z.C;
  if (C % 4 || C / 4 > BN_THREADS || z.pitch % 4 || z.coff % 4 || y.pitch % 4 || y.coff % 4) { set_thread_error("bn_train_fwd: unsupported view"); return 1; }
  const long long rows = (long long)F * z.H * z.W;
  long long rpc;
  const int ctas = bn_ctas(rows, max_ctas, &rpc);
  const int lanes = BN_THREADS / (C / 4);
  bn_colreduce_kernel<0><<<ctas, BN_THREADS, (size_t)lanes * C * 4, s>>>((const float*)z.base, z.pitch, z.coff, nullptr, 0, 0, nullptr, 0, 0, nullptr, rows, C, rpc, partial);
  SSNB_LAUNCH_CHECK("bn_colreduce_kernel<mean>");
  bn_stat_finish_kernel<<<(C + 127) / 128, 128, 0, s>>>(partial, ctas, C, (double)rows, 0, eps, momentum, stat, nullptr, nullptr);
  SSNB_LAUNCH_CHECK("bn_stat_finish_kernel");
  bn_colreduce_kernel<1><<<ctas, BN_THREADS, (size_t)lanes * C * 4, s>>>((const float*)z.base, z.pitch, z.coff, nullptr, 0, 0, nullptr, 0, 0, stat, rows, C, rpc, partial);
  SSNB_LAUNCH_CHECK("bn_colreduce_kernel<var>");
  bn_stat_finish_kernel<<<(C + 127) / 128, 128, 0, s>>>(partial, ctas, C, (double)rows, 1, eps, momentum, stat, running_mean, running_var);
  SSNB_LAUNCH_CHECK("bn_stat_finish_kernel");
  const long long n = rows * (C / 4);
  bn_apply_relu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float*)z.base, z.pitch, z.coff, stat, gamma, beta, rows, C, (float*)y.base, y.pitch,
                                                                 y.coff, (__half*)y_planes.base, y_planes.lo_off);
  SSNB_LAUNCH_CHECK("bn_apply_relu_kernel");
  return 0;
}

int launch_bn_train_bwd(View z, View dy, View y, View dz, View dz_planes, float plane_scale, int* flag, int F, const float* gamma, float* stat,
                        float* partial, int max_ctas, float* dgamma, float* dbeta, const float* unscale, int accumulate, cudaStream_t s) {
  const int C = z.C;
  if (C % 4 || C / 4 > BN_THREADS || dy.pitch % 4 || dy.coff % 4 || dz.pitch % 4 || dz.coff % 4) { set_thread_error("bn_train_bwd: unsupported view"); return 1; }
  const long long rows = (long long)F * z.H * z.W;
  long long rpc;
  const int ctas = bn_ctas(rows, max_ctas / 2, &rpc);
  const int lanes = BN_THREADS / (C / 4);
  bn_colreduce_kernel<2><<<ctas, BN_THREADS, (size_t)lanes * 2 * C * 4, s>>>((const float*)z.base, z.pitch, z.coff, (const float*)dy.base, dy.pitch, dy.coff,
                                                                           (const float*)y.base, y.pitch, y.coff, stat, rows, C, rpc, partial);
  SSNB_LAUNCH_CHECK("bn_colreduce_kernel<grad>");
  bn_grad_finish_kernel<<<(C + 127) / 128, 128, 0, s>>>(partial, ctas, C, stat, dgamma, dbeta, unscale, accumulate);
  SSNB_LAUNCH_CHECK("bn_grad_finish_kernel");
  const long long n = rows * (C / 4);
  bn_bwd_apply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float*)z.base, z.pitch, z.coff, (const float*)dy.base, dy.pitch, dy.coff,
                                                                (const float*)y.base, y.pitch, y.coff, stat, gamma, rows, C, (float)(1.0 / (double)rows),
                                                                (float*)dz.base, dz.pitch, dz.coff, (__half*)dz_planes.base, dz_planes.lo_off, plane_scale, flag);
  SSNB_LAUNCH_CHECK("bn_bwd_apply_kernel");
  return 0;
}

}  // namespace ssnb
