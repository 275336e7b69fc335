// Memory-bound glue of the BNInception graph over NHWC views: layout conversion, 7x7 global pooling
// (bn_inception.yaml:552), the backward's gradient exponent, and BN-folding weight packing (frozen
// BatchNorm2d, ssn_models.py:156-174).  Max / average pooling and the ReLU gradient mask are in glue_vec.cu.
#include <cfloat>

#include "common.cuh"

namespace ssnb {
namespace {

constexpr int TPB = 256;
inline unsigned blocks_for(long long n) { return (unsigned)((n + TPB - 1) / TPB); }

template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, int F, int C, int H, int W, T* __restrict__ dst,
                                    int pitch, int coff, float scale) {
  const long long total = (long long)F * H * W * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const long long p = i / C;           // f*H*W + y*W + x
  const long long f = p / ((long long)H * W);
  const long long yx = p % ((long long)H * W);
  dst[p * pitch + coff + c] = from_f<T>(src[(f * C + c) * (long long)H * W + yx] * scale);
}

template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ src, int F, int C, int H, int W, int pitch, int coff,
                                    float scale, float* __restrict__ dst) {
  const long long total = (long long)F * C * H * W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long yx = i % ((long long)H * W);
  const int c = (int)((i / ((long long)H * W)) % C);
  const long long f = i / ((long long)H * W * C);
  dst[i] = to_f<T>(src[(f * H * W + yx) * pitch + coff + c]) * scale;
}

template <typename T>
__global__ void gpool_fwd_kernel(const T* __restrict__ src, int HW, int C, int pitch, int coff, int F,
                                 float* __restrict__ feat) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * C) return;
  const int c = (int)(i % C);
  const long long f = i / C;
  float s = 0.f;
  for (int p = 0; p < HW; ++p) s += to_f<T>(src[(f * HW + p) * pitch + coff + c]);
  feat[i] = s / (float)HW;
}

template <typename T>
__global__ void gpool_bwd_kernel(const float* __restrict__ dfeat, float scale, const float* __restrict__ scale_dev, int HW, int C, int pitch,
                                 int coff, int F, T* __restrict__ ddst, const T* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * HW * C) return;
  if (scale_dev) scale *= __ldg(scale_dev);
  const int c = (int)(i % C);
  const long long p = i / C;
  const long long f = p / HW;
  float g = dfeat[f * C + c] / (float)HW * scale;
  if (y && !(to_f<T>(y[p * pitch + coff + c]) > 0.f)) g = 0.f;     // fused ReLU gradient mask (same view geometry)
  ddst[p * pitch + coff + c] = from_f<T>(g);
}

// one CTA: max |dfeat| (any inf / NaN noted separately: fmaxf drops NaN) -> the gradient exponent k (see launch_grad_exponent).
// The entry gradient max|dfeat| * grad_scale / HW = m * 2^e with m in [0.5, 1) is formed from the three operands' exponents, so no
// intermediate overflows: frexp(max|dfeat|) * frexp(grad_scale) / HW in fp32, whose frexp exponent is added to theirs.
constexpr int GE_THREADS = 1024;
__global__ void __launch_bounds__(GE_THREADS) grad_exponent_kernel(const float* __restrict__ dfeat, long long n, float grad_scale, int HW,
                                                                   float* __restrict__ gscale, int* __restrict__ flag) {
  __shared__ float wmax[GE_THREADS / 32];
  __shared__ int wbad[GE_THREADS / 32];
  float m = 0.f;
  int bad = 0;
  for (long long i = threadIdx.x; i < n; i += GE_THREADS) {
    const float a = fabsf(__ldg(dfeat + i));
    if (!(a <= FLT_MAX)) bad = 1;
    m = fmaxf(m, a);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o)); bad |= __shfl_xor_sync(0xffffffffu, bad, o); }
  if (threadIdx.x % 32 == 0) { wmax[threadIdx.x / 32] = m; wbad[threadIdx.x / 32] = bad; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < GE_THREADS / 32; ++w) { m = fmaxf(m, wmax[w]); bad |= wbad[w]; }
  int k = 0;
  if (bad) {
    if (flag) *flag = 1;
  } else if (m > 0.f) {
    int ea, eg, e;
    const float fa = frexpf(m, &ea), fg = frexpf(grad_scale, &eg);
    frexpf(fa * fg / (float)HW, &e);
    k = GRAD_EXP_TOP - (ea + eg + e);
    k = k < -GRAD_EXP_MAX ? -GRAD_EXP_MAX : (k > GRAD_EXP_MAX ? GRAD_EXP_MAX : k);
  }
  gscale[0] = ldexpf(1.0f, k);
  gscale[1] = ldexpf(1.0f, -k);
}

// all layers of the network in a few launches (69 per-layer launches would be mostly launch latency: the weights are
// re-packed after every optimizer step)
template <typename T>
__global__ void pack_all_kernel(const __grid_constant__ PackTable t) {
  int ei = 0;
  while (ei + 1 < t.n && (int)blockIdx.x >= t.e[ei + 1].block0) ++ei;       // <= 32 entries, uniform per block
  const PackEntry& q = t.e[ei];
  const int taps = q.taps;
  const long long total = (long long)q.cout * q.cin * taps;
  float av = 0.f;
  __shared__ float wmax[TPB / 32];
  if (taps <= PACK_TILE_TAPS) {
    // tiled path: a CTA owns PACK_TILE output x PACK_TILE input channels x taps.  The source rows ([ci][tap] runs of one output
    // channel) are read contiguously into shared memory, wf is then written with the output channel and wd with the input channel
    // as the lane index, so all three streams are coalesced (the element-wise path scatters both stores)
    __shared__ float tile[PACK_TILE][PACK_TILE * PACK_TILE_TAPS + 1];
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int ci_tiles = (q.cin + PACK_TILE - 1) / PACK_TILE;
    const int b = (int)blockIdx.x - q.block0;
    const int co0 = (b / ci_tiles) * PACK_TILE, ci0 = (b % ci_tiles) * PACK_TILE;
    const int nco = min(PACK_TILE, q.cout - co0), nci = min(PACK_TILE, q.cin - ci0);
    const int row = nci * taps;
    if (ci0 == 0 && (int)threadIdx.x < nco) {
      const int co = co0 + threadIdx.x;
      const float s = q.nofold ? 1.0f : q.gamma[co] / sqrtf(q.var[co] + 1e-5f);
      q.scale[co] = s;
      const float bf = q.nofold ? q.b[co] : (q.b[co] - q.mean[co]) * s + q.beta[co];
      q.bias[co] = bf;
      if (q.bias_b) q.bias_b[co] = bf;
    }
    for (int r = warp; r < nco; r += TPB / 32) {
      const int co = co0 + r;
      const float s = q.nofold ? 1.0f : q.gamma[co] / sqrtf(q.var[co] + 1e-5f);
      const float* src = q.w + ((long long)co * q.cin + ci0) * taps;
      for (int e = lane; e < row; e += 32) { const float fv = src[e] * s; tile[r][e] = fv; av = fmaxf(av, fabsf(fv)); }
    }
    __syncthreads();
    T* wf = reinterpret_cast<T*>(q.wf);
    T* wd = reinterpret_cast<T*>(q.wd);
    for (int e = warp; e < row; e += TPB / 32) {                 // e = local ci * taps + tap; lanes = output channels
      const int cil = e / taps, tap = e - cil * taps;
      if (lane < nco) wf[((long long)tap * q.cin + ci0 + cil) * q.cout + co0 + lane] = from_f<T>(tile[lane][e]);
    }
    for (int e = warp; e < nco * taps; e += TPB / 32) {          // e = local co * taps + tap; lanes = input channels
      const int r = e / taps, tap = e - r * taps;
      if (lane < nci) wd[((long long)tap * q.cout + co0 + r) * q.cin + ci0 + lane] = from_f<T>(tile[r][lane * taps + tap]);
    }
  } else {
  const long long base = (long long)((int)blockIdx.x - q.block0) * (PACK_PER_THREAD * TPB) + threadIdx.x;
#pragma unroll
  for (int j = 0; j < PACK_PER_THREAD; ++j) {
    const long long i = base + j * TPB;
    if (i < q.cout) {
      const float s = q.nofold ? 1.0f : q.gamma[i] / sqrtf(q.var[i] + 1e-5f);
      q.scale[i] = s;
      const float bf = q.nofold ? q.b[i] : (q.b[i] - q.mean[i]) * s + q.beta[i];
      q.bias[i] = bf;
      if (q.bias_b) q.bias_b[i] = bf;
    }
    if (i < total) {
      const int tap = (int)(i % taps);
      const int ci = (int)((i / taps) % q.cin);
      const int co = (int)(i / ((long long)taps * q.cin));
      const float s = q.nofold ? 1.0f : q.gamma[co] / sqrtf(q.var[co] + 1e-5f);
      const float fv = q.w[i] * s;
      const T v = from_f<T>(fv);
      reinterpret_cast<T*>(q.wf)[((long long)tap * q.cin + ci) * q.cout + co] = v;
      reinterpret_cast<T*>(q.wd)[((long long)tap * q.cout + co) * q.cin + ci] = v;
      av = fmaxf(av, fabsf(fv));
    }
  }
  }
  if (q.absmax) {
    // one atomic per CTA instead of one per warp (they serialise in L2 on the 69 per-layer addresses)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) av = fmaxf(av, __shfl_xor_sync(0xffffffffu, av, o));
    if (threadIdx.x % 32 == 0) wmax[threadIdx.x / 32] = av;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int w = 1; w < TPB / 32; ++w) av = fmaxf(av, wmax[w]);
      if (av > 0.f) atomicMax(reinterpret_cast<int*>(q.absmax), __float_as_int(av));
    }
  }
}

}  // namespace

template <typename T> int launch_pack_all(const PackTable& t, int total_blocks, cudaStream_t s) {
  if (t.n <= 0) return 0;
  pack_all_kernel<T><<<(unsigned)total_blocks, TPB, 0, s>>>(t);
  SSNB_LAUNCH_CHECK("pack_all_kernel");
  return 0;
}
template int launch_pack_all<float>(const PackTable&, int, cudaStream_t);
template int launch_pack_all<__half>(const PackTable&, int, cudaStream_t);

#define V(T, v) reinterpret_cast<T*>((v).base)

template <typename T> int launch_nchw_to_nhwc(const float* src, int F, int C, int H, int W, View dst, float scale, cudaStream_t s) {
  const long long n = (long long)F * C * H * W;
  nchw_to_nhwc_kernel<T><<<blocks_for(n), TPB, 0, s>>>(src, F, C, H, W, V(T, dst), dst.pitch, dst.coff, scale);
  SSNB_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return 0;
}
template <typename T> int launch_nhwc_to_nchw(View src, int F, float scale, float* dst, cudaStream_t s) {
  const long long n = (long long)F * src.C * src.H * src.W;
  nhwc_to_nchw_kernel<T><<<blocks_for(n), TPB, 0, s>>>(V(const T, src), F, src.C, src.H, src.W, src.pitch, src.coff, scale, dst);
  SSNB_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return 0;
}
template <typename T> int launch_gpool_fwd(View src, int F, float* feat, cudaStream_t s) {
  gpool_fwd_kernel<T><<<blocks_for((long long)F * src.C), TPB, 0, s>>>(V(const T, src), src.H * src.W, src.C, src.pitch,
                                                                      src.coff, F, feat);
  SSNB_LAUNCH_CHECK("gpool_fwd_kernel");
  return 0;
}
template <typename T> int launch_gpool_bwd(const float* dfeat, float scale, const float* scale_dev, View ddst, int F, const void* y,
                                           cudaStream_t s) {
  const long long n = (long long)F * ddst.H * ddst.W * ddst.C;
  gpool_bwd_kernel<T><<<blocks_for(n), TPB, 0, s>>>(dfeat, scale, scale_dev, ddst.H * ddst.W, ddst.C, ddst.pitch, ddst.coff, F, V(T, ddst),
                                                    reinterpret_cast<const T*>(y));
  SSNB_LAUNCH_CHECK("gpool_bwd_kernel");
  return 0;
}
int launch_grad_exponent(const float* dfeat, long long n, float grad_scale, int HW, float* gscale, int* flag, cudaStream_t s) {
  grad_exponent_kernel<<<1, GE_THREADS, 0, s>>>(dfeat, n, grad_scale, HW, gscale, flag);
  SSNB_LAUNCH_CHECK("grad_exponent_kernel");
  return 0;
}
#define INST(T)                                                                                              \
  template int launch_nchw_to_nhwc<T>(const float*, int, int, int, int, View, float, cudaStream_t);                 \
  template int launch_nhwc_to_nchw<T>(View, int, float, float*, cudaStream_t);                               \
  template int launch_gpool_fwd<T>(View, int, float*, cudaStream_t);                                         \
  template int launch_gpool_bwd<T>(const float*, float, const float*, View, int, const void*, cudaStream_t);
INST(float)
INST(__half)

}  // namespace ssnb
