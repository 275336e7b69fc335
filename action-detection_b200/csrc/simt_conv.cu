// SIMT (CUDA-core, fp32 accumulate) convolution family: forward, data-gradient and weight-gradient
// as implicit GEMMs over NHWC tensors.  This is the EXACT-precision engine of libssn_b200
// (SSNB_EXACT_FP32: fp32 storage, end-to-end parity with the reference's fp32 PyTorch path,
// ssn_models.py:266 / model_zoo/bninception/pytorch_load.py:37-61) and the generic-geometry kernel
// for the layers the tensor-core path does not cover.
#include "common.cuh"

namespace ssnb {

namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int AS_LD = BM + 4;

template <typename T> struct Vec8;   // 8 consecutive storage elements -> 8 floats
template <> struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, float* o) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  }
};
template <> struct Vec8<__half> {
  static __device__ __forceinline__ void load(const __half* p, float* o) {
    uint4 r = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); o[2 * i] = f.x; o[2 * i + 1] = f.y; }
  }
};
template <typename T> struct Vec4;
template <> struct Vec4<float> {
  static __device__ __forceinline__ void load(const float* p, float* o) {
    float4 a = *reinterpret_cast<const float4*>(p); o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct Vec4<__half> {
  static __device__ __forceinline__ void load(const __half* p, float* o) {
    uint2 r = *reinterpret_cast<const uint2*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&r);
    float2 a = __half22float2(h[0]), b = __half22float2(h[1]); o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
  }
  static __device__ __forceinline__ void store(__half* p, const float* v) {
    __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
    uint2 r; r.x = *reinterpret_cast<uint32_t*>(&a); r.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = r;
  }
};

// source coordinate of tap index t (0..k-1) for destination coordinate d
__device__ __forceinline__ bool src_coord(int d, int t, int stride, int pad, int limit, bool dgrad, int& out) {
  if (!dgrad) { out = d * stride + t - pad; return out >= 0 && out < limit; }
  int v = d + pad - t;
  if (v < 0 || (v % stride) != 0) return false;
  out = v / stride;
  return out < limit;
}

// rows = destination pixels (F*DH*DW), cols = Cdst, K = taps*Csrc
template <typename T, bool FLATK>
__global__ void __launch_bounds__(NT) conv_kernel(ConvArgs a) {
  __shared__ __align__(16) float As[BK][AS_LD];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const long long M = (long long)a.F * a.DH * a.DW;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const T* __restrict__ src = reinterpret_cast<const T*>(a.src);
  const T* __restrict__ wgt = reinterpret_cast<const T*>(a.wgt);

  // A loader: this thread always serves row (tid % BM), k-half (tid / BM)
  const int lrow = tid % BM, lhalf = tid / BM;
  const long long mrow = m0 + lrow;
  const bool row_ok = mrow < M;
  int rf = 0, ry = 0, rx = 0;
  if (row_ok) { rf = (int)(mrow / (a.DH * a.DW)); int rem = (int)(mrow % (a.DH * a.DW)); ry = rem / a.DW; rx = rem % a.DW; }
  // B loader: k row tid/16, 4 columns
  const int bk = tid / 16, bn = (tid % 16) * 4;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int taps = a.kh * a.kw;
  const int Ktot = taps * a.Csrc;
  const int nchunks = FLATK ? (Ktot + BK - 1) / BK : taps * (a.Csrc / BK);
  const int cpt = FLATK ? 1 : a.Csrc / BK;   // chunks per tap

  for (int ch = 0; ch < nchunks; ++ch) {
    float av[8];
    if (!FLATK) {
      const int tap = ch / cpt, c0 = (ch % cpt) * BK;
      const int tr = tap / a.kw, ts = tap % a.kw;
      int sy, sx;
      bool ok = row_ok && src_coord(ry, tr, a.stride, a.pad_h, a.SH, a.dgrad, sy) &&
                src_coord(rx, ts, a.stride, a.pad_w, a.SW, a.dgrad, sx);
      if (ok) {
        const T* p = src + ((long long)(rf * a.SH + sy) * a.SW + sx) * a.src_pitch + a.src_coff + c0 + lhalf * 8;
        Vec8<T>::load(p, av);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = 0.f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int kf = ch * BK + lhalf * 8 + j;
        float v = 0.f;
        if (row_ok && kf < Ktot) {
          const int tap = kf / a.Csrc, c = kf % a.Csrc;
          int sy, sx;
          if (src_coord(ry, tap / a.kw, a.stride, a.pad_h, a.SH, a.dgrad, sy) &&
              src_coord(rx, tap % a.kw, a.stride, a.pad_w, a.SW, a.dgrad, sx))
            v = to_f<T>(src[((long long)(rf * a.SH + sy) * a.SW + sx) * a.src_pitch + a.src_coff + c]);
        }
        av[j] = v;
      }
    }
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    {
      const int kf = ch * BK + bk;   // flat k index == tap*Csrc + c in both modes
      if (kf < Ktot && n0 + bn < a.Cdst) Vec4<T>::load(wgt + (long long)kf * a.Cdst + n0 + bn, bv);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) As[lhalf * 8 + j][lrow] = av[j];
    *reinterpret_cast<float4*>(&Bs[bk][bn]) = make_float4(bv[0], bv[1], bv[2], bv[3]);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float br[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
  }

  const int nc = n0 + tx * 4;
  if (nc >= a.Cdst) return;
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (a.bias) {
#pragma unroll
    for (int j = 0; j < 4; ++j) bias[j] = a.bias[nc + j];
  }
  T* __restrict__ dst = reinterpret_cast<T*>(a.dst);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + ty * 8 + i;
    if (m >= M) break;
    T* p = dst + m * a.dst_pitch + a.dst_coff + nc;   // rows are dense pixels of the dst tensor
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = acc[i][j] + bias[j];
    if (a.accumulate) {
      float o[4];
      Vec4<T>::load(p, o);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] += o[j];
    }
    if (a.relu) {
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = relu(v[j]);
    }
    Vec4<T>::store(p, v);
  }
}

// ---- weight gradient --------------------------------------------------------------------------
constexpr int WM = 64, WN = 64, WK = 16;

// partial[split][tap][co][ci] = sum over rows in split of dz[row][co] * x[src(row,tap)][ci]
template <typename T, bool FLATN>
__global__ void __launch_bounds__(NT) wgrad_kernel(WgradArgs a) {
  __shared__ __align__(16) float As[WK][WM];
  __shared__ __align__(16) float Bs[WK][WN];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const int taps = a.k * a.k;
  const int Ntot = FLATN ? taps * a.Cin : a.Cin;
  const int ntile = (Ntot + WN - 1) / WN;
  const int co0 = (blockIdx.x / ntile) * WM;
  const int n0 = (blockIdx.x % ntile) * WN;
  const int tap = FLATN ? 0 : blockIdx.y;
  const int tr = tap / a.k, ts = tap % a.k;
  const int split = blockIdx.z;
  const long long M = (long long)a.F * a.OH * a.OW;
  const long long r0 = (long long)split * a.rows_per_split;
  const long long r1 = (r0 + a.rows_per_split < M) ? r0 + a.rows_per_split : M;
  const T* __restrict__ dz = reinterpret_cast<const T*>(a.dz);
  const T* __restrict__ x = reinterpret_cast<const T*>(a.x);
  const int lk = tid / 16, lc = (tid % 16) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (long long rb = r0; rb < r1; rb += WK) {
    const long long row = rb + lk;
    float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (row < r1) {
      if (co0 + lc < a.Cout) Vec4<T>::load(dz + row * a.dz_pitch + a.dz_coff + co0 + lc, av);
      const int f = (int)(row / (a.OH * a.OW));
      const int rem = (int)(row % (a.OH * a.OW));
      const int oy = rem / a.OW, ox = rem % a.OW;
      if (!FLATN) {
        const int iy = oy * a.stride + tr - a.pad, ix = ox * a.stride + ts - a.pad;
        if (iy >= 0 && iy < a.IH && ix >= 0 && ix < a.IW && n0 + lc < a.Cin)
          Vec4<T>::load(x + ((long long)(f * a.IH + iy) * a.IW + ix) * a.x_pitch + a.x_coff + n0 + lc, bv);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = n0 + lc + j;
          if (n < Ntot) {
            const int tp = n / a.Cin, ci = n % a.Cin;
            const int iy = oy * a.stride + tp / a.k - a.pad, ix = ox * a.stride + tp % a.k - a.pad;
            if (iy >= 0 && iy < a.IH && ix >= 0 && ix < a.IW)
              bv[j] = to_f<T>(x[((long long)(f * a.IH + iy) * a.IW + ix) * a.x_pitch + a.x_coff + ci]);
          }
        }
      }
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&As[lk][lc]) = make_float4(av[0], av[1], av[2], av[3]);
    *reinterpret_cast<float4*>(&Bs[lk][lc]) = make_float4(bv[0], bv[1], bv[2], bv[3]);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < WK; ++kk) {
      float4 av4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 bv4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float ar[4] = {av4.x, av4.y, av4.z, av4.w};
      const float br[4] = {bv4.x, bv4.y, bv4.z, bv4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty * 4 + i;
    if (co >= a.Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= Ntot) continue;
      const int tp = FLATN ? n / a.Cin : tap;
      const int ci = FLATN ? n % a.Cin : n;
      a.partial[(((long long)split * taps + tp) * a.Cout + co) * a.Cin + ci] = acc[i][j];
    }
  }
}

// one table entry's CTAs (from q.block0 on) enumerate the partial layout [tap][co][ci] (coalesced reads of every split) and
// write the reference layout [co][ci][tap]
__device__ __forceinline__ void wgrad_finalize_entry(const FinalizeEntry& q, const float* unscale, int* flag, float out_scale, int accumulate) {
  const long long total = (long long)q.taps * q.Cout * q.Cin;
  const long long i = (long long)(blockIdx.x - q.block0) * blockDim.x + threadIdx.x;
  if (unscale) out_scale *= __ldg(unscale);
  if (q.bias_partial && q.db && i < q.Cout) {     // bias gradient from the weight-gradient kernel's ones-operand accumulator
    float sb = 0.f;
    for (int sp = 0; sp < q.splits; ++sp) sb += q.bias_partial[(long long)sp * q.Cout + i];
    q.db[i] = (accumulate ? q.db[i] : 0.f) + sb * q.mult[i] * out_scale;
  }
  if (i >= total) return;
  const int ci = (int)(i % q.Cin);
  const int co = (int)((i / q.Cin) % q.Cout);
  const int tap = (int)(i / ((long long)q.Cin * q.Cout));
  float s = 0.f;
  for (int sp = 0; sp < q.splits; ++sp) s += q.partial[(long long)sp * total + i];
  if (flag && !(fabsf(s) <= 3.0e38f)) *flag = 1;         // inf / NaN: a gradient left the fp16 range under this loss scale
  float* o = q.dw + ((long long)co * q.Cin + ci) * q.taps + tap;
  *o = (accumulate ? *o : 0.f) + s * q.mult[co] * out_scale;
}

__global__ void wgrad_finalize_kernel(const float* __restrict__ partial, int splits, int taps, int Cout, int Cin,
                                      const float* __restrict__ mult, float out_scale, float* __restrict__ dw, int accumulate,
                                      const float* __restrict__ bias_partial, float* __restrict__ db, int* __restrict__ flag,
                                      const float* __restrict__ unscale) {
  const FinalizeEntry q{partial, mult, dw, bias_partial, db, splits, taps, Cout, Cin, 0, 0};
  wgrad_finalize_entry(q, unscale, flag, out_scale, accumulate);
}

__global__ void wgrad_finalize_all_kernel(const __grid_constant__ FinalizeTable t, float out_scale, int accumulate) {
  int ei = 0;
  while (ei + 1 < t.n && (int)blockIdx.x >= t.e[ei + 1].block0) ++ei;       // <= 36 entries, uniform per block
  wgrad_finalize_entry(t.e[ei], t.unscale, t.flag, out_scale, accumulate);
}

}  // namespace

template <typename T> int launch_conv(const ConvArgs& a, cudaStream_t s) {
  const long long M = (long long)a.F * a.DH * a.DW;
  dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)((a.Cdst + BN - 1) / BN));
  if (a.Cdst % 4 != 0) { set_thread_error("launch_conv: Cdst must be a multiple of 4"); return 1; }
  if (a.Csrc % BK == 0 && a.src_coff % 8 == 0 && a.src_pitch % 8 == 0)
    conv_kernel<T, false><<<grid, NT, 0, s>>>(a);
  else
    conv_kernel<T, true><<<grid, NT, 0, s>>>(a);
  SSNB_LAUNCH_CHECK("conv_kernel");
  return 0;
}
template int launch_conv<float>(const ConvArgs&, cudaStream_t);
template int launch_conv<__half>(const ConvArgs&, cudaStream_t);

template <typename T> int launch_wgrad(const WgradArgs& a, cudaStream_t s) {
  const int taps = a.k * a.k;
  const bool flat = (a.Cin % 4 != 0) || (a.x_coff % 4 != 0) || (a.x_pitch % 4 != 0) || a.Cin < 16;
  const int Ntot = flat ? taps * a.Cin : a.Cin;
  dim3 grid((unsigned)(((a.Cout + WM - 1) / WM) * ((Ntot + WN - 1) / WN)), flat ? 1u : (unsigned)taps,
            (unsigned)a.splits);
  if (a.Cout % 4 != 0) { set_thread_error("launch_wgrad: Cout must be a multiple of 4"); return 1; }
  if (flat) wgrad_kernel<T, true><<<grid, NT, 0, s>>>(a);
  else wgrad_kernel<T, false><<<grid, NT, 0, s>>>(a);
  SSNB_LAUNCH_CHECK("wgrad_kernel");
  return 0;
}
template int launch_wgrad<float>(const WgradArgs&, cudaStream_t);
template int launch_wgrad<__half>(const WgradArgs&, cudaStream_t);

int launch_wgrad_finalize(const float* partial, int splits, int taps, int Cout, int Cin, const float* mult,
                          float out_scale, float* dw_ref, int accumulate, cudaStream_t s, const float* bias_partial, float* db, int* flag,
                          const float* unscale) {
  const long long total = (long long)taps * Cout * Cin;
  wgrad_finalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(partial, splits, taps, Cout, Cin, mult,
                                                                       out_scale, dw_ref, accumulate, bias_partial, db, flag, unscale);
  SSNB_LAUNCH_CHECK("wgrad_finalize_kernel");
  return 0;
}

int launch_wgrad_finalize_all(const FinalizeTable& t, float out_scale, int accumulate, cudaStream_t s) {
  if (t.n <= 0) return 0;
  wgrad_finalize_all_kernel<<<(unsigned)t.total_blocks, 256, 0, s>>>(t, out_scale, accumulate);
  SSNB_LAUNCH_CHECK("wgrad_finalize_all_kernel");
  return 0;
}

}  // namespace ssnb
