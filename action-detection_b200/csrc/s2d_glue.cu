// Layout helpers (FAST and EXACT_TC) that let every convolution of BNInception run on the stride-1 tensor-core kernels:
//  * conv1 (7x7 stride 2 pad 3, bn_inception.yaml:3-5) as a 4x4 stride-1 convolution over the
//    space-to-depth input  xs[f, i, j, (a*2+b)*Cin + c] = x[f, 2i+a, 2j+b, c]   (r = 2*dr + a - 1)
//  * stride-2 3x3 layers (inception_3c/4e): backward through a zero-upsampled output gradient.
#include "common.cuh"

#include <type_traits>

namespace ssnb {
namespace {

// Packed layout: Ck = 4*Cs channels per pixel, channel = ds*Cs + (a*2+b)*Cin + c holds
//   x[f, 2*i + a, 2*(j + ds - 2) + b, c]      (zero outside the image / for the pad channels)
// so the 7x7/2 convolution becomes FOUR vertical taps (dr = 0..3, dy = dr - 2) with K = 4*Cs each:
//   r = 2*dr + a - 1,  s = 2*ds + b - 1.
// T = __half (FAST) copies the value; T = float (EXACT_TC) writes its hi plane at dst and its lo plane lo_off bytes further
template <typename T>
__global__ void nhwc_to_s2d_kernel(const T* __restrict__ src, int F, int H, int W, int Cin, int spitch, int scoff,
                                   __half* __restrict__ dst, long long lo_off, int Cs) {
  const int H2 = H / 2, W2 = W / 2, Ck = 4 * Cs;
  const long long total = (long long)F * H2 * W2 * Ck;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % Ck);
  const long long p = i / Ck;
  const int x2 = (int)(p % W2), y2 = (int)((p / W2) % H2);
  const long long f = p / ((long long)W2 * H2);
  const int ds = ch / Cs, q = ch % Cs;
  T v = 0.f;
  const int xs = x2 + ds - 2;
  if (q < 4 * Cin && xs >= 0 && xs < W2) {
    const int ab = q / Cin, c = q % Cin;
    v = src[((f * H + 2 * y2 + ab / 2) * W + 2 * xs + ab % 2) * spitch + scoff + c];
  }
  if constexpr (std::is_same_v<T, float>) {
    const __half h = __float2half_rn(v);
    dst[i] = h;
    *reinterpret_cast<__half*>(reinterpret_cast<char*>(dst + i) + lo_off) = __float2half_rn(v - __half2float(h));
  } else {
    dst[i] = v;
  }
}

// ws[dr][co][ds*Cs + (a*2+b)*Cin + c] = wd[(r*7+s)][co][c],  r = 2*dr+a-1, s = 2*ds+b-1 (0 outside 0..6)
__global__ void pack_conv1_s2d_kernel(const __half* __restrict__ wd, int Cout, int Cin, int Cs, __half* __restrict__ ws) {
  const int Ck = 4 * Cs;
  const long long total = (long long)4 * Cout * Ck;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % Ck);
  const int co = (int)((i / Ck) % Cout);
  const int dr = (int)(i / ((long long)Ck * Cout));
  const int ds = ch / Cs, q = ch % Cs;
  __half v = __float2half_rn(0.f);
  if (q < 4 * Cin) {
    const int ab = q / Cin, c = q % Cin;
    const int r = 2 * dr + ab / 2 - 1, s = 2 * ds + ab % 2 - 1;
    if (r >= 0 && r < 7 && s >= 0 && s < 7) v = wd[((long long)(r * 7 + s) * Cout + co) * Cin + c];
  }
  ws[i] = v;
}

// dw_ref[co][c][r][s] = mult[co]*out_scale * sum_splits partial[sp][dr][co][ds*Cs + (a*2+b)*Cin + c]
__global__ void wgrad_finalize_s2d_kernel(const float* __restrict__ partial, int splits, int Cout, int Cin, int Cs,
                                          const float* __restrict__ mult, float out_scale, const float* __restrict__ unscale,
                                          float* __restrict__ dw, int accumulate) {
  const int Ck = 4 * Cs;
  const long long total = (long long)Cout * Cin * 49;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int s = (int)(i % 7), r = (int)((i / 7) % 7);
  const int c = (int)((i / 49) % Cin), co = (int)(i / (49LL * Cin));
  const int dr = (r + 1) / 2, a = (r + 1) % 2, ds = (s + 1) / 2, b = (s + 1) % 2;
  const int ch = ds * Cs + (a * 2 + b) * Cin + c;
  float acc = 0.f;
  for (int sp = 0; sp < splits; ++sp) acc += partial[(((long long)sp * 4 + dr) * Cout + co) * Ck + ch];
  if (unscale) out_scale *= __ldg(unscale);
  dw[i] = (accumulate ? dw[i] : 0.f) + acc * mult[co] * out_scale;
}

// fused input conversion: NCHW fp32 frames -> packed space-to-depth fp16; one thread per (pixel, ds block):
// float2 reads coalesced along x, the Cs-channel block is assembled in registers and stored as 16-byte vectors
// CIN > 0: compile-time channel count (RGB 3 / Flow 10): the channel loop unrolls and the staging arrays stay in registers
// LO (EXACT_TC): also writes the lo plane, lo_off bytes after the hi plane
template <int CS, int CIN, bool LO>
__global__ void nchw_to_s2d_kernel(const float* __restrict__ src, int F, int Cin_rt, int H, int W, __half* __restrict__ dst,
                                   long long lo_off) {
  const int Cin = CIN ? CIN : Cin_rt;
  const int H2 = H / 2, W2 = W / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * H2 * W2 * 4) return;
  const unsigned iu = (unsigned)i;                 // < 2^31 threads: 32-bit index arithmetic
  const int ds = (int)(iu & 3u);
  const unsigned pu = iu >> 2;
  const int x2 = (int)(pu % (unsigned)W2), y2 = (int)((pu / (unsigned)W2) % (unsigned)H2);
  const long long p = pu;
  const long long f = pu / (unsigned)(W2 * H2);
  __align__(16) __half vh[CS];
  __align__(16) __half vl[LO ? CS : 1];
#pragma unroll
  for (int c = 0; c < CS; ++c) {
    vh[c] = __float2half_rn(0.f);
    if constexpr (LO) vl[c] = __float2half_rn(0.f);
  }
  const int xs = x2 + ds - 2;
  if (xs >= 0 && xs < W2) {
#pragma unroll
    for (int c = 0; c < Cin; ++c) {
      const float* pl = src + ((f * Cin + c) * H + 2 * y2) * (long long)W + 2 * xs;
      const float2 r0 = __ldg(reinterpret_cast<const float2*>(pl));
      const float2 r1 = __ldg(reinterpret_cast<const float2*>(pl + W));
      const float q[4] = {r0.x, r0.y, r1.x, r1.y};
#pragma unroll
      for (int ab = 0; ab < 4; ++ab) {
        const __half h = __float2half_rn(q[ab]);
        vh[ab * Cin + c] = h;
        if constexpr (LO) vl[ab * Cin + c] = __float2half_rn(q[ab] - __half2float(h));
      }
    }
  }
  __half* o = dst + p * (4 * CS) + ds * CS;
  uint4* oh = reinterpret_cast<uint4*>(o);
  uint4* ol = reinterpret_cast<uint4*>(reinterpret_cast<char*>(o) + lo_off);
#pragma unroll
  for (int q = 0; q < CS / 8; ++q) {
    oh[q] = reinterpret_cast<const uint4*>(vh)[q];
    if constexpr (LO) ol[q] = reinterpret_cast<const uint4*>(vl)[q];
  }
}

// dst[f, y, x, c] = (y, x both even) ? src[f, y/2, x/2, c] : 0      (8 channels = 16 bytes per thread)
__global__ void upsample2_zero_kernel(const __half* __restrict__ src, int OH, int OW, int C, int spitch, int scoff,
                                      __half* __restrict__ dst, int H, int W, int F) {
  const int G = C / 8;
  const long long total = (long long)F * H * W * G;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const unsigned iu = (unsigned)i;
  const int g = (int)(iu % (unsigned)G);
  const unsigned pu = iu / (unsigned)G;
  const int x = (int)(pu % (unsigned)W), y = (int)((pu / (unsigned)W) % (unsigned)H);
  const long long p = pu;
  const long long f = pu / (unsigned)(W * H);
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (!(x & 1) && !(y & 1) && y / 2 < OH && x / 2 < OW)
    v = __ldg(reinterpret_cast<const uint4*>(src + ((f * OH + y / 2) * OW + x / 2) * spitch + scoff + g * 8));
  *reinterpret_cast<uint4*>(dst + p * C + g * 8) = v;
}

}  // namespace

int launch_nhwc_to_s2d(View src, int F, __half* dst, long long lo_off, int Cs, cudaStream_t s) {
  const long long n = (long long)F * (src.H / 2) * (src.W / 2) * 4 * Cs;
  const unsigned g = (unsigned)((n + 255) / 256);
  if (lo_off) nhwc_to_s2d_kernel<float><<<g, 256, 0, s>>>((const float*)src.base, F, src.H, src.W, src.C, src.pitch, src.coff, dst, lo_off, Cs);
  else nhwc_to_s2d_kernel<__half><<<g, 256, 0, s>>>((const __half*)src.base, F, src.H, src.W, src.C, src.pitch, src.coff, dst, lo_off, Cs);
  SSNB_LAUNCH_CHECK("nhwc_to_s2d_kernel");
  return 0;
}
template <bool LO>
static int nchw_to_s2d(const float* src, int F, int Cin, int H, int W, __half* dst, long long lo_off, int Cs, cudaStream_t s) {
  const long long n = (long long)F * (H / 2) * (W / 2) * 4;
  const unsigned g = (unsigned)((n + 255) / 256);
  if (Cs == 16 && Cin == 3) nchw_to_s2d_kernel<16, 3, LO><<<g, 256, 0, s>>>(src, F, Cin, H, W, dst, lo_off);
  else if (Cs == 40 && Cin == 10) nchw_to_s2d_kernel<40, 10, LO><<<g, 256, 0, s>>>(src, F, Cin, H, W, dst, lo_off);
  else if (Cs == 16) nchw_to_s2d_kernel<16, 0, LO><<<g, 256, 0, s>>>(src, F, Cin, H, W, dst, lo_off);
  else if (Cs == 40) nchw_to_s2d_kernel<40, 0, LO><<<g, 256, 0, s>>>(src, F, Cin, H, W, dst, lo_off);
  else { set_thread_error("nchw_to_s2d: unsupported channel count (RGB 3 or Flow 10)"); return 1; }
  SSNB_LAUNCH_CHECK("nchw_to_s2d_kernel");
  return 0;
}
int launch_nchw_to_s2d(const float* src, int F, int Cin, int H, int W, __half* dst, long long lo_off, int Cs, cudaStream_t s) {
  return lo_off ? nchw_to_s2d<true>(src, F, Cin, H, W, dst, lo_off, Cs, s) : nchw_to_s2d<false>(src, F, Cin, H, W, dst, lo_off, Cs, s);
}
int launch_pack_conv1_s2d(const __half* wd, int Cout, int Cin, int Cs, __half* ws, cudaStream_t s) {
  const long long n = 16LL * Cout * Cs;   // 4 taps x Cout x 4*Cs
  pack_conv1_s2d_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(wd, Cout, Cin, Cs, ws);
  SSNB_LAUNCH_CHECK("pack_conv1_s2d_kernel");
  return 0;
}
int launch_wgrad_finalize_s2d(const float* partial, int splits, int Cout, int Cin, int Cs, const float* mult, float out_scale,
                              const float* unscale, float* dw_ref, int accumulate, cudaStream_t s) {
  const long long n = (long long)Cout * Cin * 49;
  wgrad_finalize_s2d_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(partial, splits, Cout, Cin, Cs, mult, out_scale, unscale, dw_ref, accumulate);
  SSNB_LAUNCH_CHECK("wgrad_finalize_s2d_kernel");
  return 0;
}
int launch_upsample2_zero(View src, __half* dst, int H, int W, int F, cudaStream_t s) {
  const long long n = (long long)F * H * W * (src.C / 8);
  upsample2_zero_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const __half*)src.base, src.H, src.W, src.C, src.pitch, src.coff, dst, H, W, F);
  SSNB_LAUNCH_CHECK("upsample2_zero_kernel");
  return 0;
}

}  // namespace ssnb
