// Shared declarations for libssn_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>

namespace ssnb {

// NHWC view: a channel slice [coff, coff+C) of a buffer whose pixel pitch is `pitch` elements.
struct View {
  void* base = nullptr;
  int H = 0, W = 0, C = 0, pitch = 0, coff = 0;
  // SSNB_EXACT_TC operand planes: `base` is the fp16 HI plane and the LO plane (x - float(hi), fp16) of the same
  // geometry starts `lo_off` bytes after it; 0 = a plain single-plane view
  long long lo_off = 0;
};

extern std::atomic<long long> g_launches;  // every kernel launch of this library bumps it
void set_thread_error(const std::string& s);
const std::string& thread_error();

// Per-launch device timing (ssnb_timing_begin / ssnb_timing_report, bench.py's roofline): while a timing session is open
// on this thread, every launch records a CUDA event behind itself on its stream; a launch's time is the distance to the
// previous event (launches are back to back on one stream).  The engine tags the launches it is about to make with the
// pass they belong to, the algorithmic FLOPs of the convolution they compute and its op name; umma_conv_launch adds its
// tile count and tile width, umma_wgrad_launch its CTAs per pixel split and split count.
struct LaunchTag {
  int phase = 3;                  // 0 forward, 1 data gradient, 2 weight gradient, 3 other
  double flop = 0.0;
  const char* op = nullptr;       // copied when the launch is recorded
  int tiles = 0, block_n = 0;     // umma_wgrad_kernel: ctas, splits
};
extern thread_local bool t_timing;
extern thread_local LaunchTag t_tag;
void timing_mark(const char* what, cudaStream_t s);

// every launcher names its stream `s`
#define SSNB_LAUNCH_CHECK(what)                                                       \
  do {                                                                                \
    ssnb::g_launches.fetch_add(1, std::memory_order_relaxed);                         \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess) {                                                          \
      ssnb::set_thread_error(std::string(what) + ": " + cudaGetErrorString(_e));      \
      return 2;                                                                       \
    }                                                                                 \
    if (ssnb::t_timing) ssnb::timing_mark(what, s);                                   \
  } while (0)

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
// the ReLU of every forward epilogue: NaN stays NaN (torch.relu; fmaxf(NaN, 0) would be 0), -0 and +0 give +0
__device__ __forceinline__ float relu(float v) { return v <= 0.f ? 0.f : v; }

// SSNB_EXACT_TC operand format: an fp32 value x is carried as hi = fp16(x), lo = fp16(x - float(hi)) (tc_glue.cu)
constexpr float HALF_MAX = 65504.f;
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// 4 fp32 values -> 8 bytes of hi + 8 bytes of lo at the same element offset of the two planes
__device__ __forceinline__ void store_planes4(__half* hi, long long lo_off, const float4& v) {
  uint2 h, l;
  split2(v.x, v.y, h.x, l.x);
  split2(v.z, v.w, h.y, l.y);
  *reinterpret_cast<uint2*>(hi) = h;
  *reinterpret_cast<uint2*>(reinterpret_cast<char*>(hi) + lo_off) = l;
}

// ---- SIMT convolution family (simt_conv.cu) ---------------------------------------------------
struct ConvArgs {
  const void* src; int SH, SW, Csrc, src_pitch, src_coff;   // x (fwd) or dz (dgrad)
  void* dst;       int DH, DW, Cdst, dst_pitch, dst_coff;   // y (fwd) or dx (dgrad)
  const void* wgt;                                          // [tap][csrc][cdst], storage type
  const float* bias;                                        // [Cdst] or nullptr
  int F, kh, kw, stride, pad_h, pad_w;                      // tap t = r * kw + s (r: row, s: column of the kernel)
  int relu, accumulate, dgrad;
};
struct WgradArgs {
  const void* dz; int OH, OW, Cout, dz_pitch, dz_coff;
  const void* x;  int IH, IW, Cin, x_pitch, x_coff;
  float* partial;                                           // [splits][taps][Cout][Cin]
  int F, k, stride, pad, rows_per_split, splits;
};
template <typename T> int launch_conv(const ConvArgs& a, cudaStream_t s);
template <typename T> int launch_wgrad(const WgradArgs& a, cudaStream_t s);
// dW_ref[co][ci][r][s] = mult[co] * sum_splits partial ; mult = bn_scale * 1/loss_scale
// unscale (optional device scalar, here and in every launcher below that takes one): multiplied into out_scale on the
// device -- the 2^-k of the backward's gradient exponent (launch_grad_exponent)
int launch_wgrad_finalize(const float* partial, int splits, int taps, int Cout, int Cin, const float* mult,
                          float out_scale, float* dw_ref, int accumulate, cudaStream_t s, const float* bias_partial = nullptr,
                          float* db = nullptr, int* flag = nullptr,     // flag: set to 1 when a summed partial is inf / NaN
                          const float* unscale = nullptr);

// ---- glue (simt_glue.cu) ------------------------------------------------------------------------
template <typename T> int launch_nchw_to_nhwc(const float* src, int F, int C, int H, int W, View dst, float scale, cudaStream_t s);
template <typename T> int launch_nhwc_to_nchw(View src, int F, float scale, float* dst, cudaStream_t s);
template <typename T> int launch_gpool_fwd(View src, int F, float* feat, cudaStream_t s);
// d(in) = dfeat / HW * scale * (scale_dev ? *scale_dev : 1)
template <typename T> int launch_gpool_bwd(const float* dfeat, float scale, const float* scale_dev, View ddst, int F, const void* y,
                                           cudaStream_t s);
// the backward's gradient exponent, one CTA: k such that max|dfeat| * grad_scale * 2^k / HW lies in [2^(GRAD_EXP_TOP-1),
// 2^GRAD_EXP_TOP) (k = 0 when dfeat is all zero; k = 0 and *flag = 1 when it holds an inf or NaN), |k| <= GRAD_EXP_MAX;
// writes gscale[0] = 2^k, gscale[1] = 2^-k.  [2^7, 2^8): the largest gradient plane of the SSN step is at most 43x the
// entry value on the H100 (tests/test_gpu_grad_range.py), so the planes stay 6x below the fp16 range
constexpr int GRAD_EXP_TOP = 8, GRAD_EXP_MAX = 100;
int launch_grad_exponent(const float* dfeat, long long n, float grad_scale, int HW, float* gscale, int* flag, cudaStream_t s);

// weight packing (simt_glue.cu), many layers per launch (block0 = first CTA of the entry; 256 threads per CTA): fold BN,
// produce the kernel layouts wf [tap][ci][co], wd [tap][co][ci] in storage type T; bias' [co] fp32; scale [co] fp32;
// absmax (optional, zeroed by the caller): max |folded weight|
constexpr int PACK_MAX = 32;
constexpr int PACK_PER_THREAD = 4;     // element-wise path of pack_all_kernel (more than PACK_TILE_TAPS taps: conv1): 256 threads x 4 elements per CTA
constexpr int PACK_TILE = 32, PACK_TILE_TAPS = 9;   // tiled path: one CTA per 32 output x 32 input channels x taps
inline int pack_ctas(int cout, int cin, int taps) {
  if (taps <= PACK_TILE_TAPS) return ((cout + PACK_TILE - 1) / PACK_TILE) * ((cin + PACK_TILE - 1) / PACK_TILE);
  const long long n = (long long)cout * cin * taps, per = 256LL * PACK_PER_THREAD;
  return (int)(((n > cout ? n : cout) + per - 1) / per);
}
struct PackEntry {
  const float *w, *b, *gamma, *beta, *mean, *var;
  void *wf, *wd; float *bias, *scale, *absmax;
  int cout, cin, taps, block0;  // taps = kh * kw, the trailing extent of the reference layout [cout][cin][kh][kw]
  int nofold, pad_[3];          // nofold: scale = 1, bias' = b (the layer's BatchNorm runs in training mode, unfused)
  float* bias_b;                // optional second copy of the folded bias (stacked bias of a fused sibling block)
};
struct PackTable { int n, pad_; PackEntry e[PACK_MAX]; };
template <typename T> int launch_pack_all(const PackTable& t, int total_blocks, cudaStream_t s);
// EXACT_TC: hi/lo planes of both fp32 weight layouts of many layers per launch, see launch_split_all
struct SplitEntry {
  const float *wf, *wd; __half *wf16, *wd16; long long plane_bytes, n; const float* absmax; float* inv_scale; int block0, pad_;
  // optional second copies inside a fused sibling block's operands (1x1 layers): wd rows stacked (contiguous), wf columns inside the
  // K-concatenated matrix [cin][b_pitch]; b_plane_bytes = distance to the LO plane of those buffers
  __half *wd16_b, *wf16_b; long long b_plane_bytes; int b_pitch, cout;
};
struct SplitTable { int n, pad_; SplitEntry e[PACK_MAX]; };
// every entry is split as src * 2^e with 2^e = 8192 / 2^ceil(log2(*absmax)): the largest weight lands in [4096, 8192), so
// the LO plane stays a normal fp16 number for every weight within ~2^-13 of the largest (unscaled, a BN-folded conv1 weight
// of ~1e-3 has a subnormal LO with 3 significant bits); thread 0 of the entry writes 2^-e to *inv_scale, the consuming
// kernels' alpha_dev
int launch_split_all(const SplitTable& t, int total_blocks, cudaStream_t s);

// one launch finalises the weight (and bias) gradients of many layers: split-K partial reduction in fixed order,
// BN-fold chain rule, 1/loss-scale, reference layout [co][ci][tap]
constexpr int FIN_MAX = 36;
struct FinalizeEntry {
  const float* partial; const float* mult; float* dw; const float* bias_partial; float* db;
  int splits, taps, Cout, Cin, block0, pad_;
};
struct FinalizeTable { int n, total_blocks; int* flag; const float* unscale; FinalizeEntry e[FIN_MAX]; };
int launch_wgrad_finalize_all(const FinalizeTable& t, float out_scale, int accumulate, cudaStream_t s);

// Vectorised pooling and mask glue (glue_vec.cu), T = float (SSNB_EXACT_FP32, SSNB_EXACT_TC) or __half (SSNB_FAST_FP16): every thread
// moves VEC_WIDTH<T> channels (16 bytes), so C, pitch and coff must be multiples of it.  `*planes` views (base == nullptr: none)
// receive the fp16 hi/lo operand planes; only the float launchers accept one.
template <typename T> constexpr int VEC_WIDTH = 16 / (int)sizeof(T);
template <typename T>
int launch_maxpool_fwd_vec(View src, View dst, View dst_planes, int F, int k, int stride, int pad, uint8_t* argmax, cudaStream_t s);   // k = 3
template <typename T>
int launch_maxpool_bwd_vec(View dsrc, View ddst, int F, int k, int stride, int pad, const uint8_t* argmax, int accumulate, cudaStream_t s);
template <typename T> int launch_avgpool3_vec(View src, View dst, View dst_planes, int F, int accumulate, cudaStream_t s);
// backward pass of a convolution's output gradient: dz = dy * (y > 0) (y.base == nullptr: no mask), bias-gradient column sums
// into db (nullptr: none), planes of dz * scale; dz is written back to dy where the mask changed it and write_back is set.
// partial must hold 64 + max_ctas * C floats (first 256 bytes: completion counter)
template <typename T>
int launch_mask_bias_vec(View dy, View y, View planes, float scale, int write_back, int* flag, int F, const float* mult, float out_scale,
                         const float* unscale, float* partial, int max_ctas, float* db, int accumulate, cudaStream_t s);
// the same pass for a convolution whose only consumer is a k3/s2/pad0 max pool, with that pool's backward gather folded in:
// dpool = gradient of the pool's output, argmax from its forward; dz is written whenever write_back is set
template <typename T>
int launch_pool_mask_bias_vec(View dz, View y, View dpool, View planes, float scale, int write_back, int* flag, int F, int k, int stride, int pad,
                              const uint8_t* argmax, const float* mult, float out_scale, const float* unscale, float* partial, int max_ctas,
                              float* db, int accumulate, cudaStream_t s);
// SSNB_EXACT_TC glue (tc_glue.cu): error-compensated fp16 operand planes of fp32 tensors.
//   hi = fp16(x * scale), lo = fp16(x * scale - float(hi))  =>  hi + lo carries ~22 significand bits of x * scale
// `flag` (device int, may be null) is set to 1 when |x * scale| exceeds the fp16 range (loss-scale overflow)
int launch_split_view(View src_f32, int F, float scale, View planes, int* flag, cudaStream_t s);
int launch_planes_to_nchw(View planes, int F, float scale, float* dst, cudaStream_t s);
// training-mode BatchNorm + ReLU of the first layer (bn_train.cu); stat: 4*C floats, partial: max_ctas * 2 * C floats
int launch_bn_train_fwd(View z, View y, View y_planes, int F, const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                        float* running_var, float* stat, float* partial, int max_ctas, cudaStream_t s);
int launch_bn_train_bwd(View z, View dy, View y, View dz, View dz_planes, float plane_scale, int* flag, int F, const float* gamma, float* stat,
                        float* partial, int max_ctas, float* dgamma, float* dbeta, const float* unscale, int accumulate, cudaStream_t s);
// tensor-core layout helpers (s2d_glue.cu).  conv1's packed space-to-depth operand from an NHWC view or NCHW fp32 frames:
// lo_off == 0 (FAST) writes fp16 values (the NHWC view holds fp16); lo_off != 0 (EXACT_TC) writes the hi plane at dst and
// the lo plane lo_off bytes after it (the NHWC view holds fp32)
int launch_nhwc_to_s2d(View src, int F, __half* dst, long long lo_off, int Cs, cudaStream_t s);
int launch_nchw_to_s2d(const float* src, int F, int Cin, int H, int W, __half* dst, long long lo_off, int Cs, cudaStream_t s);
int launch_pack_conv1_s2d(const __half* wd, int Cout, int Cin, int Cs, __half* ws, cudaStream_t s);
int launch_wgrad_finalize_s2d(const float* partial, int splits, int Cout, int Cin, int Cs, const float* mult, float out_scale,
                              const float* unscale, float* dw_ref, int accumulate, cudaStream_t s);
int launch_upsample2_zero(View src, __half* dst, int H, int W, int F, cudaStream_t s);

}  // namespace ssnb
