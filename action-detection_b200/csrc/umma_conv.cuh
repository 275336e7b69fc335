// wgmma (sm_90a) implicit-GEMM convolution for the tensor-core precisions -- interface.
//
// One kernel family computes   out[p, n] = epi( sum_taps sum_c  A[p + shift(tap), c] * B[tap][n][c] )
// over NHWC fp16 tensors: A tiles are 4-D TMA boxes of the activation view (zero-filled outside
// the image = free padding), B tiles are 3-D TMA boxes of the packed weights, accumulators live
// in the registers of two ping-pong consumer warpgroups, the epilogue fuses folded-BN bias + ReLU (forward)
// or accumulation (data gradient).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace ssnb {

constexpr int UMMA_MAX_TAPS = 25;         // a 5x5 kernel in one launch (InceptionV3)

struct UmmaContext {
  void* encode_tiled = nullptr;   // cuTensorMapEncodeTiled, resolved through cudaGetDriverEntryPoint
  int num_sms = 132;
};

struct UmmaConvParams {
  int W, H, F;                    // spatial dims shared by input and output (stride-1 convolutions); F: frames this launch computes
  int bw, bh, bf;                 // TMA box in pixels; bw*bh*bf <= 128 rows of the M tile
  int tiles_w, tiles_h, tiles_f;
  // first frame of the tiles whose epilogue stores row by row instead of by TMA: a launch of fewer frames than the output
  // maps were encoded for stores its last, partial frame box this way, so no row of a frame >= F is written (1 << 30: none)
  int f_direct;
  long long out_lo, out2_lo;      // byte distance of the LO operand plane from p.out / p.out2 (EXACT_TC planes, row-by-row stores)
  int n_tiles, block_n;           // N split of Cout into ceil(N/128) tiles; block_n is a multiple of 16, at most 128
  int stages, stage_bytes;        // smem pipeline depth / stride chosen from block_n
  int kchunks, ntaps, K;          // ceil(K/64), filter taps, reduction channels per tap
  int tap_dy[UMMA_MAX_TAPS], tap_dx[UMMA_MAX_TAPS];
  __half* out; int out_pitch, out_coff, Cout;
  int a_stride;                   // 2: tiles run at OUTPUT resolution and the A box uses TMA element stride 2
  const float* bias;              // [Cout] or nullptr
  int relu, accumulate;
  // horizontal fusion of sibling 1x1 convolutions (same input):
  int kchunks_a1, K1;             // K chunks [0, kchunks_a1) come from tmap_a (K1 real channels), the rest from tmap_a2
  int n_split;                    // output columns >= n_split go to out2 (second destination), else to out
  __half* out2; int out2_pitch, out2_coff;
  // stride 1, 1 / 4 / 9 taps, images at least 7 pixels wide, 32-byte aligned output rows: the plans whose tensor-core launch
  // the split-operand (EXACT_TC) schedule requires for conv1's forward, data gradients and fused launches (ssnb_set_workspace)
  int tc_ok;
  // data gradient that is the LAST writer of its output: fuse dz = dy * (y > 0), y = activation of the same value
  const __half* mask_y; int mask_pitch, mask_coff;
  // SSNB_EXACT_TC (error-compensated split operands): nseg = 3 stages the hi and lo planes of A and B of each (tap, K chunk)
  //   together and issues (A_lo, B_hi), (A_hi, B_lo), (A_hi, B_hi) into the same accumulator; nseg = 1 is the plain fp16 product.
  // out_f32: the epilogue works in fp32 -- out32 = alpha * acc (+ bias, ReLU | + old out32) -- and, when `planes` is set,
  // also writes the result's fp16 hi / lo operand planes (same pitch / channel offset; UmmaConvPlan::tmap_o_hi / _lo).
  int nseg, out_f32;
  float alpha;
  const float* alpha_dev;         // optional device scalar multiplied into alpha (1 / the power-of-two scale of the weight planes)
  float* out32; int planes;
  float* out32_2; int planes2;    // fused sibling forward: columns >= n_split go here (pitch / offset: out2_pitch / out2_coff)
  // out_f32 data gradient that is the LAST writer of its output value v: dz = (alpha * acc + old) * (y > 0) with y = the fp32
  // activation of v; the planes written through UmmaConvPlan::tmap_mask_hi / _lo then hold dz * plane_scale (the loss scale) for v's producers'
  // weight / data gradients, and *flag is raised when that leaves the fp16 range
  // (the global reads of the epilogue -- bias, old value, mask -- go through the pointers above; its stores through the
  // output tensor maps of UmmaConvPlan)
  const float* mask32; int mask32_pitch, mask32_coff;
  float plane_scale; int* flag;
};

struct UmmaConvPlan {
  bool enabled = false;
  const __half* mask_y = nullptr; int mask_pitch = 0, mask_coff = 0;   // applied only when launched with mask=true
  CUtensorMap tmap_a, tmap_a2, tmap_b;
  CUtensorMap tmap_a_lo, tmap_a2_lo, tmap_b_lo;   // SSNB_EXACT_TC: LO planes of the three operands (copies of the HI maps otherwise)
  long long b_lo_off = 0;                        // byte offset of the LO weight plane (0: single plane)
  // epilogue stores, 4-D boxes [bf][bh][bw][16 columns] of the output: the fp32 result (EXACT_TC, SWIZZLE_64B) or the fp16
  // result (FAST, SWIZZLE_32B), then the fp16 hi / lo operand planes (EXACT_TC, SWIZZLE_32B).  The *2 maps serve columns
  // >= n_split of a fused sibling forward.  dims[0] of each map is its destination's channel count, so TMA clips a tile
  // overhanging N or the image instead of writing past it.  Maps a plan does not use are copies of tmap_o.
  CUtensorMap tmap_o, tmap_o_hi, tmap_o_lo, tmap_o2, tmap_o2_hi, tmap_o2_lo;
  // SSNB_EXACT_TC mask fusion, applied only when launched with mask=true (see UmmaConvParams::mask32); the gradient planes
  // it writes replace tmap_o_hi / tmap_o_lo
  const float* mask32 = nullptr; int mask32_pitch = 0, mask32_coff = 0;
  CUtensorMap tmap_mask_hi, tmap_mask_lo; bool mask_planes = false; float mask_plane_scale = 1.0f; int* mask_flag = nullptr;
  UmmaConvParams p;
};

// SSNB_EXACT_TC binding options: split weights (LO plane `w_lo_off` bytes after the HI plane), fp32 output view `out32`
// (the bind call's own out/dx view then names the fp16 HI plane of the result, lo_off its LO plane; base == nullptr: no
// planes are written), accumulator scale alpha
struct UmmaTcOpts { long long w_lo_off = 0; float* out32 = nullptr; float alpha = 1.0f; const float* alpha_dev = nullptr; float* out32_2 = nullptr; };
void umma_context_init(UmmaContext& ctx);
void umma_context_destroy(UmmaContext& ctx);
// forward convolution plan (stride 1): in/out views, weights wd = [tap][cout][cin] fp16
int umma_conv_bind_fwd(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out, int F, int cin, int cout, int k, int pad,
                       int stride, const __half* w_tap_n_k, const float* bias, const UmmaTcOpts* tc = nullptr);
// generic tap table variant (BNInception's conv1 in space-to-depth form: 4 taps over the packed input; InceptionV3's
// kh x kw layers).  Tiles run at the output's geometry; the A map keeps the input's dims, so an output smaller than the input
// (valid padding) reads in[out * stride + (dy, dx)] with TMA zero fill outside the image.  stride: 1 or 2
int umma_conv_bind_taps(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out, int F, int cin, int cout, int ntaps,
                        const int* dy, const int* dx, const __half* w_tap_n_k, const float* bias, int relu, const UmmaTcOpts* tc = nullptr,
                        int stride = 1);
// data-gradient plan (stride 1): dz/dx gradient views, weights wf = [tap][cin][cout] fp16
int umma_conv_bind_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz, View dx, int F, int cin, int cout, int k, int pad,
                         const __half* w_tap_k_n, int accumulate, const UmmaTcOpts* tc = nullptr);
// fused forward of sibling 1x1 convs: one input view, weights [n1+n2][cin] (rows stacked), columns [0,n1) -> out1, rest -> out2
int umma_conv_bind_fused_fwd(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out1, View out2, int F, int cin, int n1, int n2,
                             const __half* w_n_k, const float* bias, const UmmaTcOpts* tc = nullptr);
// fused data gradient of sibling 1x1 convs: dx (+)= [dz1 | dz2] * W, weights [cin][pad64(k1) + k2]; dz1 may be empty (k1 = 0)
int umma_conv_bind_fused_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz1, View dz2, View dx, int F, int cin, int k1, int k2,
                               const __half* w_n_k, int accumulate, const UmmaTcOpts* tc = nullptr);
// frames = 0: the plan's frame count; 1 .. F (forward plans, mask = false): the first `frames` frames only, with that many
// frames' tiles, the maps as bound and no store to a frame >= frames
int umma_conv_launch(UmmaContext& ctx, const UmmaConvPlan& plan, cudaStream_t s, bool mask = false, int frames = 0);
void umma_conv_set_mask(UmmaConvPlan& plan, View y);
// EXACT_TC: y32 = fp32 activation of the output value, dplanes = that value's gradient operand planes (hi base + lo_off)
int umma_conv_set_mask_tc(UmmaContext& ctx, UmmaConvPlan& plan, View y32, View dplanes, float plane_scale, int* flag);

// host helpers shared by the tensor-core kernels
int umma_resolve_encode(UmmaContext& ctx);
int umma_encode_f16(UmmaContext& ctx, CUtensorMap* m, int rank, void* addr, const cuuint64_t* dims,
                    const cuuint64_t* strides, const cuuint32_t* box, int spatial_stride = 1);

// ---- weight gradient on wgmma (umma_wgrad.cu) ---------------------------------------------------------
// partial[split][tap][co][ci] = sum over the split's pixels of dz[p, co] * x[p + (r-pad, s-pad), ci]
// (both operands MN-major: the reduction dimension is the pixel index).
struct UmmaWgradParams {
  int W, H, F;
  int bw, bh, bf;                 // 64-pixel TMA box
  int tiles_w, tiles_h, tiles_f;
  int ptiles_per_split, splits;
  int ntaps, tap_dy[UMMA_MAX_TAPS], tap_dx[UMMA_MAX_TAPS];
  int Cout, Cin, m_tiles, n_tiles, block_n;
  int x_stride;                   // 2: stride-2 layers, the x box steps over the input with TMA element stride 2
  float* bias_partial;            // [split][Cout] column sums of dz (bias gradient) from an extra ones-operand MMA, or nullptr
  int taps_per_cta, tap_groups;   // taps sharing one dz tile per CTA (taps_per_cta * block_n <= 256 accumulator columns)
  int stages, stage_bytes;        // pipeline depth / stride
  float* partial;
  int nseg;                       // 3: SSNB_EXACT_TC, a stage holds the hi and lo planes of dz and x and the consumer issues
                                  //    (dz_lo, x_hi), (dz_hi, x_lo), (dz_hi, x_hi) from it; 1: the plain fp16 product
  int sub_dh, sub_df;             // EXACT_TC stages half a pixel tile: the second half starts sub_dh rows / sub_df frames on
};
struct UmmaWgradPlan {
  bool enabled = false;
  CUtensorMap tmap_dz, tmap_x;
  CUtensorMap tmap_dz_lo, tmap_x_lo;              // SSNB_EXACT_TC: LO planes (View::lo_off of the bound views)
  UmmaWgradParams p;
};
// Longest pixel range of one split, in 64-pixel tiles.  A split sums its pixels in the wgmma's fp32 accumulators, whose error
// grows in proportion to the number of tiles summed: EXACT_TC's dW rel-L2 is about 1.6e-7 per tile (H100: conv2_3x3 1.1e-4 at
// 642 tiles, 2.1e-4 at 1283; conv1 of Flow 2.1e-4 / 9.9e-5 / 6.3e-5 at 1711 / 856 / 571), so 768 keeps it near 1.3e-4.
constexpr int UMMA_WGRAD_MAX_PTILES = 768;
// pixel tiles of a weight gradient over a W x H x F dz (the box is chosen by W)
int umma_wgrad_ptiles(int W, int H, int F);
// split count before the caps of the bind (max_splits, the pixel tile count): `waves` waves of ctas-CTA splits (num_sms / ctas
// per wave, at least 1), and as many more whole waves as keep every split at most UMMA_WGRAD_MAX_PTILES tiles long
int umma_wgrad_splits(int ctas, int ptiles, int num_sms, int waves = 1);
// returns the number of splits chosen through *splits (the caller sizes `partial` from it)
int umma_wgrad_bind(UmmaContext& ctx, UmmaWgradPlan& plan, View dz, View x, int F, int cin, int cout, int k, int pad,
                    float* partial, int max_splits, int x_stride = 1);
int umma_wgrad_bind_taps(UmmaContext& ctx, UmmaWgradPlan& plan, View dz, View x, int F, int cin, int cout, int ntaps,
                         const int* dy, const int* dx, float* partial, int max_splits, int x_stride = 1);
int umma_wgrad_launch(UmmaContext& ctx, const UmmaWgradPlan& plan, cudaStream_t s, float* bias_partial = nullptr);

}  // namespace ssnb
