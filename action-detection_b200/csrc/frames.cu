// Frame transforms on the GPU: the reference's PIL group transforms (transforms.py:41-206) followed by Stack(roll=True),
// ToTorchFormatTensor(div=False) and GroupNormalize, for many groups of uint8 frames of different sizes in one call.
//
// Every value matches PIL bit for bit.  Image.resize(BILINEAR) on 8-bit bands (libImaging/Resample.c) is fixed-point
// arithmetic: per output index the filter weights are computed in double, normalised by their sum and rounded to ints with
// 22 fraction bits; the horizontal pass then the vertical pass each compute (sum px * k + 2^21) >> 22, clipped to [0, 255],
// into a uint8 intermediate.  The weights are computed here on the device with explicitly rounded double operations (no
// FMA contraction), so the call needs no host-side tables and can be captured in a CUDA graph.  An axis whose size does not
// change gets the single weight 2^22, which is the copy PIL makes when it skips that pass.
//
//   frames_scale_kernel  GroupScale (torchvision Resize of the shorter edge) of OVERSAMPLE / CENTER images whose shorter
//                        edge is not already scale_size, into uint8 HWC scratch in the workspace
//   frames_out_kernel    one CTA per (image, window, band of TR output rows, TX output columns): the window of the source
//                        (or scaled) image, zero outside it as PIL's crop fills, resized to out_size x out_size; flip, Flow
//                        inversion, the RGB -> BGR roll and normalisation on the way out to planar fp32.  OVERSAMPLE's plain
//                        and flipped crops of one window come from the same CTA; the five windows overlap but are read by
//                        separate CTAs (the second read of a pixel mostly hits L2, and the fp32 stores bound the call)
#include <algorithm>
#include <climits>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

// TX x TR output pixels per CTA; KMAX weights per output index (2 * ceil(support) + 1 for a scale factor up to
// kMaxScale); CAP intermediate rows staged in shared memory at a time (>= KMAX, so one output row always fits)
constexpr int TX = 112, TR = 16, kMaxScale = 16, KMAX = 2 * kMaxScale + 1, CAP = 80, kThreads = 256;
constexpr int kMaxMean = 8, kMaxSide = 16384;
constexpr int PREC = 22;

struct FrameParams {
  int mode, C, out, scale_size, invert_even, n_mean, n_groups;
  float mean[kMaxMean], stdv[kMaxMean];
};

__host__ __device__ inline int crops_of(int mode) { return mode == SSNB_FRAMES_OVERSAMPLE ? 10 : 1; }
// output windows per image: OVERSAMPLE's five fill_fix_offset windows (each written plain and flipped), else one
__host__ __device__ inline int windows_of(int mode) { return mode == SSNB_FRAMES_OVERSAMPLE ? 5 : 1; }

// torchvision Resize(size) of the shorter edge: long = int(size * long / short); the identity when short == size
__host__ __device__ inline void scaled_dims(int H, int W, int S, int& sh, int& sw) {
  const bool w_short = W <= H;
  const int sht = w_short ? W : H, lng = w_short ? H : W;
  const int nl = (int)((double)((long long)S * lng) / (double)sht);
  sh = w_short ? nl : S;
  sw = w_short ? S : nl;
}

__device__ __forceinline__ double tri(double x) {
  if (x < 0.0) x = -x;
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// PIL's precompute_coeffs + normalize_coeffs_8bpc for output index o of an in -> out axis
__device__ void pil_coeffs(int in, int out, int o, int* lo, int* n, int* k) {
  if (in == out) { *lo = o; *n = 1; k[0] = 1 << PREC; return; }
  const double scale = __ddiv_rn((double)in, (double)out);
  const double fs = scale < 1.0 ? 1.0 : scale;        // filterscale; support = 1.0 * filterscale
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn((double)o, 0.5), scale);
  int xmin = (int)__dadd_rn(__dsub_rn(center, fs), 0.5);
  int xmax = (int)__dadd_rn(__dadd_rn(center, fs), 0.5);
  if (xmin < 0) xmin = 0;
  if (xmax > in) xmax = in;
  const int cnt = min(max(xmax - xmin, 0), KMAX);
  double ww = 0.0;
  for (int j = 0; j < cnt; ++j) ww = __dadd_rn(ww, tri(__dmul_rn(__dadd_rn(__dsub_rn((double)(j + xmin), center), 0.5), ss)));
  for (int j = 0; j < cnt; ++j) {
    double w = tri(__dmul_rn(__dadd_rn(__dsub_rn((double)(j + xmin), center), 0.5), ss));
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    k[j] = (int)__dadd_rn(0.5, __dmul_rn(w, (double)(1 << PREC)));
  }
  *lo = xmin;
  *n = cnt;
}

__device__ __forceinline__ int clip8(int v) {
  if (v >= (1 << PREC << 8)) return 255;
  if (v <= 0) return 0;
  return v >> PREC;
}

// the group owning global image index img (first_image ascending)
__device__ __forceinline__ int group_of(const ssnb_frame_group* __restrict__ g, int n, int img) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (g[mid].first_image <= img) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct Smem {
  int hk[TX][KMAX], hlo[TX], hn[TX];
  int vk[TR][KMAX], vlo[TR], vn[TR];
  uint8_t inter[CAP * TX * 3];
};

// Resize the window (wx0, wy0, ww, wh) of img [H, W, C] to ow x oh and hand the output tile at (tx0, ty0) to store(x, y, c, v).
// Uniform across the CTA (every thread calls it with the same arguments).
template <int C, class Store>
__device__ void resample_tile(Smem& sm, const uint8_t* __restrict__ img, int H, int W, int wx0, int wy0, int ww, int wh, int ow, int oh,
                              int tx0, int ty0, const Store& store) {
  const int t = threadIdx.x;
  const int nx = min(TX, ow - tx0), nr = min(TR, oh - ty0);
  if (t < nx) pil_coeffs(ww, ow, tx0 + t, &sm.hlo[t], &sm.hn[t], sm.hk[t]);
  else if (t >= TX && t - TX < nr) pil_coeffs(wh, oh, ty0 + t - TX, &sm.vlo[t - TX], &sm.vn[t - TX], sm.vk[t - TX]);
  __syncthreads();
  for (int r = 0; r < nr;) {
    // output rows r .. re-1 whose source rows fit the staging buffer (both bounds are non-decreasing in the row)
    const int ylo = sm.vlo[r];
    int re = r + 1;
    while (re < nr && sm.vlo[re] + sm.vn[re] - ylo <= CAP) ++re;
    const int rows = sm.vlo[re - 1] + sm.vn[re - 1] - ylo;
    for (int i = t; i < rows * nx; i += blockDim.x) {
      const int row = i / nx, xi = i - row * nx;
      const int sy = wy0 + ylo + row;
      const bool yin = sy >= 0 && sy < H;
      const int x0 = wx0 + sm.hlo[xi], n = sm.hn[xi];
      int acc[C];
      for (int c = 0; c < C; ++c) acc[c] = 1 << (PREC - 1);
      if (yin) {
        const uint8_t* rowp = img + (long long)sy * W * C;
        for (int j = 0; j < n; ++j) {
          const int sx = x0 + j;
          if (sx < 0 || sx >= W) continue;
          const int k = sm.hk[xi][j];
          for (int c = 0; c < C; ++c) acc[c] += (int)rowp[sx * C + c] * k;
        }
      }
      for (int c = 0; c < C; ++c) sm.inter[(row * TX + xi) * C + c] = (uint8_t)clip8(acc[c]);
    }
    __syncthreads();
    for (int i = t; i < (re - r) * nx; i += blockDim.x) {
      const int rr = r + i / nx, xi = i % nx;
      const int y0 = sm.vlo[rr] - ylo, n = sm.vn[rr];
      int acc[C];
      for (int c = 0; c < C; ++c) acc[c] = 1 << (PREC - 1);
      for (int j = 0; j < n; ++j) {
        const int k = sm.vk[rr][j];
        for (int c = 0; c < C; ++c) acc[c] += (int)sm.inter[((y0 + j) * TX + xi) * C + c] * k;
      }
      for (int c = 0; c < C; ++c) store(tx0 + xi, ty0 + rr, c, clip8(acc[c]));
    }
    __syncthreads();
    r = re;
  }
}

template <int C>
__global__ void __launch_bounds__(kThreads) frames_scale_kernel(const uint8_t* __restrict__ src, const ssnb_frame_group* __restrict__ groups,
                                                                 FrameParams p, uint8_t* __restrict__ ws) {
  __shared__ Smem sm;
  const int img = blockIdx.x;
  const ssnb_frame_group g = groups[group_of(groups, p.n_groups, img)];
  const int i = img - g.first_image;
  if (i < 0 || i >= g.images) return;
  int sh, sw;
  scaled_dims(g.height, g.width, p.scale_size, sh, sw);
  if (sh == g.height && sw == g.width) return;
  const uint8_t* in = src + g.src_offset + (long long)i * g.height * g.width * C;
  uint8_t* out = ws + g.scratch_offset + (long long)i * sh * sw * C;
  const auto store = [&](int x, int y, int c, int v) { out[((long long)y * sw + x) * C + c] = (uint8_t)v; };
  for (int ty = blockIdx.y * TR; ty < sh; ty += gridDim.y * TR)
    for (int tx = blockIdx.z * TX; tx < sw; tx += gridDim.z * TX)
      resample_tile<C>(sm, in, g.height, g.width, 0, 0, g.width, g.height, sw, sh, tx, ty, store);
}

template <int C>
__global__ void __launch_bounds__(kThreads) frames_out_kernel(const uint8_t* __restrict__ src, const ssnb_frame_group* __restrict__ groups,
                                                               FrameParams p, const uint8_t* __restrict__ ws, float* __restrict__ dst) {
  __shared__ Smem sm;
  const int wins = windows_of(p.mode);
  const int img = blockIdx.x / wins, o = blockIdx.x % wins;
  const ssnb_frame_group g = groups[group_of(groups, p.n_groups, img)];
  const int i = img - g.first_image;
  if (i < 0 || i >= g.images) return;
  const int S = p.out;
  const uint8_t* in = src + g.src_offset + (long long)i * g.height * g.width * C;
  int H = g.height, W = g.width, wx0, wy0, ww = S, wh = S, flip = 0;
  if (p.mode == SSNB_FRAMES_TRAIN) {
    wx0 = g.crop_x; wy0 = g.crop_y; ww = g.crop_w; wh = g.crop_h; flip = g.flip != 0;
  } else {
    int sh, sw;
    scaled_dims(H, W, p.scale_size, sh, sw);
    if (sh != H || sw != W) { in = ws + g.scratch_offset + (long long)i * sh * sw * C; H = sh; W = sw; }
    if (p.mode == SSNB_FRAMES_CENTER) {       // torchvision center_crop: int(round((h - th) / 2.0)), half to even
      wx0 = (int)rint((double)(W - S) / 2.0);
      wy0 = (int)rint((double)(H - S) / 2.0);
    } else {                                  // fill_fix_offset(False, ...) window o
      const int ws_ = (int)floor((double)(W - S) / 4.0), hs_ = (int)floor((double)(H - S) / 4.0);
      wx0 = (o == 1 || o == 3) ? 4 * ws_ : (o == 4 ? 2 * ws_ : 0);
      wy0 = (o == 2 || o == 3) ? 4 * hs_ : (o == 4 ? 2 * hs_ : 0);
    }
  }
  // OVERSAMPLE: crop 2o (plain) and crop 2o + 1 (flipped) share every pixel, so one CTA writes both
  const bool both = p.mode == SSNB_FRAMES_OVERSAMPLE;
  const int k0 = both ? 2 * o : 0;
  const bool inv_flipped = p.invert_even && (i % 2 == 0);
  float* out = dst + g.dst_offset;
  const long long area = (long long)S * S;
  const auto put = [&](int k, bool fl, int x, int y, int co, int v) {
    const long long pl = ((long long)k * g.images + i) * C + co;
    const int m = (int)(pl % p.n_mean);
    const float f = __fdiv_rn(__fsub_rn((float)(fl && inv_flipped ? 255 - v : v), p.mean[m]), p.stdv[m]);
    out[pl * area + (long long)y * S + (fl ? S - 1 - x : x)] = f;
  };
  const auto store = [&](int x, int y, int c, int v) {
    const int co = C == 3 ? 2 - c : c;        // Stack(roll=True): RGB -> BGR
    put(k0, flip, x, y, co, v);
    if (both) put(k0 + 1, true, x, y, co, v);
  };
  resample_tile<C>(sm, in, H, W, wx0, wy0, ww, wh, S, S, blockIdx.z * TX, blockIdx.y * TR, store);
}

int cdiv(long long a, int b) { return (int)((a + b - 1) / b); }

// host-side validation and layout (first_image, dst_offset, scratch_offset) of the groups
const char* frames_layout(const ssnb_frame_cfg* cfg, const ssnb_frame_group* g, int n, std::vector<ssnb_frame_group>& lay,
                          size_t& ws_bytes, int64_t& dst_floats, int& max_sh, int& max_sw) {
  if (!cfg || !g) return "NULL cfg or groups";
  if (cfg->mode != SSNB_FRAMES_TRAIN && cfg->mode != SSNB_FRAMES_OVERSAMPLE && cfg->mode != SSNB_FRAMES_CENTER) return "unknown mode";
  if (cfg->channels != 1 && cfg->channels != 3) return "channels must be 1 (L) or 3 (RGB)";
  if (cfg->out_size < 1 || cfg->out_size > 1024) return "out_size must be in 1..1024";
  if (cfg->mode != SSNB_FRAMES_TRAIN && (cfg->scale_size < cfg->out_size || cfg->scale_size > 4096))
    return "scale_size must be in out_size..4096";
  if (cfg->n_mean < 1 || cfg->n_mean > kMaxMean) return "n_mean must be in 1..8";
  if (n < 1) return "no group";
  const int C = cfg->channels, S = cfg->out_size, crops = crops_of(cfg->mode);
  lay.assign(g, g + n);
  long long img = 0, dst = 0, ws = 0;
  max_sh = max_sw = 0;
  for (int j = 0; j < n; ++j) {
    ssnb_frame_group& e = lay[j];
    if (e.height < 1 || e.width < 1 || e.height > kMaxSide || e.width > kMaxSide) return "height / width outside 1..16384";
    if (e.images < 1) return "a group without images";
    if (((long long)e.images * C) % cfg->n_mean) return "a group's stacked channels are not a multiple of n_mean";
    if (e.src_offset < 0) return "negative src_offset";
    if (cfg->mode == SSNB_FRAMES_TRAIN) {
      if (e.crop_w < 1 || e.crop_h < 1) return "empty crop window";
      if (e.crop_w > kMaxScale * S || e.crop_h > kMaxScale * S) return "crop window more than 16x the output size";
      if (std::abs((long long)e.crop_x) > kMaxSide || std::abs((long long)e.crop_y) > kMaxSide) return "crop offset outside +-16384";
    } else {
      int sh, sw;
      scaled_dims(e.height, e.width, cfg->scale_size, sh, sw);
      if (sh < 1 || sw < 1 || sh > kMaxSide || sw > kMaxSide) return "scaled size outside 1..16384";
      if (e.height > kMaxScale * sh || e.width > kMaxScale * sw) return "source more than 16x the scaled size";
      e.scratch_offset = 0;
      if (sh != e.height || sw != e.width) {
        e.scratch_offset = ws;
        ws += ((long long)e.images * sh * sw * C + 255) & ~255LL;
        max_sh = std::max(max_sh, sh);
        max_sw = std::max(max_sw, sw);
      }
    }
    e.first_image = (int32_t)img;
    e.dst_offset = dst;
    img += e.images;
    dst += (long long)crops * e.images * C * S * S;
    if (img * crops > INT_MAX) return "more than INT_MAX output images";
  }
  ws_bytes = (size_t)ws;
  dst_floats = dst;
  return nullptr;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_frame_transform_workspace_bytes(const ssnb_frame_cfg* cfg, ssnb_frame_group* groups, int n_groups, size_t* workspace_bytes,
                                         int64_t* dst_floats) {
  std::vector<ssnb_frame_group> lay;
  size_t ws = 0;
  int64_t nd = 0;
  int mh, mw;
  if (const char* bad = frames_layout(cfg, groups, n_groups, lay, ws, nd, mh, mw)) {
    set_thread_error(std::string("frame_transform: ") + bad);
    return SSNB_EINVAL;
  }
  std::copy(lay.begin(), lay.end(), groups);
  if (workspace_bytes) *workspace_bytes = ws;
  if (dst_floats) *dst_floats = nd;
  return SSNB_OK;
}

int ssnb_frame_transform(const ssnb_frame_cfg* cfg, const ssnb_frame_group* groups, const ssnb_frame_group* groups_dev, int n_groups,
                         const uint8_t* src, size_t src_bytes, float* dst, int64_t dst_floats, void* workspace, size_t workspace_bytes,
                         void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("frame_transform: " + m); return (int)SSNB_EINVAL; };
  std::vector<ssnb_frame_group> lay;
  size_t ws = 0;
  int64_t nd = 0;
  int max_sh, max_sw;
  if (const char* bad = frames_layout(cfg, groups, n_groups, lay, ws, nd, max_sh, max_sw)) return fail(bad);
  if (!groups_dev || !src || !dst) return fail("NULL groups_dev, src or dst");
  const int C = cfg->channels;
  long long images = 0;
  for (int j = 0; j < n_groups; ++j) {
    const ssnb_frame_group &e = groups[j], &l = lay[j];
    if (e.first_image != l.first_image || e.dst_offset != l.dst_offset || e.scratch_offset != l.scratch_offset)
      return fail("first_image / dst_offset / scratch_offset differ from ssnb_frame_transform_workspace_bytes' layout");
    if ((unsigned long long)e.src_offset + (unsigned long long)e.images * e.height * e.width * C > src_bytes) return fail("a group reads past src_bytes");
    images += e.images;
  }
  if (dst_floats < nd) return fail("dst holds fewer floats than the groups write");
  if (workspace_bytes < ws || (ws > 0 && !workspace)) return fail("workspace too small (ssnb_frame_transform_workspace_bytes)");
  FrameParams p{};
  p.mode = cfg->mode; p.C = C; p.out = cfg->out_size; p.scale_size = cfg->scale_size; p.n_groups = n_groups;
  p.invert_even = cfg->invert_even != 0; p.n_mean = cfg->n_mean;
  for (int m = 0; m < cfg->n_mean; ++m) { p.mean[m] = cfg->mean[m]; p.stdv[m] = cfg->std[m]; }
  if (ws > 0) {
    const dim3 grid((unsigned)images, cdiv(max_sh, TR), cdiv(max_sw, TX));
    if (C == 3) frames_scale_kernel<3><<<grid, kThreads, 0, s>>>(src, groups_dev, p, (uint8_t*)workspace);
    else frames_scale_kernel<1><<<grid, kThreads, 0, s>>>(src, groups_dev, p, (uint8_t*)workspace);
    SSNB_LAUNCH_CHECK("frames_scale_kernel");
  }
  const dim3 grid((unsigned)(images * windows_of(p.mode)), cdiv(p.out, TR), cdiv(p.out, TX));
  if (C == 3) frames_out_kernel<3><<<grid, kThreads, 0, s>>>(src, groups_dev, p, (const uint8_t*)workspace, dst);
  else frames_out_kernel<1><<<grid, kThreads, 0, s>>>(src, groups_dev, p, (const uint8_t*)workspace, dst);
  SSNB_LAUNCH_CHECK("frames_out_kernel");
  return SSNB_OK;
}

}  // extern "C"
