// Frame resize on the GPU: DenseFlow's cv::resize(frame, image, Size(new_width, new_height)) of every decoded frame before
// the grey conversion, the flow and imwrite (extract_gpu --new_width 340 --new_height 256), bitwise equal to OpenCV 4's
// cv2.resize(frame, (dst_w, dst_h), interpolation=cv2.INTER_LINEAR) on uint8 3-channel frames.  The rules are the ones
// oracle/frame_resize_oracle.py restates from resize.cpp (hal::resize, resizeGeneric_, HResizeLinear, VResizeLinearVec_32s8u):
//
//   coefficients  scale = 1 / (dst / src) in double; f = float((d + 0.5) * scale - 0.5), the product and the difference each
//                 rounded once (no FMA); s = floor(f), f -= s; weights saturate_cast<short>((1 - f) * 2048) and
//                 saturate_cast<short>(f * 2048), both rounded half to even.
//   columns       s < 0 becomes s = 0, f = 0, and s >= W - 1 becomes s = W - 1, f = 0 (the column taps are clamped).
//   rows          the row taps s, s + 1 are clipped to 0 .. H - 1 but the row weights are NOT reset: above the first and
//                 below the last source row both taps read the same row with weights that still sum to 2048.
//   horizontal    h = S[s] * a0 + S[s + 1] * a1 in int32 (exact).
//   vertical      OpenCV's vector rounding, used for every element: ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16),
//                 then (v + 2) >> 2 saturated to 0 .. 255.  The scalar rule (h0 b0 + h1 b1 + 2^21) >> 22 differs from it
//                 in about one value in eight, and cv2 4.13 does not use it for any element of a 3-channel uint8 row.
//   special cases cv::resize copies a frame of the destination size, and hal::resize sends an exact 2 x 2 downscale to the
//                 area fast path ((a + b + c + d + 2) >> 2).  Both equal the rules above bit for bit (weights 2048 / 0 and
//                 1024 / 1024), so the kernel has no separate path for them; the oracle takes OpenCV's paths and its tests
//                 check the equality.
//
// This is not frames.cu's resize (PIL's resample: a different support, float coefficients normalised per pixel and
// 22-bit rounding) nor optical_flow.cu's pyramid resize (fp32 planes); neither computes OpenCV's fixed-point uint8 rule.
// cv2 4.13 is the yardstick.  DenseFlow builds link OpenCV 2.4, whose vertical pass may round a row's last few values with
// the scalar rule; parity with that build is not checked by this project.
//
// One thread per output pixel (its three channels), a CTA a 32 x 32 tile of one output frame: 32 x 8 threads, 4 rows each,
// so a warp writes 96 contiguous bytes per row.  The tile's 32 column and 32 row coefficients are derived from the shapes
// by one thread each into shared memory (the double-precision divisions are the costly part), so there is no table in
// global memory and no workspace.  The grid is (tiles of the destination, frames); a CTA finds its
// frame's video by binary search in the device table.  Every frame has the destination's tile count, so no CTA idles, the
// grid is a function of host shapes only, and a call can be captured in a CUDA graph; a frame's output depends on its own
// pixels and its video's size only.
#include <algorithm>
#include <string>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int kTx = 32, kTy = 8, kRows = 4, kTileH = kTy * kRows;  // a CTA's tile: 32 x 32 output pixels
constexpr int kMaxFramesPerLaunch = 65535;                          // gridDim.y
constexpr int kMaxSide = 65500;

// resize.cpp's per-axis coordinate of destination index d: the tap s and its fraction f, in OpenCV's float / double mix
__device__ __forceinline__ float source_coord(int d, int src, int dst, int& s) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
  const float f = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
  const float fl = floorf(f);
  s = (int)fl;
  return __fsub_rn(f, fl);
}

// saturate_cast<short>(w * INTER_RESIZE_COEF_SCALE) of both taps; lrint rounds half to even, as __float2int_rn does
__device__ __forceinline__ void weights(float f, int& w0, int& w1) {
  w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  w1 = __float2int_rn(__fmul_rn(f, 2048.f));
}

__global__ void __launch_bounds__(kTx * kTy) resize_kernel(const ssnb_resize_video* __restrict__ videos, int n_videos, int64_t frame0,
                                                            int tiles_x, int dst_h, int dst_w, const uint8_t* __restrict__ src,
                                                            uint8_t* __restrict__ dst) {
  __shared__ int col_x0[kTx], col_x1[kTx], col_w[kTx];          // byte offsets of the two column taps, weights a0 | a1 << 16
  __shared__ int row_y0[kTileH], row_y1[kTileH], row_w[kTileH];  // the two row taps (clipped rows), weights b0 | b1 << 16
  const int64_t frame = frame0 + blockIdx.y;
  int lo = 0, hi = n_videos - 1;                     // the last video whose first frame is at or before this one
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (videos[mid].first_frame <= frame) lo = mid;
    else hi = mid - 1;
  }
  const int H = videos[lo].height, W = videos[lo].width;
  const int tx0 = (int)(blockIdx.x % tiles_x) * kTx, ty0 = (int)(blockIdx.x / tiles_x) * kTileH;
  const int t = threadIdx.y * kTx + threadIdx.x;
  if (t < kTx) {                                     // the tile's column coefficients, one thread each
    int sx, a0, a1;
    float fx = source_coord(tx0 + t, W, dst_w, sx);
    if (sx < 0) sx = 0, fx = 0.f;
    if (sx >= W - 1) sx = W - 1, fx = 0.f;
    weights(fx, a0, a1);
    col_x0[t] = sx * 3;
    col_x1[t] = min(sx + 1, W - 1) * 3;
    col_w[t] = a0 | a1 << 16;
  } else if (t < kTx + kTileH) {                     // its row coefficients
    const int i = t - kTx;
    int sy, b0, b1;
    weights(source_coord(ty0 + i, H, dst_h, sy), b0, b1);
    row_y0[i] = min(max(sy, 0), H - 1);
    row_y1[i] = min(max(sy + 1, 0), H - 1);
    row_w[i] = b0 | b1 << 16;
  }
  __syncthreads();
  const int dx = tx0 + threadIdx.x;
  if (dx >= dst_w) return;
  const int x0 = col_x0[threadIdx.x], x1 = col_x1[threadIdx.x];
  const int a0 = col_w[threadIdx.x] & 0xffff, a1 = col_w[threadIdx.x] >> 16;
  const uint8_t* __restrict__ f = src + videos[lo].src_offset + (frame - videos[lo].first_frame) * H * W * 3;
  uint8_t* __restrict__ o = dst + (frame * dst_h * dst_w + dx) * 3;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int i = threadIdx.y + r * kTy;
    if (ty0 + i >= dst_h) break;
    const int b0 = row_w[i] & 0xffff, b1 = row_w[i] >> 16;
    const uint8_t* __restrict__ r0 = f + (int64_t)row_y0[i] * W * 3;
    const uint8_t* __restrict__ r1 = f + (int64_t)row_y1[i] * W * 3;
    uint8_t* __restrict__ out = o + (int64_t)(ty0 + i) * dst_w * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = __ldg(r0 + x0 + c) * a0 + __ldg(r0 + x1 + c) * a1;
      const int h1 = __ldg(r1 + x0 + c) * a0 + __ldg(r1 + x1 + c) * a1;
      const int v = ((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16)) + 2) >> 2;
      out[c] = (uint8_t)min(v, 255);
    }
  }
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_frame_resize(const uint8_t* src, int64_t src_bytes, const ssnb_resize_video* videos, const ssnb_resize_video* videos_dev,
                      int n_videos, int dst_height, int dst_width, uint8_t* dst, int64_t dst_bytes, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("frame_resize: " + m); return (int)SSNB_EINVAL; };
  if (n_videos < 1 || !videos) return fail("no video, or NULL videos");
  if (dst_height < 1 || dst_width < 1 || dst_height > kMaxSide || dst_width > kMaxSide)
    return fail("destination height and width must be 1 .. " + std::to_string(kMaxSide));
  int64_t frames = 0;
  for (int v = 0; v < n_videos; ++v) {
    const ssnb_resize_video& e = videos[v];
    const std::string name = "video " + std::to_string(v) + ": ";
    if (e.height < 1 || e.width < 1 || e.height > kMaxSide || e.width > kMaxSide)
      return fail(name + "height and width must be 1 .. " + std::to_string(kMaxSide));
    if (e.frames < 1) return fail(name + "frames must be >= 1");
    if (e.first_frame != frames) return fail(name + "first_frame must be the frames of the videos before it (" + std::to_string(frames) + ")");
    const int64_t bytes = (int64_t)e.frames * e.height * e.width * 3;
    if (e.src_offset < 0 || e.src_offset > src_bytes - bytes) return fail(name + "pixels outside src");
    frames += e.frames;
  }
  const int64_t frame_bytes = (int64_t)dst_height * dst_width * 3;
  if (frames > dst_bytes / frame_bytes) return fail("dst holds fewer than the call's " + std::to_string(frames) + " frames");
  if (!src || !videos_dev || !dst) return fail("NULL src, videos_dev or dst");
  if ((uintptr_t)dst < (uintptr_t)src + (uint64_t)src_bytes && (uintptr_t)src < (uintptr_t)dst + (uint64_t)(frames * frame_bytes))
    return fail("dst overlaps src");
  cudaStream_t s = (cudaStream_t)stream;
  const int tiles_x = (dst_width + kTx - 1) / kTx, tiles = tiles_x * ((dst_height + kTileH - 1) / kTileH);
  for (int64_t f0 = 0; f0 < frames; f0 += kMaxFramesPerLaunch) {
    const dim3 grid((unsigned)tiles, (unsigned)std::min<int64_t>(frames - f0, kMaxFramesPerLaunch)), block(kTx, kTy);
    resize_kernel<<<grid, block, 0, s>>>(videos_dev, n_videos, f0, tiles_x, dst_height, dst_width, src, dst);
    SSNB_LAUNCH_CHECK("resize_kernel");
  }
  return SSNB_OK;
}

}  // extern "C"
