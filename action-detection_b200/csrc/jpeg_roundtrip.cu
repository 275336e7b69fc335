// JPEG round trip on the GPU: for uint8 images, the pixels Pillow reads back from the files Pillow writes, i.e.
// np.asarray(Image.open(BytesIO(f)).convert(mode)) of f = Image.save(quality=q), and so ssnb_jpeg_decode of ssnb_jpeg_encode's
// files, without the files.  JPEG loses information only where it quantises DCT coefficients; the entropy coding, the byte
// stuffing and the file layout are lossless, so a block goes from the encoder's samples to the decoder's samples in one
// thread and its coefficients never leave the SM.  The per-block stages are jpeg_block.cuh's, the ones jpeg_encode.cu and
// jpeg.cu run.
//
//   roundtrip_kernel<1>  'L': one CTA per 128 x 128 pixel tile, a thread per 8x8 block: edge-expanded samples, islow FDCT,
//                        rounded quantisation, dequantisation, islow IDCT with the range limit, into shared memory; then the
//                        tile's pixels are copied out row by row.
//   roundtrip_kernel<3>  'RGB' (YCbCr 4:2:0): one CTA per 8 x 4 MCU tile (128 x 64 pixels): 128 threads take its luma blocks
//                        and 120 its Cb and Cr blocks with a one-block halo (the fancy upsampling of a tile's edge pixels
//                        reads the neighbouring MCU's chroma; halo blocks are recomputed by every tile that needs them);
//                        then every pixel of the tile is upsampled and converted to RGB from shared memory.
//
// A tile writes only its own pixels.  The grid is (largest tile count of the call's images, images); CTAs past an image's
// tiles return at once, so nothing depends on a device-side size and a call can be captured in a CUDA graph.
#include <algorithm>
#include <string>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "jpeg_block.cuh"

namespace ssnb {
namespace {

constexpr int kThreads = 256, kTileW = 128;                   // a tile is 128 pixels wide in both modes
constexpr int kHaloW = kTileW / 16 + 2, kHaloH = 64 / 16 + 2; // 'RGB': chroma blocks of a tile with their one-block halo
constexpr int kMaxImagesPerLaunch = 65535;                    // gridDim.y

template <int C>
__host__ __device__ constexpr int tile_h() { return C == 1 ? 128 : 64; }

struct RtConst {
  int32_t div[2][64];              // quantval << 3 (the islow FDCT's output is scaled by 8), natural order
  int32_t quant[2][64];            // quantval, the decoder's dequantisation
};

template <int C>
__global__ void __launch_bounds__(kThreads) roundtrip_kernel(const ssnb_jpeg_encode_image* __restrict__ images, RtConst c,
                                                             const uint8_t* __restrict__ src, uint8_t* __restrict__ out) {
  constexpr int TH = tile_h<C>(), kLuma = TH / 8 * (kTileW / 8);
  __shared__ __align__(16) uint8_t luma[TH][kTileW];
  __shared__ __align__(16) uint8_t chro[C == 1 ? 1 : 2][kHaloH * 8][kHaloW * 8];
  const ssnb_jpeg_encode_image im = images[blockIdx.y];
  const int H = im.height, W = im.width;
  const int tiles_x = (W + kTileW - 1) / kTileW;
  if ((int)blockIdx.x >= tiles_x * ((H + TH - 1) / TH)) return;
  const int y0 = (int)blockIdx.x / tiles_x * TH, x0 = (int)blockIdx.x % tiles_x * kTileW;
  const int t = threadIdx.x;
  int comp = 0, by = 0, bx = 0;
  bool active = false;
  if (t < kLuma) {
    by = y0 / 8 + t / (kTileW / 8);
    bx = x0 / 8 + t % (kTileW / 8);
    active = by * 8 < H && bx * 8 < W;
  } else if (C == 3 && t < kLuma + 2 * kHaloH * kHaloW) {
    const int k = (t - kLuma) % (kHaloH * kHaloW);
    comp = 1 + (t - kLuma) / (kHaloH * kHaloW);
    by = y0 / 16 - 1 + k / kHaloW;
    bx = x0 / 16 - 1 + k % kHaloW;
    active = by >= 0 && bx >= 0 && by < (H + 15) / 16 && bx < (W + 15) / 16;
  }
  if (active) {
    int s[64];
    block_samples(src + im.src_offset, H, W, C, comp, by, bx, s);
    fdct_block(s);
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = quantise(s[i], comp ? c.div[1][i] : c.div[0][i]) * (comp ? c.quant[1][i] : c.quant[0][i]);
    uint32_t px[16];
    idct_block(s, px);
    uint8_t* dst = comp == 0 ? &luma[by * 8 - y0][bx * 8 - x0]
                             : &chro[comp - 1][(by - (y0 / 16 - 1)) * 8][(bx - (x0 / 16 - 1)) * 8];
    const int stride = comp == 0 ? kTileW : kHaloW * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) *reinterpret_cast<uint2*>(dst + r * stride) = make_uint2(px[2 * r], px[2 * r + 1]);
  }
  __syncthreads();
  const int h = min(TH, H - y0), w = min(kTileW, W - x0);
  uint8_t* __restrict__ dst = out + im.src_offset;
  for (int i = t; i < h * kTileW; i += kThreads) {
    const int ly = i / kTileW, lx = i % kTileW;
    if (lx >= w) continue;
    const int64_t o = ((int64_t)(y0 + ly) * W + x0 + lx) * C;
    if (C == 1) {
      dst[o] = luma[ly][lx];
    } else {
      const int dw = (W + 1) / 2, dh = (H + 1) / 2, i0 = y0 / 2 - 8, j0 = x0 / 2 - 8;
      const int cb = chroma(&chro[0][0][0], kHaloW * 8, i0, j0, dw, dh, 2, 2, x0 + lx, y0 + ly) - 128;
      const int cr = chroma(&chro[1][0][0], kHaloW * 8, i0, j0, dw, dh, 2, 2, x0 + lx, y0 + ly) - 128;
      int R, G, B;
      ycc_rgb(luma[ly][lx], cb, cr, R, G, B);
      dst[o] = (uint8_t)R;
      dst[o + 1] = (uint8_t)G;
      dst[o + 2] = (uint8_t)B;
    }
  }
}

template <int C>
int64_t tiles(int h, int w) {
  return (int64_t)((w + kTileW - 1) / kTileW) * ((h + tile_h<C>() - 1) / tile_h<C>());
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_jpeg_roundtrip(int mode, int quality, const uint8_t* src, int64_t src_bytes, const ssnb_jpeg_encode_image* images,
                        const ssnb_jpeg_encode_image* images_dev, int n, uint8_t* out, int64_t out_bytes, void* stream) {
  auto fail = [](const std::string& m) { set_thread_error("jpeg_roundtrip: " + m); return (int)SSNB_EINVAL; };
  if (mode != SSNB_JPEG_ENC_L && mode != SSNB_JPEG_ENC_RGB) return fail("mode must be SSNB_JPEG_ENC_L (1) or SSNB_JPEG_ENC_RGB (3)");
  if (quality < 1 || quality > 100) return fail("quality must be 1 .. 100");
  if (n < 1 || !images) return fail("no image, or NULL images");
  int64_t max_tiles = 0;
  for (int i = 0; i < n; ++i) {
    const ssnb_jpeg_encode_image& e = images[i];
    if (e.height < 1 || e.width < 1 || e.height > kJpegEncMaxSide || e.width > kJpegEncMaxSide)
      return fail("image " + std::to_string(i) + ": height and width must be 1 .. " + std::to_string(kJpegEncMaxSide));
    const int64_t end = e.src_offset + (int64_t)e.height * e.width * mode;
    if (e.src_offset < 0 || end > src_bytes) return fail("image " + std::to_string(i) + ": pixels outside src");
    if (end > out_bytes) return fail("image " + std::to_string(i) + ": pixels outside out");
    max_tiles = std::max(max_tiles, mode == 1 ? tiles<1>(e.height, e.width) : tiles<3>(e.height, e.width));
  }
  if (!src || !images_dev || !out) return fail("NULL src, images_dev or out");
  if ((uintptr_t)out < (uintptr_t)src + (uint64_t)src_bytes && (uintptr_t)src < (uintptr_t)out + (uint64_t)out_bytes)
    return fail("out overlaps src");
  RtConst c;
  int q[2][64];
  quant_tables(quality, q);
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i < 64; ++i) {
      c.quant[t][i] = q[t][i];
      c.div[t][i] = q[t][i] << 3;
    }
  cudaStream_t s = (cudaStream_t)stream;
  for (int i0 = 0; i0 < n; i0 += kMaxImagesPerLaunch) {
    const dim3 grid((unsigned)max_tiles, (unsigned)std::min(n - i0, kMaxImagesPerLaunch));
    if (mode == SSNB_JPEG_ENC_L) roundtrip_kernel<1><<<grid, kThreads, 0, s>>>(images_dev + i0, c, src, out);
    else roundtrip_kernel<3><<<grid, kThreads, 0, s>>>(images_dev + i0, c, src, out);
    SSNB_LAUNCH_CHECK("roundtrip_kernel");
  }
  return SSNB_OK;
}

}  // extern "C"
