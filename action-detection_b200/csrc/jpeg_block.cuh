// The per-block arithmetic of libjpeg-turbo's baseline path, shared by the encoder (jpeg_encode.cu), the decoder (jpeg.cu) and
// the round trip (jpeg_roundtrip.cu): on the encoder's side the quantisation tables, rgb_ycc_convert, edge expansion with h2v2
// downsampling, the islow FDCT and the rounded quantiser; on the decoder's side the islow IDCT with the SIMD range limit, h2v2
// fancy upsampling and the YCbCr -> RGB tables.  oracle/jpeg_encode_oracle.py and oracle/jpeg_oracle.py restate each one.
#pragma once
#include <stdint.h>

#include "jpeg_common.cuh"

namespace ssnb {
namespace {

constexpr int kJpegEncMaxSide = 65500;           // libjpeg's JPEG_MAX_DIMENSION, the encoder's largest side

// Annex K.1, natural order
constexpr uint8_t kStdQuant[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
     103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

// jcparam.c jpeg_set_quality(quality, force_baseline = TRUE): luminance (t = 0) and chrominance (t = 1) tables, natural order
inline void quant_tables(int quality, int (&q)[2][64]) {
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i < 64; ++i) {
      const int v = (kStdQuant[t][i] * scale + 50) / 100;
      q[t][i] = v < 1 ? 1 : (v > 255 ? 255 : v);
    }
}

// ------------------------------------------------------------------------------------------------------------ encoder side

__device__ __forceinline__ int rgb_y(const uint8_t* p) {
  return (fix16(0.29900) * p[0] + fix16(0.58700) * p[1] + fix16(0.11400) * p[2] + (1 << 15)) >> 16;
}
__device__ __forceinline__ int rgb_c(const uint8_t* p, int cr) {      // ONE_HALF - 1: never above 255
  const int v = cr ? fix16(0.5) * p[0] - fix16(0.41869) * p[1] - fix16(0.08131) * p[2]
                   : -fix16(0.16874) * p[0] - fix16(0.33126) * p[1] + fix16(0.5) * p[2];
  return (v + (128 << 16) + (1 << 15) - 1) >> 16;
}

// the samples of one 8x8 block of an image (uint8 [H, W, comps] at px, rows packed), edge-expanded as the encoder does: comp 0
// is the grey plane ('L') or Y, block (by, bx) of the full-resolution plane; comp 1 / 2 is Cb / Cr at h2v2, block (by, bx) of
// the chroma plane, rows taken in pairs (the last one repeated) and full-resolution columns clamped before downsampling
__device__ __forceinline__ void block_samples(const uint8_t* __restrict__ px, int H, int W, int comps, int comp, int by, int bx, int (&s)[64]) {
  if (comps == 1) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint8_t* row = px + (int64_t)min(by * 8 + r, H - 1) * W;
#pragma unroll
      for (int q = 0; q < 8; ++q) s[r * 8 + q] = __ldg(row + min(bx * 8 + q, W - 1));
    }
  } else if (comp == 0) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint8_t* row = px + (int64_t)min(by * 8 + r, H - 1) * W * 3;
#pragma unroll
      for (int q = 0; q < 8; ++q) s[r * 8 + q] = rgb_y(row + 3 * min(bx * 8 + q, W - 1));
    }
  } else {                                              // h2v2: rows in pairs (the last one repeated), columns clamped
    const int ch = (H + 1) / 2, cr = comp == 2;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int r0 = 2 * min(by * 8 + r, ch - 1), r1 = min(r0 + 1, H - 1);
      const uint8_t* row0 = px + (int64_t)r0 * W * 3;
      const uint8_t* row1 = px + (int64_t)r1 * W * 3;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int c0 = 3 * min(2 * (bx * 8 + q), W - 1), c1 = 3 * min(2 * (bx * 8 + q) + 1, W - 1);
        s[r * 8 + q] = (rgb_c(row0 + c0, cr) + rgb_c(row0 + c1, cr) + rgb_c(row1 + c0, cr) + rgb_c(row1 + c1, cr) + 1 + (q & 1)) >> 2;
      }
    }
  }
}

constexpr int CONST_BITS = 13, PASS1_BITS = 2;

// one jfdctint.c pass over x[0], x[s], ... x[7 s]
template <bool first>
__device__ __forceinline__ void fdct8(int* x, int s) {
  const int t0 = x[0] + x[7 * s], t7 = x[0] - x[7 * s], t1 = x[s] + x[6 * s], t6 = x[s] - x[6 * s];
  const int t2 = x[2 * s] + x[5 * s], t5 = x[2 * s] - x[5 * s], t3 = x[3 * s] + x[4 * s], t4 = x[3 * s] - x[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int sh = first ? CONST_BITS - PASS1_BITS : CONST_BITS + PASS1_BITS;
  constexpr int r = 1 << (sh - 1);
  if (first) {
    x[0] = (t10 + t11) * (1 << PASS1_BITS);
    x[4 * s] = (t10 - t11) * (1 << PASS1_BITS);
  } else {
    x[0] = (t10 + t11 + (1 << (PASS1_BITS - 1))) >> PASS1_BITS;
    x[4 * s] = (t10 - t11 + (1 << (PASS1_BITS - 1))) >> PASS1_BITS;
  }
  int z1 = (t12 + t13) * 4433;
  x[2 * s] = (z1 + t13 * 6270 + r) >> sh;
  x[6 * s] = (z1 - t12 * 15137 + r) >> sh;
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  const int a4 = t4 * 2446, a5 = t5 * 16819, a6 = t6 * 25172, a7 = t7 * 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  x[7 * s] = (a4 + z1 + z3 + r) >> sh;
  x[5 * s] = (a5 + z2 + z4 + r) >> sh;
  x[3 * s] = (a6 + z2 + z3 + r) >> sh;
  x[s] = (a7 + z1 + z4 + r) >> sh;
}

// jcdctmgr.c convsamp's level shift, then jfdctint.c: rows, then columns (output scaled by 8, natural order)
__device__ __forceinline__ void fdct_block(int (&s)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] -= 128;
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct8<true>(s + r * 8, 1);
#pragma unroll
  for (int q = 0; q < 8; ++q) fdct8<false>(s + q, 8);
}

// jcdctmgr.c quantize: |x| / d rounded half away from zero, the sign restored (d = quantval << 3)
__device__ __forceinline__ int quantise(int x, int d) {
  const int a = (abs(x) + (d >> 1)) / d;
  return x < 0 ? -a : a;
}

// ------------------------------------------------------------------------------------------------------------ decoder side

constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
              F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// one islow butterfly (jidctint.c); x[0..7] in, o[0..7] out descaled by `shift`
template <int shift>
__device__ __forceinline__ void idct8(const int* x, int* o) {
  int z1 = (x[2] + x[6]) * F0541;
  const int t2 = z1 - x[6] * F1847, t3 = z1 + x[2] * F0765;
  const int t0 = (x[0] + x[4]) * (1 << CONST_BITS), t1 = (x[0] - x[4]) * (1 << CONST_BITS);
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  z1 = o0 + o3;
  int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const int z5 = (z3 + z4) * F1175;
  o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
  z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
  o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
  constexpr int r = 1 << (shift - 1);
  o[0] = (t10 + o3 + r) >> shift; o[7] = (t10 - o3 + r) >> shift;
  o[1] = (t11 + o2 + r) >> shift; o[6] = (t11 - o2 + r) >> shift;
  o[2] = (t12 + o1 + r) >> shift; o[5] = (t12 - o1 + r) >> shift;
  o[3] = (t13 + o0 + r) >> shift; o[4] = (t13 - o0 + r) >> shift;
}

// the islow IDCT of a dequantised block v (natural order; overwritten) -> its samples, row r in px[2 r] (columns 0..3, low byte
// first) and px[2 r + 1] (columns 4..7), after the range limit libjpeg-turbo's SIMD islow applies: saturate to [-128, 127],
// then + 128
__device__ __forceinline__ void idct_block(int (&v)[64], uint32_t (&px)[16]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {             // pass 1: columns
    int x[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) x[r] = v[r * 8 + c];
    idct8<CONST_BITS - PASS1_BITS>(x, o);
#pragma unroll
    for (int r = 0; r < 8; ++r) v[r * 8 + c] = o[r];
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {             // pass 2: rows, then the range limit
    int o[8];
    idct8<CONST_BITS + PASS1_BITS + 3>(v + r * 8, o);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      lo |= (uint32_t)(min(max(o[c], -128), 127) + 128) << (8 * c);
      hi |= (uint32_t)(min(max(o[c + 4], -128), 127) + 128) << (8 * c);
    }
    px[2 * r] = lo;
    px[2 * r + 1] = hi;
  }
}

// the upsampled chroma sample at output pixel (x, y) of a plane dw x dh samples whose sample (i, j) is p[(i - i0) * stride + j -
// j0]: h1 copies; h2v1 / h2v2 use libjpeg's fancy triangle filter with its edge replication and alternating rounding bias,
// except that a plane at most 2 samples wide is replicated
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ p, int stride, int i0, int j0, int dw, int dh, int hs, int vs, int x,
                                      int y) {
  if (hs == 1) return p[(int64_t)(y - i0) * stride + x - j0];
  const int j = x >> 1, odd = x & 1;
  if (dw <= 2) return p[(int64_t)((vs == 2 ? y >> 1 : y) - i0) * stride + j - j0];     // libjpeg replicates planes this narrow
  const int jn = odd ? min(j + 1, dw - 1) : max(j - 1, 0);
  if (vs == 1) {
    const int64_t row = (int64_t)(y - i0) * stride - j0;
    return (3 * p[row + j] + p[row + jn] + 1 + odd) >> 2;
  }
  const int i = y >> 1, in_ = (y & 1) ? min(i + 1, dh - 1) : max(i - 1, 0);
  const int64_t r0 = (int64_t)(i - i0) * stride - j0, r1 = (int64_t)(in_ - i0) * stride - j0;
  const int cs = 3 * p[r0 + j] + p[r1 + j], csn = 3 * p[r0 + jn] + p[r1 + jn];
  return (3 * cs + csn + 8 - odd) >> 4;
}

// jdcolor.c ycc_rgb_convert's fixed-point tables (16 fraction bits), clipped; cb and cr already less 128
__device__ __forceinline__ void ycc_rgb(int Y, int cb, int cr, int& R, int& G, int& B) {
  R = min(max(Y + ((fix16(1.40200) * cr + (1 << 15)) >> 16), 0), 255);
  G = min(max(Y + ((-fix16(0.34414) * cb + (1 << 15) - fix16(0.71414) * cr) >> 16), 0), 255);
  B = min(max(Y + ((fix16(1.77200) * cb + (1 << 15)) >> 16), 0), 255);
}

// PIL's RGB -> L
__device__ __forceinline__ int rgb_l(int R, int G, int B) { return (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16; }

}  // namespace
}  // namespace ssnb
