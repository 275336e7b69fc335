// What the JPEG decoder (jpeg.cu) and encoder (jpeg_encode.cu) share: the zig-zag order and libjpeg's 16-bit fixed point
// (jpeg_block.cuh has the per-block arithmetic).
#pragma once
#include <stdint.h>

namespace ssnb {

// kNatural[k] / c_natural[k]: row-major index of the k-th coefficient in zig-zag order (T.81 figure A.6)
#define SSNB_JPEG_NATURAL                                                                                                    \
  {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, \
   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}

namespace {
const uint8_t kNatural[64] = SSNB_JPEG_NATURAL;
__constant__ uint8_t c_natural[64] = SSNB_JPEG_NATURAL;

// the same order as a constant expression, for fully unrolled loops that keep a block in registers
struct NaturalOrder {
  uint8_t v[64];
};
__host__ __device__ constexpr NaturalOrder natural_order() { return NaturalOrder{SSNB_JPEG_NATURAL}; }

// libjpeg's FIX(x) at 16 fraction bits (jccolor.c / jdcolor.c SCALEBITS)
__host__ __device__ constexpr int fix16(double x) { return (int)(x * 65536.0 + 0.5); }
}  // namespace

}  // namespace ssnb
