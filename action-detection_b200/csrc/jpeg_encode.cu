// JPEG encode on the GPU, byte for byte Image.save(f, quality=q) through libjpeg-turbo (and cv2.imencode at the same quality):
// the img_%05d.jpg / flow_{x,y}_%05d.jpg files of DenseFlow's extraction step, many ragged images per call, optionally with
// Pillow's restart_marker_blocks / restart_marker_rows.  The stages are those of oracle/jpeg_encode_oracle.py, which names
// the libjpeg-turbo function each one follows, and the restart rules those of oracle/jpeg_restart_oracle.py.  Device, in
// launch order:
//
//   enc_setup_kernel    one CTA: each image's MCU, bit-buffer word, chunk and output-slot offsets (exclusive scans of sizes
//                       the host computes the same way, so the call needs no host round trip) and its restart interval.
//   enc_coef_kernel     one thread per 8x8 block (a warp per block position of the MCU, 32 MCUs per CTA): samples with edge
//                       expansion, rgb_ycc_convert and h2v2 downsampling, islow FDCT, rounded quantisation, stored in zig-zag
//                       order; and the bits of the block's AC codes.  Dummy blocks (past the luma plane's right / bottom edge
//                       inside the last MCU) are zero with an EOB.
//   enc_scan_kernel     one CTA per image: each block's bit length (its AC bits plus its DC difference's code, the predictor
//                       reset at each restart interval), a segmented scan into bit offsets in which every interval starts on
//                       a byte, the image's byte count; zeroes the image's bit buffer and its interval-end bitmap.
//   enc_pack_kernel     one thread per block: Huffman codes ORed into the bit buffer (32-bit words, most significant bit first);
//                       the last block of each interval adds the 1-bit padding and marks the interval's last byte.
//   enc_count_kernel    one CTA per 4 KB chunk of an image's bytes: its 0xFF bytes and interval ends.
//   enc_finish_kernel   one CTA per image: an exclusive scan of the chunk counts into stuffing and marker offsets, the header
//                       (with the image's size in SOF0 and its interval in DRI), EOI and the file's length.
//   enc_scatter_kernel  one CTA per chunk: the bytes at their stuffed positions, 0x00 after every 0xFF, FF D0+k after the last
//                       byte of interval k (mod 8) but the image's last.
//
// Without a restart interval an image is one interval: no marker, no DRI, the bytes of Image.save(f, quality=q).  Grids are
// sized for each image's worst case (known from its size); CTAs past an image's actual bytes return at once.  The per-block
// stages of enc_coef_kernel live in jpeg_block.cuh, which the round trip (jpeg_roundtrip.cu) calls too.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "jpeg_block.cuh"

namespace ssnb {
namespace {

constexpr int kMaxBlockBits = 22 + 63 * 26;      // a DC code of <= 11 bits + 11 value bits, 63 AC codes of <= 16 + 10 bits
constexpr int kChunk = 4096, kChunkThreads = 256, kChunkBytesPerThread = kChunk / kChunkThreads;
constexpr int kScanThreads = 1024, kMcusPerCta = 32;
constexpr int kMaxHeader = 632;                   // RGB: 623 bytes, 629 with DRI
constexpr int kMaxInterval = 65535;               // DRI's 16 bits (jcmaster.c clamps restart_in_rows * MCUs_per_row to it)
constexpr int kMarkShift = 36;                    // a chunk count: its 0xFF bytes + (its interval ends << kMarkShift)

// ---------------------------------------------------------------------------------------------------------------- tables

// Annex K.3: DC luminance, AC luminance, DC chrominance, AC chrominance (table t of class c is kHuff[2 t + c])
struct HuffSpec {
  uint8_t bits[16];
  uint8_t vals[162];
  int count;
};
constexpr HuffSpec kHuff[4] = {
    {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12},
    {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
     {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
      0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
      0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
      0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
      0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
      0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
      0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
      0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
     162},
    {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12},
    {{0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
     {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
      0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
      0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
      0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
      0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
      0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
      0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
      0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
     162}};

// jchuff.c jpeg_make_c_derived_tbl: the canonical code and its length per symbol
struct HuffEnc {
  uint16_t code[256];
  uint8_t size[256];
};
struct HuffSet {
  HuffEnc t[4];
};
constexpr HuffSet make_huff() {
  HuffSet h{};
  for (int t = 0; t < 4; ++t) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
      for (int i = 0; i < kHuff[t].bits[l - 1]; ++i, ++code, ++k) {
        h.t[t].code[kHuff[t].vals[k]] = (uint16_t)code;
        h.t[t].size[kHuff[t].vals[k]] = (uint8_t)l;
      }
      code <<= 1;
    }
  }
  return h;
}
__device__ const HuffSet d_huff = make_huff();
enum { kDC0 = 0, kAC0 = 1, kDC1 = 2, kAC1 = 3 };

// the call's constants, passed by value: quantisation divisors and the header with SOF0's size and DRI's interval left for
// each image
struct EncConst {
  int32_t div[2][64];              // quantval << 3 (the islow FDCT's output is scaled by 8), natural order
  uint8_t header[kMaxHeader];
  int32_t header_len, sof_size;    // sof_size: offset of SOF0's height (then width), big-endian 16-bit each
  int32_t dri;                     // offset of DRI's interval (big-endian 16-bit), 0 when the call writes no DRI
  int32_t comps, bpm;              // components, blocks per MCU (1 or 6)
};

struct DevEnc {
  int64_t src, out;                // the image's first byte in src, its output slot
  int64_t mcu0, word0, chunk0;     // first MCU, bit-buffer word and byte chunk in the call's arrays
  int64_t mark0;                   // first word of the interval-end bitmap (bit j of word i: byte 32 i + j ends an interval)
  int64_t nbytes;                  // entropy-coded bytes before stuffing, padding included (enc_scan_kernel)
  int32_t h, w, mcux, mcuy;
  int32_t rst, dri, intervals;     // MCUs per interval (the image's MCUs without one), DRI's value (0: none), intervals
};

// an image's sizes.  Interval k of K carries b_k bits, at most its blocks times kMaxBlockBits, padded to ceil(b_k / 8) <=
// (b_k + 7) / 8 bytes, so raw = floor((blocks * kMaxBlockBits + 7 K) / 8) bounds the entropy-coded bytes; the slot holds the
// header (with DRI when the call has an interval), raw bytes each stuffed, 2 marker bytes per interval but the first, EOI.
struct Geo {
  int mcux, mcuy, dri;
  int64_t mcus, blocks, intervals, raw, words, marks, chunks, capacity;
};

__host__ __device__ inline Geo geometry(int comps, int header_len, int h, int w, int restart_blocks, int restart_rows) {
  Geo g;
  const int m = comps == 1 ? 8 : 16;
  g.mcux = (w + m - 1) / m;
  g.mcuy = (h + m - 1) / m;
  g.mcus = (int64_t)g.mcux * g.mcuy;
  g.blocks = g.mcus * (comps == 1 ? 1 : 6);
  // jcmaster.c per_scan_setup: restart_in_rows * MCUs_per_row, clamped to 65535, per image
  g.dri = restart_blocks ? restart_blocks : restart_rows ? (int)((int64_t)restart_rows * g.mcux < kMaxInterval ? (int64_t)restart_rows * g.mcux : kMaxInterval) : 0;
  g.intervals = g.dri ? (g.mcus + g.dri - 1) / g.dri : 1;
  g.raw = (g.blocks * kMaxBlockBits + 7 * g.intervals) / 8;
  g.words = (g.raw + 3) / 4;
  g.marks = g.intervals > 1 ? (g.raw + 31) / 32 : 0;
  g.chunks = (g.raw + kChunk - 1) / kChunk;
  g.capacity = header_len + 2 * g.raw + 2 * (g.intervals - 1) + 2;
  return g;
}

// ------------------------------------------------------------------------------------------------------------- setup

__global__ void __launch_bounds__(kScanThreads) enc_setup_kernel(const ssnb_jpeg_encode_image* __restrict__ img, int n, int comps,
                                                                  int header_len, int restart_blocks, int restart_rows,
                                                                  DevEnc* __restrict__ t) {
  using Scan = cub::BlockScan<long long, kScanThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ typename Scan::TempStorage tmp;
  long long carry[4] = {0, 0, 0, 0};
  for (int base = 0; base < n; base += kScanThreads) {
    const int i = base + threadIdx.x;
    long long v[4] = {0, 0, 0, 0}, words = 0;
    if (i < n) {                                        // every field but the offsets; those follow each scan
      const ssnb_jpeg_encode_image e = img[i];
      const Geo g = geometry(comps, header_len, e.height, e.width, restart_blocks, restart_rows);
      DevEnc d;
      d.src = e.src_offset;
      d.nbytes = 0;
      d.h = e.height; d.w = e.width; d.mcux = g.mcux; d.mcuy = g.mcuy;
      d.rst = g.dri ? g.dri : (int)g.mcus;
      d.dri = g.dri;
      d.intervals = (int)g.intervals;
      t[i] = d;
      v[0] = g.mcus; v[1] = g.words + g.marks; v[2] = g.chunks; v[3] = g.capacity;
      words = g.words;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      long long o, tot;
      Scan(tmp).ExclusiveSum(v[k], o, tot);
      __syncthreads();
      o += carry[k];
      carry[k] += tot;
      if (i < n) {
        if (k == 0) t[i].mcu0 = o;
        if (k == 1) { t[i].word0 = o; t[i].mark0 = o + words; }
        if (k == 2) t[i].chunk0 = o;
        if (k == 3) t[i].out = o;
      }
    }
  }
}

// the image whose range of field F holds x (every image has at least one MCU and one chunk, so the starts increase)
template <int64_t DevEnc::*F>
__device__ __forceinline__ int find_image(const DevEnc* __restrict__ t, int n, int64_t x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t[mid].*F <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------- samples, FDCT, quantise

__device__ __forceinline__ int nbits(int v) { return 32 - __clz(abs(v)); }

// position kb of the MCU at local index m: is it a dummy block (luma past the plane's right / bottom edge)?
__device__ __forceinline__ bool is_dummy(const DevEnc& im, int bpm, int64_t lb) {
  if (bpm == 1) return false;
  const int kb = (int)(lb % 6);
  if (kb >= 4) return false;
  const int64_t m = lb / 6;
  const int by = 2 * (int)(m / im.mcux) + (kb >> 1), bx = 2 * (int)(m % im.mcux) + (kb & 1);
  return by * 8 >= im.h || bx * 8 >= im.w;
}

__global__ void __launch_bounds__(kMcusPerCta * 6) enc_coef_kernel(const DevEnc* __restrict__ t, int n, int64_t total_mcus, EncConst c,
                                                                  const uint8_t* __restrict__ src, int16_t* __restrict__ coef,
                                                                  int64_t* __restrict__ bits) {
  const int64_t mcu = (int64_t)blockIdx.x * kMcusPerCta + (threadIdx.x & 31);
  const int kb = threadIdx.x >> 5;
  if (mcu >= total_mcus) return;
  const DevEnc im = t[find_image<&DevEnc::mcu0>(t, n, mcu)];
  const int64_t m = mcu - im.mcu0;
  const int my = (int)(m / im.mcux), mx = (int)(m % im.mcux);
  const int64_t b = mcu * c.bpm + kb;
  const int H = im.h, W = im.w;
  const uint8_t* __restrict__ px = src + im.src;
  int4* dst = reinterpret_cast<int4*>(coef + b * 64);
  int s[64];
  const int comp = kb < 4 ? 0 : kb - 3;
  if (c.comps == 3 && kb < 4) {
    const int by = 2 * my + (kb >> 1), bx = 2 * mx + (kb & 1);
    if (by * 8 >= H || bx * 8 >= W) {                   // dummy block: zero, coded as DC difference 0 and EOB
#pragma unroll
      for (int i = 0; i < 8; ++i) dst[i] = make_int4(0, 0, 0, 0);
      bits[b] = d_huff.t[kAC0].size[0];
      return;
    }
    block_samples(px, H, W, 3, 0, by, bx, s);
  } else {
    block_samples(px, H, W, c.comps, comp, my, mx, s);
  }
  fdct_block(s);
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = quantise(s[i], comp ? c.div[1][i] : c.div[0][i]);
  constexpr NaturalOrder N = natural_order();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = (int)(((uint32_t)s[N.v[8 * i + 2 * j]] & 0xFFFFu) | ((uint32_t)s[N.v[8 * i + 2 * j + 1]] << 16));
    dst[i] = make_int4(u[0], u[1], u[2], u[3]);
  }
  const HuffEnc& ac = d_huff.t[comp ? kAC1 : kAC0];
  int run = 0, total = 0;
#pragma unroll
  for (int k = 1; k < 64; ++k) {
    const int v = s[N.v[k]];
    if (v == 0) { ++run; continue; }
    for (; run > 15; run -= 16) total += ac.size[0xF0];
    const int nb = nbits(v);
    total += ac.size[(run << 4) | nb] + nb;
    run = 0;
  }
  if (run) total += ac.size[0];
  bits[b] = total;
}

// ---------------------------------------------------------------------------------------------------- DC differences

// the previous block of the same component in scan order (-1 before the image's first)
__device__ __forceinline__ int64_t prev_same(int bpm, int64_t lb) {
  if (bpm == 1) return lb - 1;
  const int kb = (int)(lb % 6);
  const int64_t p = kb == 0 ? lb - 3 : (kb < 4 ? lb - 1 : lb - 6);
  return p < 0 ? -1 : p;
}

// the DC difference of block lb of an image whose blocks start at coef + b0 * 64.  A dummy block carries the DC of the block
// before it (jccoefct.c), so its difference is 0 and the next block predicts from the last real block.  The predictors
// restart at 0 with each interval (jchuff.c emit_restart), whose first block is an MCU's first luma block, never a dummy.
__device__ int dc_diff(const DevEnc& im, int bpm, const int16_t* __restrict__ coef, int64_t b0, int64_t lb) {
  if (is_dummy(im, bpm, lb)) return 0;
  int64_t first = 0;                                  // the interval's first block (an image's blocks fit 31 bits)
  if (im.intervals > 1) {
    const int m = bpm == 1 ? (int)lb : (int)lb / 6;
    first = (int64_t)(m - m % im.rst) * bpm;
  }
  int64_t p = prev_same(bpm, lb);
  while (p >= first && is_dummy(im, bpm, p)) p = prev_same(bpm, p);
  return coef[(b0 + lb) * 64] - (p < first ? 0 : coef[(b0 + p) * 64]);
}

__device__ __forceinline__ bool chroma_block(int bpm, int64_t lb) { return bpm == 6 && lb % 6 >= 4; }

// the bit offset after a run of blocks as a function of the offset before it: x + a when no interval starts inside the run,
// else ceil8(x + a) + b (a: the bits before the first interval start, b: those after the last, intervals between whole
// bytes).  Composition is associative, so a block scan of one element per block gives every block's offset with each
// interval byte aligned.  Within one pass of kScanThreads blocks a and b stay below kScanThreads * (kMaxBlockBits + 7) <
// 2^21, so the block scan runs on one 64-bit word per run (a, b and the flag packed); the carry between passes is a Seg.
struct Seg {
  long long a, b;
  bool starts;                     // does an interval start in the run?
};
__device__ __forceinline__ long long ceil8(long long x) { return (x + 7) & ~7ll; }
__device__ __forceinline__ Seg seg_then(const Seg& l, const Seg& r) {          // l, then r
  if (!r.starts) return l.starts ? Seg{l.a, l.b + r.a, true} : Seg{l.a + r.a, 0, false};
  return l.starts ? Seg{l.a, ceil8(l.b + r.a) + r.b, true} : Seg{l.a + r.a, r.b, true};
}
__device__ __forceinline__ long long seg_end(const Seg& f) { return f.starts ? ceil8(f.a) + f.b : f.a; }
constexpr int kSegBits = 22;
static_assert(kScanThreads * (kMaxBlockBits + 7) < (1 << kSegBits), "a pass's bits must fit a packed Seg field");
__device__ __forceinline__ unsigned long long seg_pack(const Seg& f) {
  return (unsigned long long)f.a | (unsigned long long)f.b << kSegBits | (unsigned long long)f.starts << (2 * kSegBits);
}
__device__ __forceinline__ Seg seg_unpack(unsigned long long v) {
  constexpr unsigned long long m = (1ull << kSegBits) - 1;
  return Seg{(long long)(v & m), (long long)(v >> kSegBits & m), (bool)(v >> (2 * kSegBits))};
}
struct PackedSegThen {
  __device__ __forceinline__ unsigned long long operator()(unsigned long long l, unsigned long long r) const {
    return seg_pack(seg_then(seg_unpack(l), seg_unpack(r)));
  }
};

// block lb's bit length: its AC bits (enc_coef_kernel) and its DC difference's code
__device__ __forceinline__ long long block_bits(const DevEnc& im, int bpm, const int16_t* __restrict__ coef,
                                                const int64_t* __restrict__ bits, int64_t b0, int64_t lb) {
  const int d = dc_diff(im, bpm, coef, b0, lb), n = nbits(d);
  return bits[b0 + lb] + d_huff.t[chroma_block(bpm, lb) ? kDC1 : kDC0].size[n] + n;
}

__global__ void __launch_bounds__(kScanThreads) enc_scan_kernel(DevEnc* __restrict__ t, int bpm, const int16_t* __restrict__ coef,
                                                                 int64_t* __restrict__ bits, uint32_t* __restrict__ words) {
  using Sum = cub::BlockScan<long long, kScanThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  using SegScan = cub::BlockScan<unsigned long long, kScanThreads, cub::BLOCK_SCAN_WARP_SCANS>;
  __shared__ union {
    typename Sum::TempStorage sum;
    typename SegScan::TempStorage seg;
  } tmp;
  const DevEnc im = t[blockIdx.x];
  const int64_t b0 = im.mcu0 * bpm, nb = (int64_t)im.mcux * im.mcuy * bpm;
  long long end = 0;                                    // the image's bits, each interval padded to a byte but the last
  if (im.intervals == 1) {                              // one interval: a sum of the block lengths
    for (int64_t base = 0; base < nb; base += kScanThreads) {
      const int64_t lb = base + threadIdx.x;
      long long len = 0, off, tot;
      if (lb < nb) len = block_bits(im, bpm, coef, bits, b0, lb);
      Sum(tmp.sum).ExclusiveSum(len, off, tot);
      if (lb < nb) bits[b0 + lb] = end + off;
      end += tot;
      __syncthreads();
    }
  } else {
    Seg carry{0, 0, false};
    for (int64_t base = 0; base < nb; base += kScanThreads) {
      const int64_t lb = base + threadIdx.x;
      long long len = 0;
      unsigned long long v = 0, inc, tot;
      if (lb < nb) {
        len = block_bits(im, bpm, coef, bits, b0, lb);
        const int m = bpm == 1 ? (int)lb : (int)lb / 6;
        const bool starts = lb > 0 && m * bpm == lb && m % im.rst == 0;
        v = seg_pack(starts ? Seg{0, len, true} : Seg{len, 0, false});
      }
      SegScan(tmp.seg).InclusiveScan(v, inc, PackedSegThen(), tot);
      if (lb < nb) bits[b0 + lb] = seg_end(seg_then(carry, seg_unpack(inc))) - len;
      carry = seg_then(carry, seg_unpack(tot));
      __syncthreads();
    }
    end = seg_end(carry);
  }
  const int64_t nbytes = (end + 7) >> 3, nwords = (nbytes + 3) >> 2;
  const int64_t nmarks = im.intervals > 1 ? (nbytes + 31) >> 5 : 0;
  uint32_t* w = words + im.word0;
  for (int64_t j = threadIdx.x; j < nwords; j += blockDim.x) w[j] = 0;
  for (int64_t j = threadIdx.x; j < nmarks; j += blockDim.x) words[im.mark0 + j] = 0;
  if (threadIdx.x == 0) t[blockIdx.x].nbytes = nbytes;
}

// ------------------------------------------------------------------------------------------------------------------ pack

struct BitWriter {
  uint32_t* w;
  int64_t word;
  uint64_t acc;                    // the pending bits, the last `n` of them valid
  int n;

  __device__ __forceinline__ void put(uint32_t v, int len) {          // len <= 27
    acc = (acc << len) | v;
    n += len;
    if (n >= 32) {
      n -= 32;
      atomicOr(w + word, (uint32_t)(acc >> n));
      ++word;
      acc &= (1ull << n) - 1;
    }
  }
  __device__ __forceinline__ void flush() {
    if (n) atomicOr(w + word, (uint32_t)(acc << (32 - n)));
  }
  __device__ __forceinline__ int64_t pos() const { return word * 32 + n; }
};

__global__ void __launch_bounds__(kMcusPerCta * 6) enc_pack_kernel(const DevEnc* __restrict__ t, int n, int64_t total_mcus, int bpm,
                                                                  const int16_t* __restrict__ coef, const int64_t* __restrict__ bits,
                                                                  uint32_t* __restrict__ words) {
  const int64_t mcu = (int64_t)blockIdx.x * kMcusPerCta + (threadIdx.x & 31);
  const int kb = threadIdx.x >> 5;
  if (mcu >= total_mcus) return;
  const DevEnc im = t[find_image<&DevEnc::mcu0>(t, n, mcu)];
  const int64_t b0 = im.mcu0 * bpm, lb = (mcu - im.mcu0) * bpm + kb;
  const bool chroma = kb >= 4;
  const HuffEnc& dc = d_huff.t[chroma ? kDC1 : kDC0];
  const HuffEnc& ac = d_huff.t[chroma ? kAC1 : kAC0];
  const int64_t pos = bits[b0 + lb];
  BitWriter bw{words + im.word0, pos >> 5, 0ull, (int)(pos & 31)};
  const int d = dc_diff(im, bpm, coef, b0, lb), nd = nbits(d);
  bw.put(((uint32_t)dc.code[nd] << nd) | ((uint32_t)(d - (d < 0)) & ((1u << nd) - 1)), dc.size[nd] + nd);
  const int16_t* __restrict__ z = coef + (b0 + lb) * 64;
  int run = 0;
  for (int k = 1; k < 64; ++k) {
    const int v = z[k];
    if (v == 0) { ++run; continue; }
    for (; run > 15; run -= 16) bw.put(ac.code[0xF0], ac.size[0xF0]);
    const int nb = nbits(v), sym = (run << 4) | nb;
    bw.put(((uint32_t)ac.code[sym] << nb) | ((uint32_t)(v - (v < 0)) & ((1u << nb) - 1)), ac.size[sym] + nb);
    run = 0;
  }
  if (run) bw.put(ac.code[0], ac.size[0]);
  const int m = (int)(mcu - im.mcu0);
  if (kb == bpm - 1 && (m + 1 == im.mcux * im.mcuy || (im.intervals > 1 && (m + 1) % im.rst == 0))) {
    const int npad = (int)(-bw.pos() & 7);             // jchuff.c flush_bits: the interval's last byte padded with 1-bits
    bw.put((1u << npad) - 1, npad);
    if (m + 1 < im.mcux * im.mcuy) {                    // an RST follows this byte
      const int64_t last = (bw.pos() >> 3) - 1;
      atomicOr(words + im.mark0 + (last >> 5), 1u << (last & 31));
    }
  }
  bw.flush();
}

// ------------------------------------------------------------------------------------------------------------- stuffing

// this thread's bytes of an image's entropy-coded data: [start, start + 16) clipped to nbytes; returns how many are 0xFF
__device__ __forceinline__ int load_bytes(const uint32_t* __restrict__ w, int64_t start, int64_t nbytes, uint8_t (&b)[kChunkBytesPerThread]) {
  int ff = 0;
#pragma unroll
  for (int q = 0; q < kChunkBytesPerThread / 4; ++q) {
    const int64_t k = start + 4 * q;
    const uint32_t v = k < nbytes ? w[k >> 2] : 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      b[4 * q + j] = (uint8_t)(v >> (24 - 8 * j));
      ff += (k + j < nbytes) && b[4 * q + j] == 0xFF;
    }
  }
  return ff;
}

// which of this thread's bytes [start, start + 16) end an interval that an RST follows: bit j for byte start + j
__device__ __forceinline__ uint32_t load_marks(const DevEnc& im, const uint32_t* __restrict__ words, int64_t start) {
  if (im.intervals == 1 || start >= im.nbytes) return 0u;
  return (words[im.mark0 + (start >> 5)] >> (start & 31)) & 0xFFFFu;
}

__global__ void __launch_bounds__(kChunkThreads) enc_count_kernel(const DevEnc* __restrict__ t, int n, const uint32_t* __restrict__ words,
                                                                   int64_t* __restrict__ counts) {
  using Reduce = cub::BlockReduce<int, kChunkThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const DevEnc im = t[find_image<&DevEnc::chunk0>(t, n, blockIdx.x)];
  const int64_t first = ((int64_t)blockIdx.x - im.chunk0) * kChunk;
  if (first >= im.nbytes) return;
  const int64_t start = first + threadIdx.x * kChunkBytesPerThread;
  uint8_t b[kChunkBytesPerThread];
  const int ff = load_bytes(words + im.word0, start, im.nbytes, b);
  const int total = Reduce(tmp).Sum(ff | __popc(load_marks(im, words, start)) << 16);    // each <= 4096 per chunk
  if (threadIdx.x == 0) counts[blockIdx.x] = (total & 0xFFFF) | (int64_t)(total >> 16) << kMarkShift;
}

__global__ void __launch_bounds__(kChunkThreads) enc_finish_kernel(const DevEnc* __restrict__ t, EncConst c, int64_t* __restrict__ counts,
                                                                    uint8_t* __restrict__ out, int64_t* __restrict__ lengths) {
  using Scan = cub::BlockScan<long long, kChunkThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const DevEnc im = t[blockIdx.x];
  const int64_t used = (im.nbytes + kChunk - 1) / kChunk;
  int64_t* cc = counts + im.chunk0;
  long long carry = 0;
  for (int64_t base = 0; base < used; base += kChunkThreads) {
    const int64_t j = base + threadIdx.x;
    long long v = j < used ? cc[j] : 0, off, tot;
    Scan(tmp).ExclusiveSum(v, off, tot);
    if (j < used) cc[j] = carry + off;
    carry += tot;
    __syncthreads();
  }
  uint8_t* dst = out + im.out;
  const uint8_t size[4] = {(uint8_t)(im.h >> 8), (uint8_t)im.h, (uint8_t)(im.w >> 8), (uint8_t)im.w};
  for (int j = threadIdx.x; j < c.header_len; j += blockDim.x) {
    const int k = j - c.sof_size, r = j - c.dri;
    dst[j] = k >= 0 && k < 4 ? size[k] : c.dri && r >= 0 && r < 2 ? (uint8_t)(im.dri >> (8 - 8 * r)) : c.header[j];
  }
  if (threadIdx.x == 0) {
    const int64_t e = c.header_len + im.nbytes + (carry & ((1ll << kMarkShift) - 1)) + 2 * (carry >> kMarkShift);
    dst[e] = 0xFF;
    dst[e + 1] = 0xD9;
    lengths[blockIdx.x] = e + 2;
  }
}

__global__ void __launch_bounds__(kChunkThreads) enc_scatter_kernel(const DevEnc* __restrict__ t, int n, int header_len,
                                                                     const uint32_t* __restrict__ words, const int64_t* __restrict__ counts,
                                                                     uint8_t* __restrict__ out) {
  using Scan = cub::BlockScan<int, kChunkThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const DevEnc im = t[find_image<&DevEnc::chunk0>(t, n, blockIdx.x)];
  const int64_t first = ((int64_t)blockIdx.x - im.chunk0) * kChunk;
  if (first >= im.nbytes) return;
  const int64_t start = first + threadIdx.x * kChunkBytesPerThread;
  uint8_t b[kChunkBytesPerThread];
  const int ff = load_bytes(words + im.word0, start, im.nbytes, b);
  const uint32_t mk = load_marks(im, words, start);
  int before;
  Scan(tmp).ExclusiveSum(ff | __popc(mk) << 16, before);
  const int64_t c = counts[blockIdx.x];
  const int64_t ff_before = (c & ((1ll << kMarkShift) - 1)) + (before & 0xFFFF), rst_before = (c >> kMarkShift) + (before >> 16);
  uint8_t* dst = out + im.out + header_len + start + ff_before + 2 * rst_before;
  int rst = (int)(rst_before & 7);
#pragma unroll
  for (int j = 0; j < kChunkBytesPerThread; ++j) {
    if (start + j >= im.nbytes) break;
    *dst++ = b[j];
    if (b[j] == 0xFF) *dst++ = 0;
    if (mk >> j & 1) {                                  // jchuff.c emit_restart: RSTk after the interval's padded last byte
      *dst++ = 0xFF;
      *dst++ = (uint8_t)(0xD0 + rst);
      rst = (rst + 1) & 7;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------- host

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

void put16(std::vector<uint8_t>& h, int v) {
  h.push_back((uint8_t)(v >> 8));
  h.push_back((uint8_t)v);
}

// jcparam.c jpeg_set_quality(quality, TRUE) and jcmarker.c's header (oracle/jpeg_encode_oracle.py quant_tables / header), with
// write_scan_header's DRI before SOS when the call has a restart interval (oracle/jpeg_restart_oracle.py header)
EncConst make_const(int comps, int quality, bool restart) {
  EncConst c;
  memset(&c, 0, sizeof c);
  int q[2][64];
  quant_tables(quality, q);
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i < 64; ++i) c.div[t][i] = q[t][i] << 3;
  const int tables = comps == 1 ? 1 : 2;
  std::vector<uint8_t> h = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (int t = 0; t < tables; ++t) {
    h.insert(h.end(), {0xFF, 0xDB, 0, 67, (uint8_t)t});
    for (int k = 0; k < 64; ++k) h.push_back((uint8_t)q[t][kNatural[k]]);
  }
  h.insert(h.end(), {0xFF, 0xC0});
  put16(h, 8 + 3 * comps);
  h.push_back(8);
  c.sof_size = (int)h.size();
  h.insert(h.end(), {0, 0, 0, 0, (uint8_t)comps});
  if (comps == 1) h.insert(h.end(), {1, 0x11, 0});
  else h.insert(h.end(), {1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
  for (int t = 0; t < tables; ++t)
    for (int cls = 0; cls < 2; ++cls) {
      const HuffSpec& s = kHuff[2 * t + cls];
      h.insert(h.end(), {0xFF, 0xC4});
      put16(h, 2 + 1 + 16 + s.count);
      h.push_back((uint8_t)(cls << 4 | t));
      h.insert(h.end(), s.bits, s.bits + 16);
      h.insert(h.end(), s.vals, s.vals + s.count);
    }
  if (restart) {
    h.insert(h.end(), {0xFF, 0xDD, 0, 4});
    c.dri = (int)h.size();
    h.insert(h.end(), {0, 0});
  }
  h.insert(h.end(), {0xFF, 0xDA});
  put16(h, 6 + 2 * comps);
  h.push_back((uint8_t)comps);
  if (comps == 1) h.insert(h.end(), {1, 0x00});
  else h.insert(h.end(), {1, 0x00, 2, 0x11, 3, 0x11});
  h.insert(h.end(), {0, 63, 0});
  memcpy(c.header, h.data(), h.size());
  c.header_len = (int)h.size();
  c.comps = comps;
  c.bpm = comps == 1 ? 1 : 6;
  return c;
}

int header_len(int comps, bool restart) { return make_const(comps, 50, restart).header_len; }

struct Layout {
  int64_t mcus = 0, blocks = 0, words = 0, chunks = 0, out_bytes = 0;
  size_t off_coef = 0, off_bits = 0, off_words = 0, off_counts = 0, workspace = 0;
};

bool check_image_size(int h, int w) { return h >= 1 && w >= 1 && h <= kJpegEncMaxSide && w <= kJpegEncMaxSide; }

// an empty string when the restart options are acceptable, else the reason
std::string check_restart(int restart_blocks, int restart_rows) {
  if (restart_blocks < 0 || restart_rows < 0) return "restart_blocks and restart_rows must be >= 0";
  if (restart_blocks && restart_rows) return "restart_blocks and restart_rows cannot both be set";
  if (restart_blocks > kMaxInterval) return "restart_blocks must be <= " + std::to_string(kMaxInterval);
  return "";
}

// the call's sizes; an empty string when the arguments are acceptable, else the reason
std::string plan(int mode, int quality, int restart_blocks, int restart_rows, const ssnb_jpeg_encode_image* images, int n,
                 int64_t src_bytes, Layout& L) {
  if (mode != SSNB_JPEG_ENC_L && mode != SSNB_JPEG_ENC_RGB) return "mode must be SSNB_JPEG_ENC_L (1) or SSNB_JPEG_ENC_RGB (3)";
  if (quality < 1 || quality > 100) return "quality must be 1 .. 100";
  const std::string why = check_restart(restart_blocks, restart_rows);
  if (!why.empty()) return why;
  if (n < 1 || !images) return "no image, or NULL images";
  const int hl = header_len(mode, restart_blocks || restart_rows);
  for (int i = 0; i < n; ++i) {
    const ssnb_jpeg_encode_image& e = images[i];
    if (!check_image_size(e.height, e.width))
      return "image " + std::to_string(i) + ": height and width must be 1 .. " + std::to_string(kJpegEncMaxSide);
    if (src_bytes >= 0 && (e.src_offset < 0 || e.src_offset + (int64_t)e.height * e.width * mode > src_bytes))
      return "image " + std::to_string(i) + ": pixels outside src";
    const Geo g = geometry(mode, hl, e.height, e.width, restart_blocks, restart_rows);
    L.mcus += g.mcus; L.blocks += g.blocks; L.words += g.words + g.marks; L.chunks += g.chunks; L.out_bytes += g.capacity;
  }
  if ((L.mcus + kMcusPerCta - 1) / kMcusPerCta > INT32_MAX || L.chunks > INT32_MAX) return "too many blocks in one call";
  size_t o = align256((size_t)n * sizeof(DevEnc));
  L.off_coef = o; o = align256(o + (size_t)L.blocks * 128);
  L.off_bits = o; o = align256(o + (size_t)L.blocks * 8);
  L.off_words = o; o = align256(o + (size_t)L.words * 4);
  L.off_counts = o; o = align256(o + (size_t)L.chunks * 8);
  L.workspace = o;
  return "";
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int64_t ssnb_jpeg_encode_restart_capacity(int mode, int height, int width, int restart_blocks, int restart_rows) {
  if ((mode != SSNB_JPEG_ENC_L && mode != SSNB_JPEG_ENC_RGB) || !check_image_size(height, width) ||
      !check_restart(restart_blocks, restart_rows).empty())
    return 0;
  return geometry(mode, header_len(mode, restart_blocks || restart_rows), height, width, restart_blocks, restart_rows).capacity;
}

int64_t ssnb_jpeg_encode_capacity(int mode, int height, int width) { return ssnb_jpeg_encode_restart_capacity(mode, height, width, 0, 0); }

int ssnb_jpeg_encode_restart_sizes(int mode, int quality, int restart_blocks, int restart_rows, const ssnb_jpeg_encode_image* images, int n,
                                   size_t* workspace_bytes, int64_t* out_bytes) {
  Layout L;
  const std::string why = plan(mode, quality, restart_blocks, restart_rows, images, n, -1, L);
  if (!why.empty()) {
    set_thread_error("jpeg_encode: " + why);
    return SSNB_EINVAL;
  }
  if (workspace_bytes) *workspace_bytes = L.workspace;
  if (out_bytes) *out_bytes = L.out_bytes;
  return SSNB_OK;
}

int ssnb_jpeg_encode_sizes(int mode, int quality, const ssnb_jpeg_encode_image* images, int n, size_t* workspace_bytes, int64_t* out_bytes) {
  return ssnb_jpeg_encode_restart_sizes(mode, quality, 0, 0, images, n, workspace_bytes, out_bytes);
}

int ssnb_jpeg_encode_restart(int mode, int quality, int restart_blocks, int restart_rows, const uint8_t* src, int64_t src_bytes,
                             const ssnb_jpeg_encode_image* images, const ssnb_jpeg_encode_image* images_dev, int n, uint8_t* out,
                             int64_t out_bytes, int64_t* lengths, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("jpeg_encode: " + m); return (int)SSNB_EINVAL; };
  Layout L;
  const std::string why = plan(mode, quality, restart_blocks, restart_rows, images, n, src_bytes, L);
  if (!why.empty()) return fail(why);
  if (!src || !images_dev || !out || !lengths || !workspace) return fail("NULL src, images_dev, out, lengths or workspace");
  if ((uintptr_t)workspace % 256) return fail("workspace must be 256-byte aligned");
  if (out_bytes < L.out_bytes) return fail("out holds fewer bytes than the images' slots (ssnb_jpeg_encode_sizes)");
  if (workspace_bytes < L.workspace) return fail("workspace too small (ssnb_jpeg_encode_sizes)");
  const EncConst c = make_const(mode, quality, restart_blocks || restart_rows);
  uint8_t* ws = (uint8_t*)workspace;
  DevEnc* t = (DevEnc*)ws;
  int16_t* coef = (int16_t*)(ws + L.off_coef);
  int64_t* bits = (int64_t*)(ws + L.off_bits);
  uint32_t* words = (uint32_t*)(ws + L.off_words);
  int64_t* counts = (int64_t*)(ws + L.off_counts);
  const unsigned mcu_ctas = (unsigned)((L.mcus + kMcusPerCta - 1) / kMcusPerCta);
  enc_setup_kernel<<<1, kScanThreads, 0, s>>>(images_dev, n, mode, c.header_len, restart_blocks, restart_rows, t);
  SSNB_LAUNCH_CHECK("enc_setup_kernel");
  enc_coef_kernel<<<mcu_ctas, kMcusPerCta * c.bpm, 0, s>>>(t, n, L.mcus, c, src, coef, bits);
  SSNB_LAUNCH_CHECK("enc_coef_kernel");
  enc_scan_kernel<<<n, kScanThreads, 0, s>>>(t, c.bpm, coef, bits, words);
  SSNB_LAUNCH_CHECK("enc_scan_kernel");
  enc_pack_kernel<<<mcu_ctas, kMcusPerCta * c.bpm, 0, s>>>(t, n, L.mcus, c.bpm, coef, bits, words);
  SSNB_LAUNCH_CHECK("enc_pack_kernel");
  enc_count_kernel<<<(unsigned)L.chunks, kChunkThreads, 0, s>>>(t, n, words, counts);
  SSNB_LAUNCH_CHECK("enc_count_kernel");
  enc_finish_kernel<<<n, kChunkThreads, 0, s>>>(t, c, counts, out, lengths);
  SSNB_LAUNCH_CHECK("enc_finish_kernel");
  enc_scatter_kernel<<<(unsigned)L.chunks, kChunkThreads, 0, s>>>(t, n, c.header_len, words, counts, out);
  SSNB_LAUNCH_CHECK("enc_scatter_kernel");
  return SSNB_OK;
}

int ssnb_jpeg_encode(int mode, int quality, const uint8_t* src, int64_t src_bytes, const ssnb_jpeg_encode_image* images,
                     const ssnb_jpeg_encode_image* images_dev, int n, uint8_t* out, int64_t out_bytes, int64_t* lengths, void* workspace,
                     size_t workspace_bytes, void* stream) {
  return ssnb_jpeg_encode_restart(mode, quality, 0, 0, src, src_bytes, images, images_dev, n, out, out_bytes, lengths, workspace,
                                  workspace_bytes, stream);
}

}  // extern "C"
