// JPEG decode on the GPU, bitwise equal to Image.open(f).convert('RGB' | 'L') over libjpeg-turbo: the frame loading of the data
// sets (ssn_dataset.py:187-194, load_binary_score.py:198-205) for many ragged images per call.
//
// Host: jpeg_parse reads each image's markers up to its SOS (ITU-T T.81 B.2) and the plan stores, per image, the geometry, the
// dequantisation tables (natural order) and the Huffman tables expanded for decoding (a 9-bit prefix lookup plus maxcode /
// value offsets for the longer codes, F.2.2.3), identical tables once for the whole call; then the restart intervals of its
// scan, each with its byte range (the scan is split at its RSTn markers).  Device:
//
//   jpeg_entropy_kernel  one thread per restart interval (frames from video carry no DRI: one thread per image): Huffman
//                        decode of its MCUs to int16 coefficient blocks, DC prediction from zero.  The bit reader only reads
//                        its interval's bytes; past them it shifts in zeros and counts them, so reading into them is a
//                        TRUNCATED status.  From a corrupt block on, the interval's blocks are zero.
//   jpeg_idct_kernel     one thread per 8x8 block: libjpeg's islow IDCT (jidctint's two passes, CONST_BITS 13, PASS1_BITS
//                        2) into a uint8 plane per component at its own resolution.  The range limit is the one
//                        libjpeg-turbo's SIMD islow applies: saturate to [-128, 127], then + 128.
//   jpeg_colour_kernel   one thread per output pixel: fancy upsampling of the chroma (libjpeg's h2v1 / h2v2 triangle filter
//                        with its edge replication and alternating rounding bias; a plane at most 2 samples wide is
//                        replicated, as libjpeg does), the fixed-point YCbCr -> RGB of jdcolor (16 fraction bits), and for
//                        'L' PIL's (R 19595 + G 38470 + B 7471 + 0x8000) >> 16; a grayscale JPEG's 'RGB' repeats Y.
//
// The IDCT, the upsampling and the colour tables are jpeg_block.cuh's, which the round trip (jpeg_roundtrip.cu) calls too.
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "jpeg_block.cuh"

namespace ssnb {
namespace {

constexpr int kLookBits = 9, kMaxSide = 65535;

struct DevHuff {          // one expanded Huffman table
  uint16_t look[1 << kLookBits];   // (code length << 8) | symbol for codes of <= 9 bits, indexed by the next 9 bits; 0: longer
  int32_t maxcode[18];             // largest code of each length (-1: none); maxcode[17] > any 17-bit value
  int32_t valoff[18];              // index in vals of a length-l code: valoff[l] + code
  uint8_t vals[256];
};

struct DevImage {
  int64_t out;                     // first output byte
  int32_t width, height, comps, hs, vs, channels, mcux;
  int32_t plane[3];                // DevPlane index of each component
};

struct DevPlane {
  int64_t block;                   // first coefficient block in the workspace
  int64_t pix;                     // first byte of the plane in the workspace: [bh * 8, bw * 8] uint8
  int32_t bw, bh, h, v, quant, dc, ac, image;
};

struct DevInterval {
  int64_t begin, end;              // the interval's bytes in src (stuffed, markers excluded)
  int32_t image, mcu_begin, mcu_end, status;   // status: a fault the host already saw (a restart marker out of sequence)
};

struct Tables {
  const DevImage* images;
  const DevPlane* planes;
  const DevInterval* intervals;
  const DevHuff* huff;
  const int32_t* quant;            // [n_quant][64], natural order
};

// ---------------------------------------------------------------------------------------------------------------- entropy

struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;                    // the next bits, most significant first
  int nbits;                       // valid bits in acc
  int pad;                         // how many of the last bits in acc are zeros shifted in past the data

  __device__ void fill() {
    while (nbits <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF) {           // stuffed 0xFF 0x00 is a data byte; anything else is a marker and ends the data
          if (p < end && *p == 0x00) ++p;
          else { p = end; b = 0; pad += 8; }
        }
      } else {
        pad += 8;
      }
      acc |= (uint64_t)b << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek16() const { return (uint32_t)(acc >> 48); }
  __device__ __forceinline__ void skip(int n) { acc <<= n; nbits -= n; }
  __device__ __forceinline__ int bits(int n) {     // 1 <= n <= 16
    const int v = (int)(acc >> (64 - n));
    skip(n);
    return v;
  }
  __device__ __forceinline__ bool overrun() const { return nbits < pad; }
};

// one Huffman symbol (F.2.2.3); -1 when no code matches
__device__ __forceinline__ int huff_decode(BitReader& br, const DevHuff* __restrict__ t) {
  br.fill();
  const uint32_t w = br.peek16();
  const uint32_t e = t->look[w >> (16 - kLookBits)];
  if (e) { br.skip(e >> 8); return e & 255; }
  int l = kLookBits + 1;
  int code = (int)(w >> (16 - l));
  while (l <= 16 && code > __ldg(&t->maxcode[l])) { ++l; code = (int)(w >> (16 - l)); }
  if (l > 16) return -1;
  br.skip(l);
  return t->vals[__ldg(&t->valoff[l]) + code];
}

__device__ __forceinline__ int extend(int v, int s) { return v < (1 << (s - 1)) ? v + 1 - (1 << s) : v; }

__device__ __forceinline__ void zero_block(int16_t* blk) {
  int4* q = reinterpret_cast<int4*>(blk);
#pragma unroll
  for (int i = 0; i < 8; ++i) q[i] = make_int4(0, 0, 0, 0);
}

// decode one block into blk (zeroed first); returns a SSNB_JPEG_* status
__device__ int decode_block(BitReader& br, const DevHuff* __restrict__ dc, const DevHuff* __restrict__ ac, int& pred, int16_t* blk) {
  zero_block(blk);
  int s = huff_decode(br, dc);
  if (s < 0) return SSNB_JPEG_BAD_CODE;
  if (s) s = extend(br.bits(s), s);
  pred += s;
  blk[0] = (int16_t)pred;          // JCOEF is 16-bit
  for (int k = 1; k < 64; ++k) {
    const int rs = huff_decode(br, ac);
    if (rs < 0) return SSNB_JPEG_BAD_CODE;
    const int r = rs >> 4;
    s = rs & 15;
    if (s) {
      k += r;
      if (k > 63) return SSNB_JPEG_BAD_RUN;
      blk[c_natural[k]] = (int16_t)extend(br.bits(s), s);
    } else {
      if (r != 15) break;
      k += 15;
    }
  }
  return br.overrun() ? SSNB_JPEG_TRUNCATED : SSNB_JPEG_OK;
}

__global__ void __launch_bounds__(32) jpeg_entropy_kernel(Tables t, int n_intervals, const uint8_t* __restrict__ src,
                                                          int16_t* __restrict__ coef, int32_t* __restrict__ status) {
  const int it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= n_intervals) return;
  const DevInterval iv = t.intervals[it];
  const DevImage& im = t.images[iv.image];
  const int comps = im.comps, mcux = im.mcux;
  BitReader br{src + iv.begin, src + iv.end, 0ull, 0, 0};
  int err = iv.status;
  int pred0 = 0, pred1 = 0, pred2 = 0;
  for (int mcu = iv.mcu_begin; mcu < iv.mcu_end; ++mcu) {
    const int my = mcu / mcux, mx = mcu - my * mcux;
    for (int c = 0; c < comps; ++c) {
      const DevPlane& pl = t.planes[im.plane[c]];
      const DevHuff* dc = t.huff + pl.dc;
      const DevHuff* ac = t.huff + pl.ac;
      int pred = c == 0 ? pred0 : (c == 1 ? pred1 : pred2);
      for (int v = 0; v < pl.v; ++v)
        for (int h = 0; h < pl.h; ++h) {
          int16_t* blk = coef + (pl.block + (int64_t)(my * pl.v + v) * pl.bw + mx * pl.h + h) * 64;
          if (err) { zero_block(blk); continue; }
          err = decode_block(br, dc, ac, pred, blk);
          if (err) zero_block(blk);
        }
      if (c == 0) pred0 = pred; else if (c == 1) pred1 = pred; else pred2 = pred;
    }
  }
  if (err) atomicMax(&status[iv.image], err);
}

// ------------------------------------------------------------------------------------------------------------------- IDCT

__device__ __forceinline__ int plane_of(const DevPlane* __restrict__ p, int n, int64_t blk) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p[mid].block <= blk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(Tables t, int n_planes, int64_t n_blocks, const int16_t* __restrict__ coef,
                                                        uint8_t* __restrict__ pix) {
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_blocks) return;
  const DevPlane pl = t.planes[plane_of(t.planes, n_planes, b)];
  const int64_t local = b - pl.block;
  const int by = (int)(local / pl.bw), bx = (int)(local - (int64_t)by * pl.bw);
  const int32_t* __restrict__ q = t.quant + pl.quant * 64;
  int v[64];
  const int4* src = reinterpret_cast<const int4*>(coef + b * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int4 w = __ldg(src + i);
    const int u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[i * 8 + 2 * j] = (int)(int16_t)(u[j] & 0xFFFF) * __ldg(q + i * 8 + 2 * j);
      v[i * 8 + 2 * j + 1] = (u[j] >> 16) * __ldg(q + i * 8 + 2 * j + 1);
    }
  }
  uint32_t px[16];
  idct_block(v, px);
  uint8_t* out = pix + pl.pix + (int64_t)by * 8 * (pl.bw * 8) + bx * 8;
#pragma unroll
  for (int r = 0; r < 8; ++r) *reinterpret_cast<uint2*>(out + (int64_t)r * pl.bw * 8) = make_uint2(px[2 * r], px[2 * r + 1]);
}

// ------------------------------------------------------------------------------------------------- upsample, colour, store

__global__ void __launch_bounds__(256) jpeg_colour_kernel(Tables t, const uint8_t* __restrict__ pix, uint8_t* __restrict__ out) {
  const DevImage im = t.images[blockIdx.x];
  const int W = im.width, H = im.height;
  const int64_t npx = (int64_t)W * H;
  const DevPlane p0 = t.planes[im.plane[0]];
  const uint8_t* y_pl = pix + p0.pix;
  const int ys = p0.bw * 8;
  uint8_t* dst = out + im.out;
  if (im.comps == 1) {
    for (int64_t i = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; i < npx; i += (int64_t)gridDim.y * blockDim.x) {
      const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
      const uint8_t v = y_pl[(int64_t)y * ys + x];
      if (im.channels == 3) { dst[i * 3] = v; dst[i * 3 + 1] = v; dst[i * 3 + 2] = v; }
      else dst[i] = v;
    }
    return;
  }
  const DevPlane p1 = t.planes[im.plane[1]], p2 = t.planes[im.plane[2]];
  const uint8_t* cb_pl = pix + p1.pix;
  const uint8_t* cr_pl = pix + p2.pix;
  const int cstride = p1.bw * 8, hs = im.hs, vs = im.vs;
  const int dw = (W + hs - 1) / hs, dh = (H + vs - 1) / vs;
  for (int64_t i = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; i < npx; i += (int64_t)gridDim.y * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
    const int Y = y_pl[(int64_t)y * ys + x];
    const int cb = chroma(cb_pl, cstride, 0, 0, dw, dh, hs, vs, x, y) - 128;
    const int cr = chroma(cr_pl, cstride, 0, 0, dw, dh, hs, vs, x, y) - 128;
    int R, G, B;
    ycc_rgb(Y, cb, cr, R, G, B);
    if (im.channels == 3) { dst[i * 3] = (uint8_t)R; dst[i * 3 + 1] = (uint8_t)G; dst[i * 3 + 2] = (uint8_t)B; }
    else dst[i] = (uint8_t)rgb_l(R, G, B);
  }
}

// ------------------------------------------------------------------------------------------------------------ host plan

struct Fail {
  int code;
  std::string why;
};

struct HuffSpec {
  uint8_t bits[16];
  std::vector<uint8_t> vals;
  bool set = false;
};

struct Parsed {
  int width = 0, height = 0, comps = 0, hs = 1, vs = 1, restart = 0;
  int id[3] = {}, h[3] = {}, v[3] = {}, tq[3] = {}, td[3] = {}, ta[3] = {};
  int32_t quant[4][64];
  bool quant_set[4] = {};
  HuffSpec dc[4], ac[4];
  int64_t scan = 0;                // offset of the entropy-coded segment within the image
};

const char* refused_sof(int m) {
  switch (m) {
    case 0xC2: return "progressive JPEG (SOF2) is not supported";
    case 0xC3: return "lossless JPEG (SOF3) is not supported";
    case 0xC5: return "hierarchical JPEG (SOF5) is not supported";
    case 0xC6: return "hierarchical JPEG (SOF6) is not supported";
    case 0xC7: return "hierarchical JPEG (SOF7) is not supported";
    case 0xC9: return "arithmetic-coded JPEG (SOF9) is not supported";
    case 0xCA: return "arithmetic-coded JPEG (SOF10) is not supported";
    case 0xCB: return "arithmetic-coded JPEG (SOF11) is not supported";
    case 0xCD: return "arithmetic-coded JPEG (SOF13) is not supported";
    case 0xCE: return "arithmetic-coded JPEG (SOF14) is not supported";
    case 0xCF: return "arithmetic-coded JPEG (SOF15) is not supported";
    case 0xDE: return "hierarchical JPEG (DHP) is not supported";
    case 0xCC: return "arithmetic-coded JPEG (DAC) is not supported";
    default: return nullptr;
  }
}

// markers up to the first SOS (the same rules and wording as oracle/jpeg_oracle.py's parse)
bool jpeg_parse(const uint8_t* b, int64_t n, Parsed& P, Fail& f) {
  auto bad = [&](int code, const std::string& why) { f = Fail{code, why}; return false; };
  const int EINV = SSNB_EINVAL, ENOS = SSNB_ENOSUPPORT;
  if (n < 4 || b[0] != 0xFF || b[1] != 0xD8) return bad(EINV, "not a JPEG stream (no SOI marker)");
  int64_t pos = 2;
  bool frame = false, jfif = false;
  int adobe = -1;
  while (true) {
    if (pos >= n) return bad(EINV, "truncated header (no SOS marker)");
    if (b[pos] != 0xFF) return bad(EINV, "malformed header (a marker was expected)");
    while (pos < n && b[pos] == 0xFF) ++pos;
    if (pos >= n) return bad(EINV, "truncated header (no SOS marker)");
    const int m = b[pos++];
    if (m == 0xD9) return bad(EINV, "malformed header (EOI before SOS)");
    if (m == 0xD8 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) || m == 0x00) {
      char buf[64];
      snprintf(buf, sizeof buf, "malformed header (unexpected marker 0x%02X)", m);
      return bad(EINV, buf);
    }
    if (pos + 2 > n) return bad(EINV, "truncated header");
    const int L = (b[pos] << 8) | b[pos + 1];
    if (L < 2 || pos + L > n) return bad(EINV, "truncated header");
    const uint8_t* s = b + pos + 2;
    const int len = L - 2;
    pos += L;
    if (const char* r = refused_sof(m)) return bad(ENOS, r);
    if (m == 0xC0 || m == 0xC1) {
      if (frame) return bad(EINV, "malformed header (two SOF markers)");
      if (len < 6) return bad(EINV, "malformed header (short SOF)");
      const int prec = s[0], nf = s[5];
      P.height = (s[1] << 8) | s[2];
      P.width = (s[3] << 8) | s[4];
      if (prec != 8) return bad(ENOS, std::to_string(prec) + "-bit samples are not supported");
      if (len != 6 + 3 * nf) return bad(EINV, "malformed header (SOF length)");
      if (P.height == 0 || P.width == 0) return bad(EINV, "malformed header (zero width or height)");
      if (nf == 4) return bad(ENOS, "CMYK / YCCK JPEG is not supported");
      if (nf != 1 && nf != 3) return bad(ENOS, std::to_string(nf) + "-component JPEG is not supported");
      P.comps = nf;
      for (int i = 0; i < nf; ++i) {
        P.id[i] = s[6 + 3 * i]; P.h[i] = s[7 + 3 * i] >> 4; P.v[i] = s[7 + 3 * i] & 15; P.tq[i] = s[8 + 3 * i];
        if (P.tq[i] > 3 || P.h[i] < 1 || P.h[i] > 4 || P.v[i] < 1 || P.v[i] > 4) return bad(EINV, "malformed header (SOF components)");
        for (int j = 0; j < i; ++j)
          if (P.id[j] == P.id[i]) return bad(EINV, "malformed header (SOF components)");
      }
      frame = true;
    } else if (m == 0xC4) {
      int i = 0;
      while (i < len) {
        if (i + 17 > len) return bad(EINV, "malformed header (short DHT)");
        const int tc = s[i] >> 4, th = s[i] & 15;
        int cnt = 0;
        for (int l = 0; l < 16; ++l) cnt += s[i + 1 + l];
        if (tc > 1 || th > 3 || cnt > 256 || i + 17 + cnt > len) return bad(EINV, "malformed header (bad DHT)");
        int code = 0;
        for (int l = 0; l < 16; ++l) {
          code += s[i + 1 + l];
          if (code > (1 << (l + 1))) return bad(EINV, "malformed header (bad Huffman table)");
          code <<= 1;
        }
        if (tc == 0)
          for (int k = 0; k < cnt; ++k)
            if (s[i + 17 + k] > 15) return bad(EINV, "malformed header (bad Huffman table)");
        HuffSpec& hs = tc ? P.ac[th] : P.dc[th];
        memcpy(hs.bits, s + i + 1, 16);
        hs.vals.assign(s + i + 17, s + i + 17 + cnt);
        hs.set = true;
        i += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int i = 0;
      while (i < len) {
        const int pq = s[i] >> 4, tq = s[i] & 15, size = pq ? 128 : 64;
        if (pq > 1 || tq > 3 || i + 1 + size > len) return bad(EINV, "malformed header (bad DQT)");
        for (int k = 0; k < 64; ++k)
          P.quant[tq][kNatural[k]] = pq ? (s[i + 1 + 2 * k] << 8) | s[i + 2 + 2 * k] : s[i + 1 + k];
        P.quant_set[tq] = true;
        i += 1 + size;
      }
    } else if (m == 0xDD) {
      if (len != 2) return bad(EINV, "malformed header (bad DRI)");
      P.restart = (s[0] << 8) | s[1];
    } else if (m == 0xE0) {
      jfif = jfif || (len >= 5 && memcmp(s, "JFIF\0", 5) == 0);
    } else if (m == 0xEE) {
      if (len >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = s[11];
    } else if (m == 0xDA) {
      if (!frame) return bad(EINV, "malformed header (SOS before SOF)");
      if (len < 1 || len != 4 + 2 * s[0]) return bad(EINV, "malformed header (SOS length)");
      const int ns = s[0];
      if (ns != P.comps) return bad(ENOS, "multi-scan sequential JPEG is not supported");
      for (int i = 0; i < ns; ++i) {
        if (s[1 + 2 * i] != P.id[i]) return bad(EINV, "malformed header (SOS components)");
        P.td[i] = s[2 + 2 * i] >> 4;
        P.ta[i] = s[2 + 2 * i] & 15;
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0)
        return bad(EINV, "malformed header (sequential scan with a spectral selection)");
      if (P.comps == 3) {
        const bool ok = P.h[1] == 1 && P.v[1] == 1 && P.h[2] == 1 && P.v[2] == 1 &&
                        ((P.h[0] == 1 && P.v[0] == 1) || (P.h[0] == 2 && P.v[0] == 1) || (P.h[0] == 2 && P.v[0] == 2));
        if (!ok) {
          char buf[96];
          snprintf(buf, sizeof buf, "sampling factors %d%dx%d%dx%d%d are not supported", P.h[0], P.v[0], P.h[1], P.v[1], P.h[2], P.v[2]);
          return bad(ENOS, buf);
        }
        // libjpeg's colour space rules: JFIF means YCbCr; else Adobe's transform; else component ids R, G, B mean RGB
        if (!jfif && adobe == 0) return bad(ENOS, "Adobe RGB (transform 0) JPEG is not supported");
        if (!jfif && adobe < 0 && P.id[0] == 82 && P.id[1] == 71 && P.id[2] == 66)
          return bad(ENOS, "RGB (component ids R, G, B) JPEG is not supported");
        P.hs = P.h[0];
        P.vs = P.v[0];
      } else {
        P.h[0] = P.v[0] = 1;
      }
      for (int i = 0; i < P.comps; ++i) {
        if (!P.quant_set[P.tq[i]]) return bad(EINV, "scan references undefined quantisation table " + std::to_string(P.tq[i]));
        if (P.td[i] > 3 || !P.dc[P.td[i]].set) return bad(EINV, "scan references undefined DC Huffman table " + std::to_string(P.td[i]));
        if (P.ta[i] > 3 || !P.ac[P.ta[i]].set) return bad(EINV, "scan references undefined AC Huffman table " + std::to_string(P.ta[i]));
      }
      P.scan = pos;
      return true;
    }
  }
}

DevHuff expand(const HuffSpec& s) {
  DevHuff t;
  memset(&t, 0, sizeof t);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t.valoff[l] = k - code;
    t.maxcode[l] = s.bits[l - 1] ? code + s.bits[l - 1] - 1 : -1;
    for (int i = 0; i < s.bits[l - 1]; ++i, ++code, ++k) {
      t.vals[k] = s.vals[k];
      if (l <= kLookBits)
        for (int w = code << (kLookBits - l); w < (code + 1) << (kLookBits - l); ++w) t.look[w] = (uint16_t)((l << 8) | s.vals[k]);
    }
    code <<= 1;
  }
  t.maxcode[0] = -1;
  t.maxcode[17] = INT_MAX;
  return t;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace
}  // namespace ssnb

using namespace ssnb;

struct ssnb_jpeg_plan_s {
  std::vector<ssnb_jpeg_image_info> info;
  std::vector<DevImage> images;
  std::vector<DevPlane> planes;
  std::vector<DevInterval> intervals;
  std::vector<DevHuff> huff;
  std::vector<int32_t> quant;
  size_t off_images = 0, off_planes = 0, off_intervals = 0, off_huff = 0, off_quant = 0, table_bytes = 0;
  int64_t blocks = 0, pix_bytes = 0, out_bytes = 0, max_pixels = 0, src_bytes = 0;
  size_t coef_bytes() const { return align256((size_t)blocks * 128); }
  size_t workspace_bytes() const { return coef_bytes() + align256((size_t)pix_bytes); }
};

namespace {

// the restart intervals of one image's scan [seg, n): split at RSTn (fill 0xFF bytes may precede a marker), ended by any other
// marker or the end of the bytes.  Intervals the scan lacks get an empty range at its end (their decode is TRUNCATED); an RSTn
// out of sequence marks the interval that follows it.  Both are decoded as zeros with that status.
void split_intervals(const uint8_t* b, int64_t base, int64_t seg, int64_t n, int image, int total_mcus, int ri, ssnb_jpeg_plan_s& pl,
                     int64_t& scan_end) {
  std::vector<DevInterval> found;
  int64_t p = seg, q = seg;
  int num = -1;
  while (true) {
    const uint8_t* f = q < n ? (const uint8_t*)memchr(b + q, 0xFF, (size_t)(n - q)) : nullptr;
    if (!f) { q = n; break; }
    q = f - b;
    if (q + 1 >= n) break;             // a last 0xFF starts a marker the bytes cut off
    const int nx = b[q + 1];
    if (nx == 0x00) { q += 2; continue; }
    int64_t r = q + 1;
    while (r < n && b[r] == 0xFF) ++r;
    if (r < n && b[r] >= 0xD0 && b[r] <= 0xD7) {
      found.push_back(DevInterval{base + p, base + q, image, 0, 0, num});
      num = b[r] - 0xD0;
      p = q = r + 1;
      continue;
    }
    break;
  }
  found.push_back(DevInterval{base + p, base + q, image, 0, 0, num});
  scan_end = q;
  const int per = ri ? ri : total_mcus;
  const int count = (total_mcus + per - 1) / per;
  for (int i = 0; i < count; ++i) {
    DevInterval iv{base + q, base + q, image, 0, 0, SSNB_JPEG_TRUNCATED};
    if (i < (int)found.size()) {
      iv = found[i];
      iv.status = (i > 0 && iv.status != (i - 1) % 8) ? SSNB_JPEG_BAD_RESTART : 0;
    }
    iv.mcu_begin = i * per;
    iv.mcu_end = std::min(total_mcus, (i + 1) * per);
    pl.intervals.push_back(iv);
  }
}

}  // namespace

extern "C" {

int ssnb_jpeg_plan_create(const uint8_t* src, size_t src_bytes, const ssnb_jpeg_input* in, int n, ssnb_jpeg_plan* out_plan, int* bad_image) {
  if (bad_image) *bad_image = -1;
  if (!out_plan) { set_thread_error("jpeg: NULL plan"); return SSNB_EINVAL; }
  *out_plan = nullptr;
  if (n < 1 || !in || !src) { set_thread_error("jpeg: no image, or NULL images / src"); return SSNB_EINVAL; }
  auto* pl = new ssnb_jpeg_plan_s();
  pl->src_bytes = (int64_t)src_bytes;
  std::map<std::string, int> huff_ids, quant_ids;
  auto fail = [&](int i, int code, const std::string& why) {
    delete pl;
    if (bad_image) *bad_image = i;
    set_thread_error("jpeg: image " + std::to_string(i) + ": " + why);
    return code;
  };
  for (int i = 0; i < n; ++i) {
    const ssnb_jpeg_input& e = in[i];
    if (e.channels != 1 && e.channels != 3) return fail(i, SSNB_EINVAL, "channels must be 3 (RGB) or 1 (L)");
    if (e.offset < 0 || e.bytes < 0 || (uint64_t)e.offset + (uint64_t)e.bytes > src_bytes) return fail(i, SSNB_EINVAL, "bytes outside src");
    Parsed P;
    Fail f;
    const uint8_t* b = src + e.offset;
    if (!jpeg_parse(b, e.bytes, P, f)) return fail(i, f.code, f.why);
    if (P.width > kMaxSide || P.height > kMaxSide) return fail(i, SSNB_EINVAL, "malformed header (size)");
    DevImage im{};
    im.out = pl->out_bytes;
    im.width = P.width; im.height = P.height; im.comps = P.comps; im.hs = P.hs; im.vs = P.vs; im.channels = e.channels;
    int mcuy;
    if (P.comps == 1) { im.mcux = (P.width + 7) / 8; mcuy = (P.height + 7) / 8; }
    else { im.mcux = (P.width + 8 * P.hs - 1) / (8 * P.hs); mcuy = (P.height + 8 * P.vs - 1) / (8 * P.vs); }
    for (int c = 0; c < P.comps; ++c) {
      DevPlane p{};
      p.h = P.comps == 1 ? 1 : P.h[c];
      p.v = P.comps == 1 ? 1 : P.v[c];
      p.bw = im.mcux * p.h;
      p.bh = mcuy * p.v;
      p.block = pl->blocks;
      p.pix = pl->pix_bytes;
      p.image = i;
      pl->blocks += (int64_t)p.bw * p.bh;
      pl->pix_bytes += (int64_t)p.bw * p.bh * 64;
      const HuffSpec* hs[2] = {&P.dc[P.td[c]], &P.ac[P.ta[c]]};
      int* ids[2] = {&p.dc, &p.ac};
      for (int k = 0; k < 2; ++k) {
        std::string key((const char*)hs[k]->bits, 16);
        key.append(hs[k]->vals.begin(), hs[k]->vals.end());
        auto it = huff_ids.find(key);
        if (it == huff_ids.end()) {
          it = huff_ids.emplace(key, (int)pl->huff.size()).first;
          pl->huff.push_back(expand(*hs[k]));
        }
        *ids[k] = it->second;
      }
      std::string qk((const char*)P.quant[P.tq[c]], sizeof(P.quant[0]));
      auto qi = quant_ids.find(qk);
      if (qi == quant_ids.end()) {
        qi = quant_ids.emplace(qk, (int)(pl->quant.size() / 64)).first;
        pl->quant.insert(pl->quant.end(), P.quant[P.tq[c]], P.quant[P.tq[c]] + 64);
      }
      p.quant = qi->second;
      im.plane[c] = (int)pl->planes.size();
      pl->planes.push_back(p);
    }
    const int64_t total = (int64_t)im.mcux * mcuy;
    if (total > INT_MAX) return fail(i, SSNB_EINVAL, "malformed header (size)");
    const size_t first_iv = pl->intervals.size();
    int64_t scan_end = 0;
    split_intervals(b, e.offset, P.scan, e.bytes, i, (int)total, P.restart, *pl, scan_end);
    ssnb_jpeg_image_info info{};
    info.width = P.width; info.height = P.height; info.components = P.comps; info.h_samp = P.hs; info.v_samp = P.vs;
    info.channels = e.channels; info.restart_interval = P.restart; info.intervals = (int32_t)(pl->intervals.size() - first_iv);
    info.scan_offset = e.offset + P.scan; info.scan_bytes = scan_end - P.scan; info.out_offset = im.out;
    pl->info.push_back(info);
    pl->images.push_back(im);
    pl->out_bytes += (int64_t)P.width * P.height * e.channels;
    pl->max_pixels = std::max(pl->max_pixels, (int64_t)P.width * P.height);
  }
  if (pl->intervals.size() > (size_t)INT_MAX || pl->blocks > ((int64_t)INT_MAX) * 128) {
    delete pl;
    set_thread_error("jpeg: too many restart intervals or blocks in one call");
    return SSNB_EINVAL;
  }
  size_t o = 0;
  pl->off_images = o; o = align256(o + pl->images.size() * sizeof(DevImage));
  pl->off_planes = o; o = align256(o + pl->planes.size() * sizeof(DevPlane));
  pl->off_intervals = o; o = align256(o + pl->intervals.size() * sizeof(DevInterval));
  pl->off_huff = o; o = align256(o + pl->huff.size() * sizeof(DevHuff));
  pl->off_quant = o; o = align256(o + pl->quant.size() * sizeof(int32_t));
  pl->table_bytes = o;
  *out_plan = pl;
  return SSNB_OK;
}

int ssnb_jpeg_plan_destroy(ssnb_jpeg_plan plan) {
  delete plan;
  return SSNB_OK;
}

int ssnb_jpeg_plan_sizes(ssnb_jpeg_plan plan, size_t* table_bytes, size_t* workspace_bytes, int64_t* out_bytes) {
  if (!plan) { set_thread_error("jpeg: NULL plan"); return SSNB_EINVAL; }
  if (table_bytes) *table_bytes = plan->table_bytes;
  if (workspace_bytes) *workspace_bytes = plan->workspace_bytes();
  if (out_bytes) *out_bytes = plan->out_bytes;
  return SSNB_OK;
}

int ssnb_jpeg_plan_image(ssnb_jpeg_plan plan, int i, ssnb_jpeg_image_info* info) {
  if (!plan || !info || i < 0 || i >= (int)plan->info.size()) { set_thread_error("jpeg: NULL plan / info or image out of range"); return SSNB_EINVAL; }
  *info = plan->info[i];
  return SSNB_OK;
}

int ssnb_jpeg_plan_write_table(ssnb_jpeg_plan plan, void* dst, size_t dst_bytes) {
  if (!plan || !dst || dst_bytes < plan->table_bytes) { set_thread_error("jpeg: NULL plan / dst or dst smaller than table_bytes"); return SSNB_EINVAL; }
  uint8_t* d = (uint8_t*)dst;
  memset(d, 0, plan->table_bytes);
  memcpy(d + plan->off_images, plan->images.data(), plan->images.size() * sizeof(DevImage));
  memcpy(d + plan->off_planes, plan->planes.data(), plan->planes.size() * sizeof(DevPlane));
  memcpy(d + plan->off_intervals, plan->intervals.data(), plan->intervals.size() * sizeof(DevInterval));
  memcpy(d + plan->off_huff, plan->huff.data(), plan->huff.size() * sizeof(DevHuff));
  memcpy(d + plan->off_quant, plan->quant.data(), plan->quant.size() * sizeof(int32_t));
  return SSNB_OK;
}

int ssnb_jpeg_decode(ssnb_jpeg_plan plan, const void* table_dev, const uint8_t* src_dev, size_t src_bytes, uint8_t* out, int64_t out_bytes,
                     int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("jpeg_decode: " + m); return (int)SSNB_EINVAL; };
  if (!plan) return fail("NULL plan");
  if (!table_dev || !src_dev || !out || !status || !workspace) return fail("NULL table, src, out, status or workspace");
  if ((uintptr_t)table_dev % 256 || (uintptr_t)workspace % 256) return fail("table and workspace must be 256-byte aligned");
  if ((int64_t)src_bytes < plan->src_bytes) return fail("src holds fewer bytes than the plan was made from");
  if (out_bytes < plan->out_bytes) return fail("out holds fewer bytes than the images decode to");
  if (workspace_bytes < plan->workspace_bytes()) return fail("workspace too small (ssnb_jpeg_plan_sizes)");
  const uint8_t* tb = (const uint8_t*)table_dev;
  Tables t{(const DevImage*)(tb + plan->off_images), (const DevPlane*)(tb + plan->off_planes),
           (const DevInterval*)(tb + plan->off_intervals), (const DevHuff*)(tb + plan->off_huff), (const int32_t*)(tb + plan->off_quant)};
  int16_t* coef = (int16_t*)workspace;
  uint8_t* pix = (uint8_t*)workspace + plan->coef_bytes();
  const int n = (int)plan->images.size(), n_iv = (int)plan->intervals.size();
  if (cudaMemsetAsync(status, 0, sizeof(int32_t) * n, s) != cudaSuccess) return fail("status memset failed");
  jpeg_entropy_kernel<<<(n_iv + 31) / 32, 32, 0, s>>>(t, n_iv, src_dev, coef, status);
  SSNB_LAUNCH_CHECK("jpeg_entropy_kernel");
  jpeg_idct_kernel<<<(unsigned)((plan->blocks + 127) / 128), 128, 0, s>>>(t, (int)plan->planes.size(), plan->blocks, coef, pix);
  SSNB_LAUNCH_CHECK("jpeg_idct_kernel");
  const unsigned chunks = (unsigned)std::min<int64_t>((plan->max_pixels + 255) / 256, 1024);
  jpeg_colour_kernel<<<dim3((unsigned)n, chunks), 256, 0, s>>>(t, pix, out);
  SSNB_LAUNCH_CHECK("jpeg_colour_kernel");
  return SSNB_OK;
}

}  // extern "C"
