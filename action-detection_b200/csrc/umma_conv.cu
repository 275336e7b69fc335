// wgmma implicit-GEMM convolution (sm_90a): host-side planning and the kernel that runs every tensor-core convolution
// (forward, data gradient, fused sibling 1x1 forward / data gradient, stride-2 forward through TMA element strides).
//
//   warpgroup 0     : TMA producer (one thread; A: 4-D activation box, B: 3-D weight box, SWIZZLE_128B), stages in tile order
//   warpgroups 1, 2 : ping-pong consumers -- each owns every other tile of the CTA's persistent sequence, all 128 rows: two
//                     m64nNk16 wgmmas (N = block_n <= 128) per 16 channels, fp32 accumulators in registers; then the
//                     epilogue, one 16-column slice at a time: bias/ReLU or accumulate/mask on the accumulator fragments
//                     (fp16 result in FAST; fp32 result and its fp16 hi / lo operand planes in SSNB_EXACT_TC), written to
//                     the warpgroup's own swizzled shared-memory staging in the output box layout and stored by TMA
//                     (clipped at the image and at the destination's channel count).  An order barrier hands the tensor
//                     pipe from one warpgroup to the other once a tile's MMAs are issued, so one tile's epilogue runs
//                     under the next tile's MMAs.
//
// Rows of the M tile are the pixels of one TMA box (bw x bh x bf); taps shift the box origin and
// rely on TMA's out-of-bounds zero fill for the convolution padding.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>

#include "umma_conv.cuh"
#include "umma_dev.cuh"

namespace ssnb {

namespace {

using namespace umma;
constexpr int MAX_STAGES = 8;
constexpr int PIPE_BYTES = 192 * 1024;             // operand staging: 3 four-plane EXACT_TC stages at block_n 128
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;     // 16 KiB
constexpr int NUM_THREADS = 384;
constexpr int N_STEP = 16;                         // block_n granularity (wgmma N is any multiple of 8; the epilogue works in 16-column slices)
constexpr int MAX_BLOCK_N = 128;                   // 128 accumulators per consumer thread
constexpr int EPI_COLS = 16;                       // accumulator columns per epilogue slice = the width of one output store box
constexpr int EPI_F32_BYTES = BLOCK_M * EPI_COLS * 4;          // a slice of fp32 results: 128 rows of 64 bytes
constexpr int EPI_F16_BYTES = BLOCK_M * EPI_COLS * 2;          // a slice of fp16 values: 128 rows of 32 bytes
constexpr int EPI_BYTES = EPI_F32_BYTES + 2 * EPI_F16_BYTES;   // per consumer warpgroup: fp32 | hi | lo = 16 KiB (FAST: fp16 only)
constexpr int BAR_BYTES = 256;
constexpr int SMEM_BYTES = PIPE_BYTES + 2 * EPI_BYTES + BAR_BYTES + 1024 /*align slack*/;
// named barriers: 1 + cw orders the consumers' mainloops (256 threads: one warpgroup arrives, the other waits),
// 3 + cw guards warpgroup cw's epilogue staging (128 threads)
constexpr int ORDER_BAR = 1;
constexpr int EPI_BAR = 3;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");

struct TileCoord { int w0, h0, f0, n0; };
__device__ __forceinline__ TileCoord decode_tile(const UmmaConvParams& p, int tile) {
  TileCoord t;
  const int nt = tile % p.n_tiles;
  int m = tile / p.n_tiles;
  t.n0 = nt * p.block_n;
  t.w0 = (m % p.tiles_w) * p.bw; m /= p.tiles_w;
  t.h0 = (m % p.tiles_h) * p.bh; m /= p.tiles_h;
  t.f0 = m * p.bf;
  return t;
}

// Byte offset of (row r, column c) of a staged slice in the layout a TMA box of 16 columns reads it from: rows in
// decode_tile's numbering ([bf][bh][bw]), 16-byte chunks of each row XORed with address bits 7-8 (SWIZZLE_64B, 64-byte fp32
// rows) or bit 7 (SWIZZLE_32B, 32-byte fp16 rows).  The staging is 1024-byte aligned, so these are the absolute address bits
// the TMA unit swizzles with.
__device__ __forceinline__ uint32_t sw64_off(int r, int c) { return r * 64 + ((((c >> 2) ^ (r >> 1)) & 3) << 4) + (c & 3) * 4; }
__device__ __forceinline__ uint32_t sw32_off(int r, int c) { return r * 32 + ((((c >> 3) ^ (r >> 2)) & 1) << 4) + (c & 7) * 2; }

__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }

// the first NK 16-channel steps of a staged K chunk: A rows [sa, +128 rows) x B rows [sb, +BN rows), both K-major; one
// m64nBNk16 MMA per 64-row block, both on the same B slice
template <int BN, int NK>
__device__ __forceinline__ void mma_k(float* d0, float* d1, uint32_t sa, uint32_t sb) {
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    const uint64_t bdesc = make_desc_sw128(sb + k * MMA_K * 2);
    wgmma<BN, 0, 0>(d0, make_desc_sw128(sa + k * MMA_K * 2), bdesc);
    wgmma<BN, 0, 0>(d1, make_desc_sw128(sa + 64 * 128 + k * MMA_K * 2), bdesc);
  }
}

// one stage's MMAs: EXACT_TC (split) issues the three products of the hi / lo planes, small terms first, into the same
// accumulators; otherwise the one fp16 product
template <int BN, int NK>
__device__ __forceinline__ void mma_stage(float* d0, float* d1, uint32_t sa, uint32_t sb, uint32_t b_bytes, bool split) {
  if (split) {
    mma_k<BN, NK>(d0, d1, sa + A_BYTES, sb);               // A_lo . B_hi
    mma_k<BN, NK>(d0, d1, sa, sb + b_bytes);               // A_hi . B_lo
  }
  mma_k<BN, NK>(d0, d1, sa, sb);                           // A_hi . B_hi
}

// move a ring position n stages ahead
__device__ __forceinline__ void ring_advance(uint32_t& stage, uint32_t& phase, int n, int stages) {
  const uint32_t s = stage + (uint32_t)n;
  phase ^= (s / (uint32_t)stages) & 1u;
  stage = s % (uint32_t)stages;
}

// BN = block_n: a multiple of 16, at most 128 (BN accumulators per consumer thread).  DIRECT: the launch has a frame box
// that straddles its last frame below the maps' frame count (UmmaConvParams::f_direct)
template <int BN, bool DIRECT>
__device__ __forceinline__ void
umma_conv_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_a2, const CUtensorMap& tmap_b, const CUtensorMap& tmap_a_lo,
               const CUtensorMap& tmap_a2_lo, const CUtensorMap& tmap_b_lo, const CUtensorMap& tmap_o, const CUtensorMap& tmap_o_hi,
               const CUtensorMap& tmap_o_lo, const CUtensorMap& tmap_o2, const CUtensorMap& tmap_o2_hi, const CUtensorMap& tmap_o2_lo,
               const UmmaConvParams& p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B operand tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // pipeline depth adapts to the tile: narrow-N layers get more stages in the same staging area
  const int STAGES = p.stages, STAGE_BYTES = p.stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + PIPE_BYTES + 2 * EPI_BYTES);
  uint64_t* full_bar = bars;                     // [MAX_STAGES]
  uint64_t* empty_bar = bars + MAX_STAGES;       // [MAX_STAGES]

  // warp-uniform by construction (a shuffle from lane 0): the consumers' tile loop branches on it, and ptxas serialises
  // wgmmas it cannot prove warpgroup-convergent
  const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
  const int total_tiles = p.tiles_w * p.tiles_h * p.tiles_f * p.n_tiles;
  // SSNB_EXACT_TC: a stage holds the hi and lo planes of both operands of one (tap, K chunk): [A_hi | A_lo | B_hi | B_lo]
  const bool split = p.nseg > 1;
  const int nplanes = split ? 2 : 1;
  const uint32_t b_bytes = (uint32_t)p.block_n * BLOCK_K * 2;
  const int ksteps = p.ntaps * p.kchunks;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a2)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_b)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_o)) : "memory");
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }   // released by the consumer that owns the tile
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer: stages in tile order, whichever consumer owns the tile =====
    producer_regs();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      // bytes the two TMA boxes deliver (zero-filled out-of-bounds elements count; a 7x1x18 box has 126 rows)
      const uint32_t a_bytes = (uint32_t)(p.bw * p.bh * p.bf) * BLOCK_K * 2;
      const uint32_t tx_bytes = (a_bytes + b_bytes) * nplanes;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const TileCoord t = decode_tile(p, tile);
        for (int tap = 0; tap < p.ntaps; ++tap) {
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * STAGE_BYTES;
            uint8_t* sb = sa + nplanes * A_BYTES;
            mbar_expect_tx(&full_bar[stage], tx_bytes);
            for (int pl = 0; pl < nplanes; ++pl) {     // 0: hi (or the single fp16 plane), 1: lo
              if (kc < p.kchunks_a1)
                tma_load_4d(sa + pl * A_BYTES, pl ? &tmap_a_lo : &tmap_a, &full_bar[stage], kc * BLOCK_K, t.w0 * p.a_stride + p.tap_dx[tap],
                            t.h0 * p.a_stride + p.tap_dy[tap], t.f0);
              else
                tma_load_4d(sa + pl * A_BYTES, pl ? &tmap_a2_lo : &tmap_a2, &full_bar[stage], (kc - p.kchunks_a1) * BLOCK_K, t.w0 + p.tap_dx[tap],
                            t.h0 + p.tap_dy[tap], t.f0);
              tma_load_3d(sb + pl * b_bytes, pl ? &tmap_b_lo : &tmap_b, &full_bar[stage], kc * BLOCK_K, t.n0, tap);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===== consumers (ping-pong): warpgroup cw owns the CTA's tiles cw, cw + 2, ... of its sequence, all 128 rows =====
    consumer_regs();
    const int cw = wg - 1, row = threadIdx.x & 127;
    const int warp = row / 32, lane = row & 31;
    uint8_t* epi = smem + PIPE_BYTES + cw * EPI_BYTES;
    const float alpha = p.out_f32 ? p.alpha * (p.alpha_dev ? __ldg(p.alpha_dev) : 1.0f) : 1.0f;
    // grid <= total_tiles, so every CTA has at least one tile
    const int my_tiles = (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    uint32_t stage = 0, phase = 0;
    if (cw) ring_advance(stage, phase, ksteps, STAGES);
    for (int j = cw; j < my_tiles; j += 2) {
      const TileCoord t = decode_tile(p, (int)blockIdx.x + j * (int)gridDim.x);
      float acc[2][BN / 2];
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[b][i] = 0.f;
      // order barrier: the MMAs of tile j start once the other warpgroup has issued all of tile j - 1's, so the tensor
      // pipe runs one tile at a time while the other warpgroup is in its epilogue.  Invariant: every sync at j > 0 pairs
      // with exactly one arrive by the other warpgroup at j - 1 (guarded by j + 1 < my_tiles below).  It also keeps the
      // two consumers' full_bar parity waits from aliasing a ring phase two fills ahead.  bar.sync has no timeout, so
      // an edit that breaks the pairing hangs rather than traps: keep both guards in step.
      if (j > 0) named_bar_sync(ORDER_BAR + cw, 256);
      uint32_t prev = 0;
      int kc = 0;
      for (int ks = 0; ks < ksteps; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t sb = sa + nplanes * A_BYTES;
        // K chunks whose tail is TMA zero fill (Cin % 64 != 0) skip the all-zero MMAs
        const int kvalid = kc < p.kchunks_a1 ? p.K1 - kc * BLOCK_K : p.K - p.K1 - (kc - p.kchunks_a1) * BLOCK_K;
        const int nk = kvalid >= BLOCK_K ? BLOCK_K / MMA_K : (kvalid + MMA_K - 1) / MMA_K;
        // per 16 channels one m64nBNk16 MMA per row block: the B slice is read from shared memory for both.  Every path
        // issues a compile-time number of MMAs (no predicated wgmma inside a sequence).
        wgmma_fence();
        switch (nk) {
          case 1: mma_stage<BN, 1>(acc[0], acc[1], sa, sb, b_bytes, split); break;
          case 2: mma_stage<BN, 2>(acc[0], acc[1], sa, sb, b_bytes, split); break;
          case 3: mma_stage<BN, 3>(acc[0], acc[1], sa, sb, b_bytes, split); break;
          default: mma_stage<BN, BLOCK_K / MMA_K>(acc[0], acc[1], sa, sb, b_bytes, split); break;
        }
        wgmma_commit();
        // one group stays in flight: the previous stage's MMAs have retired, its smem slot goes back to the producer
        wgmma_wait<1>();
        if (ks > 0 && row == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
        if (++kc == p.kchunks) kc = 0;
      }
      if (j + 1 < my_tiles) named_bar_arrive(ORDER_BAR + (cw ^ 1), 256);
      wgmma_wait<0>();
      if (row == 0) mbar_arrive(&empty_bar[prev]);
      ring_advance(stage, phase, ksteps, STAGES);      // the other warpgroup's tile j + 1
      // epilogue, one 16-column slice at a time, in the accumulators' fragment layout: thread (warp, lane) holds rows
      // 64 b + 16 warp + lane / 4 + 8 h and columns 8 k + 2 (lane % 4) + {0, 1} of the slice (b, h, k in {0, 1}).  The
      // results go to this warpgroup's staging in the output box layout, from which one thread stores them by TMA.
      const bool direct = DIRECT && t.f0 >= p.f_direct;   // the partial last frame box of a launch of fewer frames than the maps'
      bool rv[2][2];                                   // the row is a pixel of the image (TMA clips the others)
      int rpix[2][2];                                  // its pixel index (f * H + h) * W + w
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = b * 64 + warp * 16 + (lane >> 2) + 8 * h;
          const int rw = r % p.bw, rh = (r / p.bw) % p.bh, rf = r / (p.bw * p.bh);
          const int w = t.w0 + rw, y = t.h0 + rh, f = t.f0 + rf;
          rv[b][h] = rf < p.bf && w < p.W && y < p.H && f < p.F;
          rpix[b][h] = (f * p.H + y) * p.W + w;
        }
      const int q2 = 2 * (lane & 3);
#pragma unroll
      for (int sl = 0; sl < BN / EPI_COLS; ++sl) {
        const int col = t.n0 + sl * EPI_COLS;          // N % 16 == 0: a slice is all inside N or all past it
        if (col >= p.Cout) break;
        const bool d1 = col < p.n_split;               // n_split % 16 == 0: a slice has one destination
        const int cd = d1 ? col : col - p.n_split;     // its first column in that destination
        const int opitch = d1 ? p.out_pitch : p.out2_pitch, ocoff = d1 ? p.out_coff : p.out2_coff;
        float v[2][2][4];                              // [b][h][2 k + e]
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const int i = sl * (EPI_COLS / 2) + 4 * k + 2 * h;   // accumulator registers [8 sl, 8 sl + 8) are slice sl's columns
              v[b][h][2 * k] = acc[b][i]; v[b][h][2 * k + 1] = acc[b][i + 1];
            }
        // the per-element operations and their order are those of the row-per-thread epilogue this replaced; explicit
        // rounding keeps the compiler from contracting alpha * acc + bias / old into an FMA
        const bool planes = p.out_f32 && (d1 ? p.planes : p.planes2);   // EXACT_TC: write the hi / lo operand planes as well
        if (p.out_f32) {
#pragma unroll
          for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int j = 0; j < 4; ++j) v[b][h][j] = __fmul_rn(v[b][h][j], alpha);
          if (p.bias) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col + 8 * k + q2));
#pragma unroll
              for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int h = 0; h < 2; ++h) { v[b][h][2 * k] = __fadd_rn(v[b][h][2 * k], bb.x); v[b][h][2 * k + 1] = __fadd_rn(v[b][h][2 * k + 1], bb.y); }
            }
          }
          if (p.accumulate) {
            const float* o32 = (d1 ? p.out32 : p.out32_2) + ocoff + cd + q2;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
                if (rv[b][h])
#pragma unroll
                  for (int k = 0; k < 2; ++k) {
                    const float2 o = *reinterpret_cast<const float2*>(o32 + (long long)rpix[b][h] * opitch + 8 * k);
                    v[b][h][2 * k] = __fadd_rn(v[b][h][2 * k], o.x); v[b][h][2 * k + 1] = __fadd_rn(v[b][h][2 * k + 1], o.y);
                  }
          }
          if (p.relu) {
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) v[b][h][j] = relu(v[b][h][j]);
          }
          if (p.mask32) {                              // ReLU gradient of the value this data gradient completes: keep where y > 0 (NaN -> 0)
            const float* m32 = p.mask32 + p.mask32_coff + col + q2;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                  const float2 y = rv[b][h] ? __ldg(reinterpret_cast<const float2*>(m32 + (long long)rpix[b][h] * p.mask32_pitch + 8 * k)) : make_float2(0.f, 0.f);
                  if (!(y.x > 0.f)) v[b][h][2 * k] = 0.f;
                  if (!(y.y > 0.f)) v[b][h][2 * k + 1] = 0.f;
                }
          }
        } else {
          if (p.bias) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + col + 8 * k + q2));
#pragma unroll
              for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int h = 0; h < 2; ++h) { v[b][h][2 * k] += bb.x; v[b][h][2 * k + 1] += bb.y; }
            }
          }
          if (p.accumulate) {
            const __half* o16 = (d1 ? p.out : p.out2) + ocoff + cd + q2;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
                if (rv[b][h])
#pragma unroll
                  for (int k = 0; k < 2; ++k) {
                    const float2 o = __half22float2(*reinterpret_cast<const __half2*>(o16 + (long long)rpix[b][h] * opitch + 8 * k));
                    v[b][h][2 * k] += o.x; v[b][h][2 * k + 1] += o.y;
                  }
          }
          if (p.relu) {
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j) v[b][h][j] = relu(v[b][h][j]);
          }
          if (p.mask_y) {
            const __half* my = p.mask_y + p.mask_coff + col + q2;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                  const float2 y = rv[b][h] ? __half22float2(__ldg(reinterpret_cast<const __half2*>(my + (long long)rpix[b][h] * p.mask_pitch + 8 * k)))
                                            : make_float2(0.f, 0.f);
                  if (!(y.x > 0.f)) v[b][h][2 * k] = 0.f;
                  if (!(y.y > 0.f)) v[b][h][2 * k + 1] = 0.f;
                }
          }
        }
        // the staging is free once the TMA has read the previous slice out of it
        if (row == 0) bulk_wait_read0();
        named_bar_sync(EPI_BAR + cw, 128);
        const bool scaled = p.flag || p.plane_scale != 1.0f;   // gradient planes: scaled by the loss scale, guarded against the fp16 range
        float m = 0.f;
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = b * 64 + warp * 16 + (lane >> 2) + 8 * h;
            if (p.out_f32) {
              // a half-warp writes rows r0..r0+3: rows with (r >> 1) & 1 write their columns 8..15 first, so that the four
              // rows' 32-byte pieces of one store fall in four different bank quarters
              const bool s = (lane >> 3) & 1;
              const float2 x0 = make_float2(v[b][h][0], v[b][h][1]), x1 = make_float2(v[b][h][2], v[b][h][3]);
              *reinterpret_cast<float2*>(epi + sw64_off(r, q2 + (s ? 8 : 0))) = s ? x1 : x0;
              *reinterpret_cast<float2*>(epi + sw64_off(r, q2 + (s ? 0 : 8))) = s ? x0 : x1;
              if (planes)
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                  float x0 = v[b][h][2 * k], x1 = v[b][h][2 * k + 1];
                  if (scaled) {
                    x0 = __fmul_rn(x0, p.plane_scale); x1 = __fmul_rn(x1, p.plane_scale);
                    if (rv[b][h]) {
                      m = fmaxf(m, fabsf(x0)); if (x0 != x0) m = INFINITY;
                      m = fmaxf(m, fabsf(x1)); if (x1 != x1) m = INFINITY;
                    }
                  }
                  const __half2 hh = __floats2half2_rn(x0, x1);
                  const float2 hf = __half22float2(hh);
                  *reinterpret_cast<uint32_t*>(epi + EPI_F32_BYTES + sw32_off(r, 8 * k + q2)) = h2_bits(hh);
                  *reinterpret_cast<uint32_t*>(epi + EPI_F32_BYTES + EPI_F16_BYTES + sw32_off(r, 8 * k + q2)) =
                      h2_bits(__floats2half2_rn(__fsub_rn(x0, hf.x), __fsub_rn(x1, hf.y)));
                }
            } else {
#pragma unroll
              for (int k = 0; k < 2; ++k)
                *reinterpret_cast<uint32_t*>(epi + sw32_off(r, 8 * k + q2)) = h2_bits(__floats2half2_rn(v[b][h][2 * k], v[b][h][2 * k + 1]));
            }
          }
        if (planes && p.flag && !(m <= 65504.f)) *p.flag = 1;
        fence_proxy_async_smem();
        named_bar_sync(EPI_BAR + cw, 128);
        if (row == 0 && !direct) {
          tma_store_4d(d1 ? &tmap_o : &tmap_o2, epi, cd, t.w0, t.h0, t.f0);
          if (planes) {
            tma_store_4d(d1 ? &tmap_o_hi : &tmap_o2_hi, epi + EPI_F32_BYTES, cd, t.w0, t.h0, t.f0);
            tma_store_4d(d1 ? &tmap_o_lo : &tmap_o2_lo, epi + EPI_F32_BYTES + EPI_F16_BYTES, cd, t.w0, t.h0, t.f0);
          }
          bulk_commit();
        }
        if (direct) {
          // the box straddles the launch's last frame below the maps' frame count, where the TMA store would also write the
          // box's rows of frames >= F: each thread copies its staged row instead, when that row is a pixel of frames < F.
          // The next slice's barrier keeps the staging until every thread has read it.
          const int rw = row % p.bw, rh = (row / p.bw) % p.bh, rf = row / (p.bw * p.bh);
          const int w = t.w0 + rw, y = t.h0 + rh, f = t.f0 + rf;
          if (rf < p.bf && w < p.W && y < p.H && f < p.F) {
            const long long po = ((long long)(f * p.H + y) * p.W + w) * opitch + ocoff + cd;
            if (p.out_f32) {
              float* o32 = (d1 ? p.out32 : p.out32_2) + po;
#pragma unroll 1
              for (int j = 0; j < EPI_COLS / 4; ++j)      // one 16-byte piece at a time: the accumulators of later slices are live
                *reinterpret_cast<float4*>(o32 + 4 * j) = *reinterpret_cast<const float4*>(epi + sw64_off(row, 4 * j));
            }
            if (!p.out_f32 || planes) {
              const uint8_t* st = epi + (p.out_f32 ? EPI_F32_BYTES : 0);
              char* o16 = reinterpret_cast<char*>((d1 ? p.out : p.out2) + po);
              const long long lo = d1 ? p.out_lo : p.out2_lo;
#pragma unroll 1
              for (int j = 0; j < EPI_COLS / 8; ++j) {
                *reinterpret_cast<uint4*>(o16 + 16 * j) = *reinterpret_cast<const uint4*>(st + sw32_off(row, 8 * j));
                if (planes) *reinterpret_cast<uint4*>(o16 + lo + 16 * j) = *reinterpret_cast<const uint4*>(st + EPI_F16_BYTES + sw32_off(row, 8 * j));
              }
            }
          }
        }
      }
    }
    if (row == 0) bulk_wait0();                        // the stores are complete before the CTA retires
  }
}

#define UMMA_CONV_PARAMS                                                                                                    \
  const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_b, \
      const __grid_constant__ CUtensorMap tmap_a_lo, const __grid_constant__ CUtensorMap tmap_a2_lo,                               \
      const __grid_constant__ CUtensorMap tmap_b_lo, const __grid_constant__ CUtensorMap tmap_o,                                   \
      const __grid_constant__ CUtensorMap tmap_o_hi, const __grid_constant__ CUtensorMap tmap_o_lo,                                \
      const __grid_constant__ CUtensorMap tmap_o2, const __grid_constant__ CUtensorMap tmap_o2_hi,                                 \
      const __grid_constant__ CUtensorMap tmap_o2_lo, const __grid_constant__ UmmaConvParams p
#define UMMA_CONV_ARGS tmap_a, tmap_a2, tmap_b, tmap_a_lo, tmap_a2_lo, tmap_b_lo, tmap_o, tmap_o_hi, tmap_o_lo, tmap_o2, tmap_o2_hi, tmap_o2_lo, p

// every convolution launch
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) umma_conv_kernel(UMMA_CONV_PARAMS) { umma_conv_body<BN, false>(UMMA_CONV_ARGS); }
// a forward launch of fewer frames than its plan whose last frame box straddles that count: the same body, whose epilogue
// copies that box's rows of the launch's frames out of the staging instead of storing the box by TMA.  A kernel of its own,
// so that the copy adds nothing to the epilogue of every other launch (inline, it made them 5-7 % slower on an H100).
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1) umma_conv_tail_kernel(UMMA_CONV_PARAMS) { umma_conv_body<BN, true>(UMMA_CONV_ARGS); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int resolve_encode(UmmaContext& ctx) {
  if (ctx.encode_tiled) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !fn) {
    cudaGetLastError();
    set_thread_error("cuTensorMapEncodeTiled not available from the driver");
    return 2;
  }
  ctx.encode_tiled = fn;
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  ctx.num_sms = sms;
  return 0;
}

int encode(UmmaContext& ctx, CUtensorMap* m, int rank, void* addr, const cuuint64_t* dims, const cuuint64_t* strides,
           const cuuint32_t* box, int spatial_stride = 1, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
           CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  // spatial_stride 2: the box traverses W and H with step 2 (box extents are given in un-strided elements)
  cuuint32_t es[5] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx.encode_tiled)(m, dtype, (cuuint32_t)rank, addr, dims, strides,
                                                                box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                                                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[128];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (CUresult %d, rank %d)", (int)r, rank);
    set_thread_error(buf);
    return 2;
  }
  return 0;
}

void pick_box(int W, int& bw, int& bh, int& bf) {
  if (W % 8 == 0 && W >= 56) { bw = 8; bh = 8; bf = 2; }
  else if (W % 4 == 0) { bw = 4; bh = 4; bf = 8; }
  else if (W % 2 == 0) { bw = 2; bh = 2; bf = 32; }
  else if (W <= 8) { bw = W; bh = 1; bf = BLOCK_M / W; }
  else { bw = 1; bh = 1; bf = 128; }
}

// the epilogue's store box over one destination: channels [0, n) of the NHWC tensor at `base` (already offset to the
// destination's first channel, `pitch` channels per pixel) at the plan's output geometry; fp32 results in 64-byte
// SWIZZLE_64B rows, fp16 values in 32-byte SWIZZLE_32B rows (the layouts of sw64_off / sw32_off)
int encode_out(UmmaContext& ctx, CUtensorMap* m, const UmmaConvParams& p, const void* base, int pitch, int n, bool f32) {
  const cuuint64_t es = f32 ? 4 : 2;
  cuuint64_t dims[4] = {(cuuint64_t)n, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.F};
  cuuint64_t str[3] = {(cuuint64_t)pitch * es, (cuuint64_t)p.W * pitch * es, (cuuint64_t)p.H * p.W * pitch * es};
  cuuint32_t box[4] = {(cuuint32_t)EPI_COLS, (cuuint32_t)p.bw, (cuuint32_t)p.bh, (cuuint32_t)p.bf};
  return encode(ctx, m, 4, const_cast<void*>(base), dims, str, box, 1, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                f32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// fp16 hi / lo operand planes of one destination: hi at `hi` (offset to the first channel), lo `lo_off` bytes later
int encode_planes(UmmaContext& ctx, CUtensorMap* mhi, CUtensorMap* mlo, const UmmaConvParams& p, const __half* hi, long long lo_off, int pitch, int n) {
  if (int rc = encode_out(ctx, mhi, p, hi, pitch, n, false)) return rc;
  return encode_out(ctx, mlo, p, reinterpret_cast<const char*>(hi) + lo_off, pitch, n, false);
}

// the output maps of one destination (second: the columns >= n_split of a fused sibling forward): view o names the fp16
// result (FAST) or the result's operand planes (EXACT_TC, o.base == nullptr: none), out32 the EXACT_TC fp32 result with
// o's pitch and channel offset
int bind_out(UmmaContext& ctx, UmmaConvPlan& plan, View o, float* out32, int n, bool second) {
  UmmaConvParams& p = plan.p;
  CUtensorMap* m = second ? &plan.tmap_o2 : &plan.tmap_o;
  CUtensorMap* mhi = second ? &plan.tmap_o2_hi : &plan.tmap_o_hi;
  CUtensorMap* mlo = second ? &plan.tmap_o2_lo : &plan.tmap_o_lo;
  const bool f32 = p.out_f32 != 0;
  if (int rc = encode_out(ctx, m, p, f32 ? (const void*)(out32 + o.coff) : (const void*)(reinterpret_cast<__half*>(o.base) + o.coff), o.pitch, n, f32))
    return rc;
  *mhi = *m; *mlo = *m;
  const int planes = f32 && o.base;
  if (planes)
    if (int rc = encode_planes(ctx, mhi, mlo, p, reinterpret_cast<__half*>(o.base) + o.coff, o.lo_off, o.pitch, n)) return rc;
  (second ? p.planes2 : p.planes) = planes;
  (second ? p.out2_lo : p.out_lo) = planes ? o.lo_off : 0;
  return 0;
}

int bind_common(UmmaContext& ctx, UmmaConvPlan& plan, View a, View o, int F, int K, int N, int ntaps, const __half* w,
                int a_stride = 1, const UmmaTcOpts* tc = nullptr) {
  plan.enabled = false;
  if (int rc = resolve_encode(ctx)) return rc;
  if (a_stride == 2 || (a_stride == 1 && (a.H != o.H || a.W != o.W))) {
    // tiles enumerate OUTPUT pixels and the A map keeps the input's dims: stride 2 (the A box steps over the input with TMA
    // element stride 2), or a valid stride-1 layer whose output is smaller than its input (taps with non-negative shifts)
    View ao = a; ao.H = o.H; ao.W = o.W;
    if (int rc = bind_common(ctx, plan, ao, o, F, K, N, ntaps, w, 1, tc)) return rc;
    plan.enabled = false;
    UmmaConvParams& q = plan.p;
    q.a_stride = a_stride;
    cuuint64_t dims[4] = {(cuuint64_t)K, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)a.pitch * 2, (cuuint64_t)a.W * a.pitch * 2, (cuuint64_t)a.H * a.W * a.pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)(a_stride * q.bw), (cuuint32_t)(a_stride * q.bh), (cuuint32_t)q.bf};
    if (int rc = encode(ctx, &plan.tmap_a, 4, reinterpret_cast<__half*>(a.base) + a.coff, dims, str, box, a_stride)) return rc;
    plan.tmap_a_lo = plan.tmap_a;
    if (a.lo_off)
      if (int rc = encode(ctx, &plan.tmap_a_lo, 4, reinterpret_cast<__half*>(reinterpret_cast<char*>(a.base) + a.lo_off) + a.coff, dims, str, box, a_stride))
        return rc;
    plan.tmap_a2 = plan.tmap_a; plan.tmap_a2_lo = plan.tmap_a_lo;
    plan.enabled = true;
    return 0;
  }
  if (a.H != o.H || a.W != o.W) { set_thread_error("umma conv: geometry mismatch"); return 1; }
  if (K % 8 || N % 16 || a.pitch % 8 || a.coff % 8 || o.pitch % 8 || o.coff % 8 || ntaps > UMMA_MAX_TAPS) {
    set_thread_error("umma conv: unsupported channel alignment"); return 1; }
  UmmaConvParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  p.W = a.W; p.H = a.H; p.F = F; p.f_direct = 1 << 30;
  pick_box(a.W, p.bw, p.bh, p.bf);
  p.tiles_w = (a.W + p.bw - 1) / p.bw; p.tiles_h = (a.H + p.bh - 1) / p.bh; p.tiles_f = (F + p.bf - 1) / p.bf;
  // N split: equal tiles of block_n <= 128 (multiple of 16); the last tile may overhang N (TMA zero-fills the
  // missing weight rows, the epilogue masks the columns)
  p.n_tiles = (N + MAX_BLOCK_N - 1) / MAX_BLOCK_N;
  p.block_n = (((N + p.n_tiles - 1) / p.n_tiles) + N_STEP - 1) / N_STEP * N_STEP;
  p.kchunks = (K + BLOCK_K - 1) / BLOCK_K;
  p.K = K;
  p.ntaps = ntaps;
  p.out = reinterpret_cast<__half*>(o.base); p.out_pitch = o.pitch; p.out_coff = o.coff; p.Cout = N;
  p.a_stride = 1; p.mask_y = nullptr; p.mask_pitch = 0; p.mask_coff = 0;
  p.kchunks_a1 = (K + BLOCK_K - 1) / BLOCK_K; p.K1 = K; p.n_split = 1 << 30; p.out2 = p.out; p.out2_pitch = o.pitch; p.out2_coff = o.coff;
  {
    cuuint64_t dims[4] = {(cuuint64_t)K, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)a.pitch * 2, (cuuint64_t)a.W * a.pitch * 2, (cuuint64_t)a.H * a.W * a.pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.bw, (cuuint32_t)p.bh, (cuuint32_t)p.bf};
    if (int rc = encode(ctx, &plan.tmap_a, 4, reinterpret_cast<__half*>(a.base) + a.coff, dims, str, box)) return rc;
    plan.tmap_a_lo = plan.tmap_a;
    if (a.lo_off)
      if (int rc = encode(ctx, &plan.tmap_a_lo, 4, reinterpret_cast<__half*>(reinterpret_cast<char*>(a.base) + a.lo_off) + a.coff, dims, str, box)) return rc;
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)N, (cuuint64_t)ntaps};
    cuuint64_t str[2] = {(cuuint64_t)K * 2, (cuuint64_t)N * K * 2};
    cuuint32_t box[3] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.block_n, 1};
    if (int rc = encode(ctx, &plan.tmap_b, 3, const_cast<__half*>(w), dims, str, box)) return rc;
    plan.b_lo_off = tc ? tc->w_lo_off : 0;
    plan.tmap_b_lo = plan.tmap_b;
    if (plan.b_lo_off)
      if (int rc = encode(ctx, &plan.tmap_b_lo, 3, reinterpret_cast<__half*>(reinterpret_cast<char*>(const_cast<__half*>(w)) + plan.b_lo_off), dims, str, box)) return rc;
  }
  plan.tmap_a2 = plan.tmap_a; plan.tmap_a2_lo = plan.tmap_a_lo;
  // SSNB_EXACT_TC: three products per (tap, K chunk) from a four-plane stage, fp32 epilogue (+ fp16 operand planes of the result)
  p.nseg = tc ? 3 : 1; p.out_f32 = tc ? 1 : 0;
  // a stage holds one (tap, K chunk) of A and B; EXACT_TC: of both planes of each
  p.stage_bytes = ((A_BYTES + p.block_n * BLOCK_K * 2) * (tc ? 2 : 1) + 1023) / 1024 * 1024;
  p.stages = PIPE_BYTES / p.stage_bytes; if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
  p.alpha = tc ? tc->alpha : 1.0f; p.alpha_dev = tc ? tc->alpha_dev : nullptr;
  p.mask32 = nullptr; p.mask32_pitch = 0; p.mask32_coff = 0; p.plane_scale = 1.0f; p.flag = nullptr;
  p.out32 = tc ? tc->out32 : nullptr;
  if (tc && (!tc->out32 || !a.lo_off || !tc->w_lo_off)) { set_thread_error("umma conv: split-operand bind needs operand planes and an fp32 output"); return 1; }
  if (int rc = bind_out(ctx, plan, o, p.out32, N, false)) return rc;
  // second destination = the first unless a fused bind redirects it
  p.out32_2 = p.out32; p.planes2 = p.planes; p.out2_lo = p.out_lo;
  plan.tmap_o2 = plan.tmap_o; plan.tmap_o2_hi = plan.tmap_o_hi; plan.tmap_o2_lo = plan.tmap_o_lo;
  plan.enabled = true;
  return 0;
}

// UmmaConvParams::tc_ok: stride-1 layers of 1, 4 or 9 taps on images at least 7 pixels wide whose outputs are 32-byte
// aligned NHWC slices; a fused sibling data gradient (two K sources) only as a 1x1 layer.  Which EXACT_TC launches require
// it: ssnb_set_workspace (engine.cu).
void mark_tc_ok(UmmaConvPlan& plan, int W, bool two_sources) {
  UmmaConvParams& p = plan.p;
  p.tc_ok = 0;
  if (!plan.enabled || p.a_stride != 1) return;
  if (!(p.ntaps == 1 || p.ntaps == 4 || p.ntaps == 9)) return;
  if (p.kchunks_a1 != p.kchunks && (p.ntaps != 1 || !two_sources)) return;
  if (p.out_pitch % 16 || p.out_coff % 16 || p.out2_pitch % 16 || p.out2_coff % 16 || p.n_split % 16 || (p.bias && p.n_tiles * p.block_n > 1024)) return;
  if (W < 7) return;
  p.tc_ok = 1;
}

}  // namespace

int umma_resolve_encode(UmmaContext& ctx) { return resolve_encode(ctx); }
int umma_encode_f16(UmmaContext& ctx, CUtensorMap* m, int rank, void* addr, const cuuint64_t* dims,
                    const cuuint64_t* strides, const cuuint32_t* box, int spatial_stride) {
  return encode(ctx, m, rank, addr, dims, strides, box, spatial_stride);
}

void umma_context_init(UmmaContext&) {}
void umma_context_destroy(UmmaContext&) {}

int umma_conv_bind_taps(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out, int F, int cin, int cout, int ntaps,
                        const int* dy, const int* dx, const __half* w_tap_n_k, const float* bias, int relu, const UmmaTcOpts* tc, int stride) {
  if (stride != 1 && stride != 2) { set_thread_error("umma conv: stride must be 1 or 2"); return 1; }
  if (int rc = bind_common(ctx, plan, in, out, F, cin, cout, ntaps, w_tap_n_k, stride, tc)) return rc;
  for (int t = 0; t < ntaps; ++t) { plan.p.tap_dy[t] = dy[t]; plan.p.tap_dx[t] = dx[t]; }
  plan.p.bias = bias; plan.p.relu = relu; plan.p.accumulate = 0;
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_fwd(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out, int F, int cin, int cout, int k, int pad,
                       int stride, const __half* w_tap_n_k, const float* bias, const UmmaTcOpts* tc) {
  // a stride-2 layer (k=3, pad=1): tiles over OUTPUT pixels whose A boxes step over the input with TMA element stride 2
  if (stride != 1 && stride != 2) { set_thread_error("umma conv: stride must be 1 or 2"); return 1; }
  if (int rc = bind_common(ctx, plan, in, out, F, cin, cout, k * k, w_tap_n_k, stride, tc)) return rc;
  for (int r = 0; r < k; ++r)
    for (int s = 0; s < k; ++s) { plan.p.tap_dy[r * k + s] = r - pad; plan.p.tap_dx[r * k + s] = s - pad; }
  plan.p.bias = bias; plan.p.relu = 1; plan.p.accumulate = 0;
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz, View dx, int F, int cin, int cout, int k, int pad,
                         const __half* w_tap_k_n, int accumulate, const UmmaTcOpts* tc) {
  // dx[p, ci] = sum_{r,s,co} dz[p + (pad-r, pad-s), co] * W[co][ci][r][s] : K = cout, N = cin
  if (int rc = bind_common(ctx, plan, dz, dx, F, cout, cin, k * k, w_tap_k_n, 1, tc)) return rc;
  for (int r = 0; r < k; ++r)
    for (int s = 0; s < k; ++s) { plan.p.tap_dy[r * k + s] = pad - r; plan.p.tap_dx[r * k + s] = pad - s; }
  plan.p.bias = nullptr; plan.p.relu = 0; plan.p.accumulate = accumulate;
  mark_tc_ok(plan, dz.W, false);
  return 0;
}

int umma_conv_bind_fused_fwd(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out1, View out2, int F, int cin, int n1, int n2,
                             const __half* w_n_k, const float* bias, const UmmaTcOpts* tc) {
  // bind as one convolution with N = n1 + n2 writing to out1's geometry, then redirect columns >= n1
  View o = out1; o.C = n1 + n2;
  if (out1.H != out2.H || out1.W != out2.W || n1 % 16 || n2 % 16 || out2.pitch % 8 || out2.coff % 8) { set_thread_error("fused fwd: bad views"); return 1; }
  if (tc && !tc->out32_2) { set_thread_error("fused fwd: the split-operand bind needs both fp32 destinations"); return 1; }
  if (int rc = bind_common(ctx, plan, in, o, F, cin, n1 + n2, 1, w_n_k, 1, tc)) return rc;
  plan.p.tap_dy[0] = 0; plan.p.tap_dx[0] = 0;
  plan.p.bias = bias; plan.p.relu = 1; plan.p.accumulate = 0;
  plan.p.n_split = n1; plan.p.out2 = reinterpret_cast<__half*>(out2.base); plan.p.out2_pitch = out2.pitch; plan.p.out2_coff = out2.coff;
  // EXACT_TC: out1 / out2 are the operand-plane views of the two destinations, tc->out32 / out32_2 their fp32 buffers.  Each
  // destination's maps end at its own channel count, so TMA clips there.
  if (tc) plan.p.out32_2 = tc->out32_2;
  if (int rc = bind_out(ctx, plan, out1, plan.p.out32, n1, false)) { plan.enabled = false; return rc; }
  if (int rc = bind_out(ctx, plan, out2, plan.p.out32_2, n2, true)) { plan.enabled = false; return rc; }
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_fused_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz1, View dz2, View dx, int F, int cin, int k1, int k2,
                               const __half* w_n_k, int accumulate, const UmmaTcOpts* tc) {
  const int k1p = (k1 + BLOCK_K - 1) / BLOCK_K * BLOCK_K;
  // bind with the first source as the A view and the full fused K; then attach the second source
  View a = k1 ? dz1 : dz2;
  if (int rc = bind_common(ctx, plan, a, dx, F, k1 ? k1 : k2, cin, 1, w_n_k, 1, tc)) return rc;
  UmmaConvParams& p = plan.p;
  p.tap_dy[0] = 0; p.tap_dx[0] = 0; p.bias = nullptr; p.relu = 0; p.accumulate = accumulate;
  if (k1) {
    if (dz2.H != dz1.H || dz2.W != dz1.W || dz2.pitch % 8 || dz2.coff % 8 || k2 % 8) { set_thread_error("fused dgrad: bad views"); return 1; }
    cuuint64_t dims[4] = {(cuuint64_t)k2, (cuuint64_t)dz2.W, (cuuint64_t)dz2.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)dz2.pitch * 2, (cuuint64_t)dz2.W * dz2.pitch * 2, (cuuint64_t)dz2.H * dz2.W * dz2.pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.bw, (cuuint32_t)p.bh, (cuuint32_t)p.bf};
    if (int rc = encode(ctx, &plan.tmap_a2, 4, reinterpret_cast<__half*>(dz2.base) + dz2.coff, dims, str, box)) { plan.enabled = false; return rc; }
    p.kchunks_a1 = k1p / BLOCK_K; p.K1 = k1; p.K = k1 + k2;
    p.kchunks = p.kchunks_a1 + (k2 + BLOCK_K - 1) / BLOCK_K;
    // the weight map covers the padded fused K
    cuuint64_t bd[3] = {(cuuint64_t)(k1p + k2), (cuuint64_t)cin, 1};
    cuuint64_t bs[2] = {(cuuint64_t)(k1p + k2) * 2, (cuuint64_t)cin * (k1p + k2) * 2};
    cuuint32_t bb[3] = {(cuuint32_t)BLOCK_K, (cuuint32_t)p.block_n, 1};
    if (int rc = encode(ctx, &plan.tmap_b, 3, const_cast<__half*>(w_n_k), bd, bs, bb)) { plan.enabled = false; return rc; }
    plan.tmap_b_lo = plan.tmap_b;
    if (plan.b_lo_off)
      if (int rc = encode(ctx, &plan.tmap_b_lo, 3, reinterpret_cast<__half*>(reinterpret_cast<char*>(const_cast<__half*>(w_n_k)) + plan.b_lo_off), bd, bs, bb)) {
        plan.enabled = false; return rc; }
    if (tc && !dz2.lo_off) { set_thread_error("fused dgrad: the split-operand bind needs the second source's operand planes"); plan.enabled = false; return 1; }
    // the second source's LO plane
    plan.tmap_a2_lo = plan.tmap_a2;
    if (dz2.lo_off)
      if (int rc = encode(ctx, &plan.tmap_a2_lo, 4, reinterpret_cast<__half*>(reinterpret_cast<char*>(dz2.base) + dz2.lo_off) + dz2.coff, dims, str, box)) {
        plan.enabled = false; return rc; }
  }
  mark_tc_ok(plan, a.W, k1 != 0);
  return 0;
}

void umma_conv_set_mask(UmmaConvPlan& plan, View y) {
  plan.mask_y = reinterpret_cast<const __half*>(y.base); plan.mask_pitch = y.pitch; plan.mask_coff = y.coff;
}

int umma_conv_set_mask_tc(UmmaContext& ctx, UmmaConvPlan& plan, View y32, View dplanes, float plane_scale, int* flag) {
  // a data gradient has one destination: the planes replace the first destination's
  if (int rc = encode_planes(ctx, &plan.tmap_mask_hi, &plan.tmap_mask_lo, plan.p, reinterpret_cast<__half*>(dplanes.base) + dplanes.coff, dplanes.lo_off,
                             dplanes.pitch, plan.p.Cout)) return rc;
  plan.mask32 = reinterpret_cast<const float*>(y32.base); plan.mask32_pitch = y32.pitch; plan.mask32_coff = y32.coff;
  plan.mask_planes = true; plan.mask_plane_scale = plane_scale; plan.mask_flag = flag;
  return 0;
}

namespace {
template <int BN, bool DIRECT>
int launch_bn(const UmmaConvPlan& plan, const UmmaConvParams& p, const CUtensorMap& o_hi, const CUtensorMap& o_lo, int grid, cudaStream_t s) {
  static bool attr_set[64] = {};          // function attributes are per device
  auto kern = DIRECT ? umma_conv_tail_kernel<BN> : umma_conv_kernel<BN>;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) {
      set_thread_error("umma conv: cannot raise dynamic shared memory limit"); cudaGetLastError(); return 2; }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  kern<<<grid, NUM_THREADS, SMEM_BYTES, s>>>(plan.tmap_a, plan.tmap_a2, plan.tmap_b, plan.tmap_a_lo, plan.tmap_a2_lo, plan.tmap_b_lo, plan.tmap_o, o_hi, o_lo,
                                             plan.tmap_o2, plan.tmap_o2_hi, plan.tmap_o2_lo, p);
  SSNB_LAUNCH_CHECK("umma_conv_kernel");      // both kernels: the launch log names the convolution kernel
  return 0;
}
template <int BN>
int launch_bn(const UmmaConvPlan& plan, const UmmaConvParams& p, const CUtensorMap& o_hi, const CUtensorMap& o_lo, int grid, cudaStream_t s) {
  return p.f_direct < (1 << 30) ? launch_bn<BN, true>(plan, p, o_hi, o_lo, grid, s) : launch_bn<BN, false>(plan, p, o_hi, o_lo, grid, s);
}
}  // namespace

int umma_conv_launch(UmmaContext& ctx, const UmmaConvPlan& plan, cudaStream_t s, bool mask, int frames) {
  if (!plan.enabled) { set_thread_error("umma conv: plan not bound"); return 3; }
  UmmaConvParams p = plan.p;
  if (frames && frames != p.F) {
    // n < F frames on the maps bound for F: frame boxes stay outermost in decode_tile, so the first ceil(n / bf) of them are
    // the whole launch; the box that straddles n is stored row by row (f_direct)
    if (frames < 1 || frames > p.F || mask || p.accumulate) { set_thread_error("umma conv: a frame count below the plan's runs forward plans only"); return 3; }
    p.F = frames;
    p.tiles_f = (frames + p.bf - 1) / p.bf;
    if (frames % p.bf) p.f_direct = frames - frames % p.bf;
  }
  if (mask && plan.mask_y) { p.mask_y = plan.mask_y; p.mask_pitch = plan.mask_pitch; p.mask_coff = plan.mask_coff; }
  const bool mplanes = mask && p.out_f32 && plan.mask32 && plan.mask_planes;
  if (mplanes) {
    p.mask32 = plan.mask32; p.mask32_pitch = plan.mask32_pitch; p.mask32_coff = plan.mask32_coff;
    p.planes = 1; p.plane_scale = plan.mask_plane_scale; p.flag = plan.mask_flag;
  }
  if (p.out_f32 && p.mask_y) { set_thread_error("umma conv: the fp32 epilogue takes its mask through mask32"); return 3; }
  const CUtensorMap& o_hi = mplanes ? plan.tmap_mask_hi : plan.tmap_o_hi;
  const CUtensorMap& o_lo = mplanes ? plan.tmap_mask_lo : plan.tmap_o_lo;
  const int total = p.tiles_w * p.tiles_h * p.tiles_f * p.n_tiles;
  const int grid = total < ctx.num_sms ? total : ctx.num_sms;
  t_tag.tiles = total; t_tag.block_n = p.block_n;
  switch (p.block_n) {
    case 16: return launch_bn<16>(plan, p, o_hi, o_lo, grid, s);
    case 32: return launch_bn<32>(plan, p, o_hi, o_lo, grid, s);
    case 48: return launch_bn<48>(plan, p, o_hi, o_lo, grid, s);
    case 64: return launch_bn<64>(plan, p, o_hi, o_lo, grid, s);
    case 80: return launch_bn<80>(plan, p, o_hi, o_lo, grid, s);
    case 96: return launch_bn<96>(plan, p, o_hi, o_lo, grid, s);
    case 112: return launch_bn<112>(plan, p, o_hi, o_lo, grid, s);
    case 128: return launch_bn<128>(plan, p, o_hi, o_lo, grid, s);
  }
  set_thread_error("umma conv: unsupported tile width"); return 3;
}

}  // namespace ssnb
