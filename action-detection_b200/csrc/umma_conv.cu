// wgmma implicit-GEMM convolution (sm_90a): host-side planning and the kernel that runs every tensor-core convolution
// (forward, data gradient, fused sibling 1x1 forward / data gradient, stride-2 forward through TMA element strides).
//
//   warpgroup 0     : TMA producer (one thread; A: 4-D activation box, B: 3-D weight box, SWIZZLE_128B), stages in tile order
//   warpgroups 1, 2 : ping-pong consumers -- each owns every other tile of the CTA's persistent sequence, all 128 rows: two
//                     m64nNk16 wgmmas (N = block_n <= 128) per 16 channels, fp32 accumulators in registers; then the
//                     epilogue: each 32-column slice of the accumulator goes through the warpgroup's own shared-memory
//                     staging so that every thread owns one output row (bias/ReLU or accumulate/mask -> fp16 NHWC stores,
//                     or the SSNB_EXACT_TC fp32 epilogue of umma_epi32.cuh).  An order barrier hands the tensor pipe from
//                     one warpgroup to the other once a tile's MMAs are issued, so one tile's epilogue runs under the
//                     next tile's MMAs.
//
// Rows of the M tile are the pixels of one TMA box (bw x bh x bf); taps shift the box origin and
// rely on TMA's out-of-bounds zero fill for the convolution padding.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>

#include "umma_conv.cuh"
#include "umma_dev.cuh"
#include "umma_epi32.cuh"

namespace ssnb {

namespace {

using namespace umma;
constexpr int MAX_STAGES = 8;
constexpr int PIPE_BYTES = 192 * 1024;             // operand staging: 3 four-plane EXACT_TC stages at block_n 128
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;     // 16 KiB
constexpr int NUM_THREADS = 384;
constexpr int N_STEP = 16;                         // block_n granularity (wgmma N is any multiple of 8; the epilogue works in 16-column chunks)
constexpr int MAX_BLOCK_N = 128;                   // 128 accumulators per consumer thread
constexpr int EPI_COLS = 16;                       // accumulator columns per staged epilogue slice
constexpr int EPI_PITCH = EPI_COLS + 4;            // floats per staged row (16-byte aligned, banks rotate)
constexpr int EPI_BYTES = BLOCK_M * EPI_PITCH * 4; // per consumer warpgroup: 10 KiB
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

// bias / accumulate / ReLU / ReLU-gradient mask on one 16-column chunk of an accumulator row, then fp16 store
__device__ __forceinline__ void epilogue_chunk(const UmmaConvParams& p, const uint32_t* r, int col, uint4* dst, const uint4& o0,
                                               const uint4& o1, const uint4& y0, const uint4& y1) {
  float v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
  if (p.bias) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] += __ldg(p.bias + col + j);
  }
  if (p.accumulate) {
    const __half2* h0 = reinterpret_cast<const __half2*>(&o0);
    const __half2* h1 = reinterpret_cast<const __half2*>(&o1);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 a = __half22float2(h0[j]), b = __half22float2(h1[j]);
      v[2 * j] += a.x; v[2 * j + 1] += a.y; v[8 + 2 * j] += b.x; v[8 + 2 * j + 1] += b.y;
    }
  }
  if (p.relu) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  if (p.mask_y) {
    const __half2* a0 = reinterpret_cast<const __half2*>(&y0);
    const __half2* a1 = reinterpret_cast<const __half2*>(&y1);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 ya = __half22float2(a0[j]), yb = __half22float2(a1[j]);
      if (!(ya.x > 0.f)) v[2 * j] = 0.f;
      if (!(ya.y > 0.f)) v[2 * j + 1] = 0.f;
      if (!(yb.x > 0.f)) v[8 + 2 * j] = 0.f;
      if (!(yb.y > 0.f)) v[8 + 2 * j + 1] = 0.f;
    }
  }
  uint4 q0, q1;
  __half2* g0 = reinterpret_cast<__half2*>(&q0);
  __half2* g1 = reinterpret_cast<__half2*>(&q1);
#pragma unroll
  for (int j = 0; j < 4; ++j) { g0[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]); g1[j] = __floats2half2_rn(v[8 + 2 * j], v[8 + 2 * j + 1]); }
  dst[0] = q0; dst[1] = q1;
}

// One 16-column chunk (tile columns [c, c + 16)) of accumulator row `row`, read from the staged slice `st`.
// Row r of the tile is pixel (x, y, f) = (r % bw, (r / bw) % bh, r / (bw*bh)).
__device__ __forceinline__ void epilogue_row_chunk(const UmmaConvParams& p, const TileCoord& t, int row, int col, const float* st) {
  const int rw = row % p.bw, rh = (row / p.bw) % p.bh, rf = row / (p.bw * p.bh);
  const int w = t.w0 + rw, h = t.h0 + rh, f = t.f0 + rf;
  const int os = p.out_stride;
  const bool valid = (rf < p.bf) && (w < p.W) && (h < p.H) && (f < p.F) && (w % os == 0) && (h % os == 0);
  if (!valid || col >= p.Cout) return;
  const long long opix = (long long)(f * p.OH + h / os) * p.OW + w / os;
  uint32_t r[16];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 q = reinterpret_cast<const float4*>(st)[j];
    r[4 * j] = __float_as_uint(q.x); r[4 * j + 1] = __float_as_uint(q.y); r[4 * j + 2] = __float_as_uint(q.z); r[4 * j + 3] = __float_as_uint(q.w);
  }
  const bool d1 = col < p.n_split;
  if (p.out_f32) {
    // SSNB_EXACT_TC: fp32 epilogue + the result's fp16 hi / lo operand planes (umma_epi32.cuh); a fused sibling forward sends
    // columns >= n_split to the second destination (its own pitch / channel offset)
    const float alpha = p.alpha * (p.alpha_dev ? __ldg(p.alpha_dev) : 1.0f);
    float* o32 = d1 ? p.out32 + opix * p.out_pitch + p.out_coff + col : p.out32_2 + opix * p.out2_pitch + p.out2_coff - p.n_split + col;
    __half* hi = d1 ? p.out_hi : p.out_hi2;
    if (hi) hi += d1 ? opix * p.out_pitch + p.out_coff + col : opix * p.out2_pitch + p.out2_coff - p.n_split + col;
    const float* m32 = p.mask32 ? p.mask32 + opix * p.mask32_pitch + p.mask32_coff + col : nullptr;
    store_chunk32(p, alpha, r, p.bias + col, o32, hi, m32, d1 ? p.out_lo_off : p.out_lo_off2);
    return;
  }
  uint4* dst = reinterpret_cast<uint4*>(d1 ? p.out + opix * p.out_pitch + p.out_coff + col : p.out2 + opix * p.out2_pitch + p.out2_coff - p.n_split + col);
  uint4 o0 = {}, o1 = {}, y0 = {}, y1 = {};
  if (p.accumulate) { o0 = dst[0]; o1 = dst[1]; }
  if (p.mask_y) {
    const uint4* my = reinterpret_cast<const uint4*>(p.mask_y + opix * p.mask_pitch + p.mask_coff + col);
    y0 = __ldg(my); y1 = __ldg(my + 1);
  }
  epilogue_chunk(p, r, col, dst, o0, o1, y0, y1);
}

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

// BN = block_n: a multiple of 16, at most 128 (BN accumulators per consumer thread)
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
umma_conv_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2,
                 const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_a_lo,
                 const __grid_constant__ CUtensorMap tmap_a2_lo, const __grid_constant__ CUtensorMap tmap_b_lo,
                 const __grid_constant__ UmmaConvParams p) {
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
    float* epi = reinterpret_cast<float*>(smem + PIPE_BYTES + cw * EPI_BYTES);
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
      // epilogue, one EPI_COLS-column slice at a time: fragments -> this warpgroup's staging -> one row per thread
#pragma unroll
      for (int sl = 0; sl < (BN + EPI_COLS - 1) / EPI_COLS; ++sl) {
        named_bar_sync(EPI_BAR + cw, 128);               // the previous slice (or tile) has been read
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int i = 0; i < EPI_COLS / 2; i += 2) {
            const int ai = sl * (EPI_COLS / 2) + i;      // accumulator registers [16 sl, 16 sl + 16) are slice sl's columns
            if (ai < BN / 2) {
              const int r = b * 64 + warp * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
              const int c = 8 * (i >> 2) + 2 * (lane & 3);
              *reinterpret_cast<float2*>(epi + r * EPI_PITCH + c) = make_float2(acc[b][ai], acc[b][ai + 1]);
            }
          }
        named_bar_sync(EPI_BAR + cw, 128);
#pragma unroll
        for (int c = 0; c < EPI_COLS; c += 16)
          if (sl * EPI_COLS + c < BN) epilogue_row_chunk(p, t, row, t.n0 + sl * EPI_COLS + c, epi + row * EPI_PITCH + c);
      }
    }
  }
}

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
           const cuuint32_t* box, int spatial_stride = 1) {
  // spatial_stride 2: the box traverses W and H with step 2 (box extents are given in un-strided elements)
  cuuint32_t es[5] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1, 1};
  CUresult r = reinterpret_cast<EncodeTiledFn>(ctx.encode_tiled)(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, addr, dims, strides,
                                                                box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
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

int bind_common(UmmaContext& ctx, UmmaConvPlan& plan, View a, View o, int F, int K, int N, int ntaps, int out_stride, const __half* w,
                int a_stride = 1, const UmmaTcOpts* tc = nullptr) {
  plan.enabled = false;
  if (int rc = resolve_encode(ctx)) return rc;
  if (a_stride == 2) {
    // strided TMA: tiles enumerate OUTPUT pixels, the A box steps over the input with stride 2
    View ao = a; ao.H = o.H; ao.W = o.W;
    if (int rc = bind_common(ctx, plan, ao, o, F, K, N, ntaps, 1, w, 1, tc)) return rc;
    plan.enabled = false;
    UmmaConvParams& q = plan.p;
    q.a_stride = 2;
    cuuint64_t dims[4] = {(cuuint64_t)K, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)a.pitch * 2, (cuuint64_t)a.W * a.pitch * 2, (cuuint64_t)a.H * a.W * a.pitch * 2};
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)(2 * q.bw), (cuuint32_t)(2 * q.bh), (cuuint32_t)q.bf};
    if (int rc = encode(ctx, &plan.tmap_a, 4, reinterpret_cast<__half*>(a.base) + a.coff, dims, str, box, 2)) return rc;
    plan.tmap_a_lo = plan.tmap_a;
    if (a.lo_off)
      if (int rc = encode(ctx, &plan.tmap_a_lo, 4, reinterpret_cast<__half*>(reinterpret_cast<char*>(a.base) + a.lo_off) + a.coff, dims, str, box, 2)) return rc;
    plan.tmap_a2 = plan.tmap_a; plan.tmap_a2_lo = plan.tmap_a_lo;
    plan.enabled = true;
    return 0;
  }
  if ((a.H + out_stride - 1) / out_stride != o.H || (a.W + out_stride - 1) / out_stride != o.W) { set_thread_error("umma conv: geometry mismatch"); return 1; }
  if (K % 8 || N % 16 || a.pitch % 8 || a.coff % 8 || o.pitch % 8 || o.coff % 8 || ntaps > UMMA_MAX_TAPS) {
    set_thread_error("umma conv: unsupported channel alignment"); return 1; }
  UmmaConvParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  p.W = a.W; p.H = a.H; p.F = F;
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
  p.out_stride = out_stride; p.OH = o.H; p.OW = o.W; p.a_stride = 1; p.mask_y = nullptr; p.mask_pitch = 0; p.mask_coff = 0;
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
  p.out32 = tc ? tc->out32 : nullptr; p.out_hi = tc ? reinterpret_cast<__half*>(o.base) : nullptr; p.out_lo_off = tc ? o.lo_off : 0;
  p.out32_2 = p.out32; p.out_hi2 = p.out_hi; p.out_lo_off2 = p.out_lo_off;       // second destination = the first unless a fused bind redirects it
  if (tc && (!tc->out32 || !a.lo_off || !tc->w_lo_off)) { set_thread_error("umma conv: split-operand bind needs operand planes and an fp32 output"); return 1; }
  plan.enabled = true;
  return 0;
}

// UmmaConvParams::tc_ok: stride-1 layers of 1, 4 or 9 taps on images at least 7 pixels wide whose outputs are 32-byte
// aligned NHWC slices; a fused sibling data gradient (two K sources) only as a 1x1 layer.  Which EXACT_TC launches require
// it: ssnb_set_workspace (engine.cu).
void mark_tc_ok(UmmaConvPlan& plan, int W, bool two_sources) {
  UmmaConvParams& p = plan.p;
  p.tc_ok = 0;
  if (!plan.enabled || p.a_stride != 1 || p.out_stride != 1) return;
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
                        const int* dy, const int* dx, const __half* w_tap_n_k, const float* bias, int relu, const UmmaTcOpts* tc) {
  if (int rc = bind_common(ctx, plan, in, out, F, cin, cout, ntaps, 1, w_tap_n_k, 1, tc)) return rc;
  for (int t = 0; t < ntaps; ++t) { plan.p.tap_dy[t] = dy[t]; plan.p.tap_dx[t] = dx[t]; }
  plan.p.bias = bias; plan.p.relu = relu; plan.p.accumulate = 0;
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_fwd(UmmaContext& ctx, UmmaConvPlan& plan, View in, View out, int F, int cin, int cout, int k, int pad,
                       int stride, const __half* w_tap_n_k, const float* bias, const UmmaTcOpts* tc) {
  // a stride-2 layer (k=3, pad=1): tiles over OUTPUT pixels whose A boxes step over the input with TMA element
  // stride 2 (default), or the stride-1 convolution sampled at even pixels (4x redundant MMAs, SSNB_TMA_STRIDED=0)
  const char* st = getenv("SSNB_TMA_STRIDED");           // default on; "0" falls back to the sampled-epilogue variant
  const bool strided = stride == 2 && !(st && st[0] == '0');
  if (int rc = strided ? bind_common(ctx, plan, in, out, F, cin, cout, k * k, 1, w_tap_n_k, 2, tc)
                       : bind_common(ctx, plan, in, out, F, cin, cout, k * k, stride, w_tap_n_k, 1, tc)) return rc;
  for (int r = 0; r < k; ++r)
    for (int s = 0; s < k; ++s) { plan.p.tap_dy[r * k + s] = r - pad; plan.p.tap_dx[r * k + s] = s - pad; }
  plan.p.bias = bias; plan.p.relu = 1; plan.p.accumulate = 0;
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz, View dx, int F, int cin, int cout, int k, int pad,
                         const __half* w_tap_k_n, int accumulate, const UmmaTcOpts* tc) {
  // dx[p, ci] = sum_{r,s,co} dz[p + (pad-r, pad-s), co] * W[co][ci][r][s] : K = cout, N = cin
  if (int rc = bind_common(ctx, plan, dz, dx, F, cout, cin, k * k, 1, w_tap_k_n, 1, tc)) return rc;
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
  if (int rc = bind_common(ctx, plan, in, o, F, cin, n1 + n2, 1, 1, w_n_k, 1, tc)) return rc;
  plan.p.tap_dy[0] = 0; plan.p.tap_dx[0] = 0;
  plan.p.bias = bias; plan.p.relu = 1; plan.p.accumulate = 0;
  plan.p.n_split = n1; plan.p.out2 = reinterpret_cast<__half*>(out2.base); plan.p.out2_pitch = out2.pitch; plan.p.out2_coff = out2.coff;
  if (tc) {        // EXACT_TC: out1 / out2 are the operand-plane views of the two destinations, tc->out32 / out32_2 their fp32 buffers
    if (!tc->out32_2) { set_thread_error("fused fwd: the split-operand bind needs both fp32 destinations"); return 1; }
    plan.p.out32_2 = tc->out32_2; plan.p.out_hi2 = reinterpret_cast<__half*>(out2.base); plan.p.out_lo_off2 = out2.lo_off;
  }
  mark_tc_ok(plan, in.W, false);
  return 0;
}

int umma_conv_bind_fused_dgrad(UmmaContext& ctx, UmmaConvPlan& plan, View dz1, View dz2, View dx, int F, int cin, int k1, int k2,
                               const __half* w_n_k, int accumulate, const UmmaTcOpts* tc) {
  const int k1p = (k1 + BLOCK_K - 1) / BLOCK_K * BLOCK_K;
  // bind with the first source as the A view and the full fused K; then attach the second source
  View a = k1 ? dz1 : dz2;
  if (int rc = bind_common(ctx, plan, a, dx, F, k1 ? k1 : k2, cin, 1, 1, w_n_k, 1, tc)) return rc;
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

void umma_conv_set_mask_tc(UmmaConvPlan& plan, View y32, View dplanes, float plane_scale, int* flag) {
  plan.mask32 = reinterpret_cast<const float*>(y32.base); plan.mask32_pitch = y32.pitch; plan.mask32_coff = y32.coff;
  plan.mask_planes = reinterpret_cast<__half*>(dplanes.base); plan.mask_planes_lo = dplanes.lo_off;
  plan.mask_plane_scale = plane_scale; plan.mask_flag = flag;
}

namespace {
template <int BN>
int launch_bn(const UmmaConvPlan& plan, const UmmaConvParams& p, int grid, cudaStream_t s) {
  static bool attr_set[64] = {};          // function attributes are per device
  auto kern = umma_conv_kernel<BN>;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) {
      set_thread_error("umma conv: cannot raise dynamic shared memory limit"); cudaGetLastError(); return 2; }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  kern<<<grid, NUM_THREADS, SMEM_BYTES, s>>>(plan.tmap_a, plan.tmap_a2, plan.tmap_b, plan.tmap_a_lo, plan.tmap_a2_lo, plan.tmap_b_lo, p);
  SSNB_LAUNCH_CHECK("umma_conv_kernel");
  return 0;
}
}  // namespace

int umma_conv_launch(UmmaContext& ctx, const UmmaConvPlan& plan, cudaStream_t s, bool mask) {
  if (!plan.enabled) { set_thread_error("umma conv: plan not bound"); return 3; }
  UmmaConvParams p = plan.p;
  if (mask && plan.mask_y) { p.mask_y = plan.mask_y; p.mask_pitch = plan.mask_pitch; p.mask_coff = plan.mask_coff; }
  if (mask && p.out_f32 && plan.mask32) {
    p.mask32 = plan.mask32; p.mask32_pitch = plan.mask32_pitch; p.mask32_coff = plan.mask32_coff;
    p.out_hi = plan.mask_planes; p.out_lo_off = plan.mask_planes_lo; p.plane_scale = plan.mask_plane_scale; p.flag = plan.mask_flag;
  }
  if (p.out_f32 && (p.mask_y || p.out_stride != 1)) { set_thread_error("umma conv: the fp32 epilogue takes its mask through mask32 and has no sampling"); return 3; }
  const int total = p.tiles_w * p.tiles_h * p.tiles_f * p.n_tiles;
  const int grid = total < ctx.num_sms ? total : ctx.num_sms;
  t_tag.tiles = total; t_tag.block_n = p.block_n;
  switch (p.block_n) {
    case 16: return launch_bn<16>(plan, p, grid, s);
    case 32: return launch_bn<32>(plan, p, grid, s);
    case 48: return launch_bn<48>(plan, p, grid, s);
    case 64: return launch_bn<64>(plan, p, grid, s);
    case 80: return launch_bn<80>(plan, p, grid, s);
    case 96: return launch_bn<96>(plan, p, grid, s);
    case 112: return launch_bn<112>(plan, p, grid, s);
    case 128: return launch_bn<128>(plan, p, grid, s);
  }
  set_thread_error("umma conv: unsupported tile width"); return 3;
}

}  // namespace ssnb
