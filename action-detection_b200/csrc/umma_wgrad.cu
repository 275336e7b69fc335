// wgmma weight-gradient kernel (sm_90a).  dW[tap][co][ci] = sum_p dz[p, co] * x[p + shift(tap), ci]
// is a GEMM whose reduction runs over pixels, so both operands are MN-major in shared memory:
// a TMA box is [64 pixels][64 channels] (128-byte rows, SWIZZLE_128B) and the wgmma descriptors walk
// it with 8-pixel groups every 1024 B (SBO).
//
//   CTA = (co tile of 128, ci tile of block_n <= 256, taps, pixel split); K loop over 64-pixel boxes (EXACT_TC: 32-pixel halves).
//   warpgroup 0: TMA producer; warpgroups 1, 2: co rows [64 * (wg - 1), +64), one m64nNk16 wgmma per 16 pixels covering
//   every (tap, 64 input channels) block of the CTA, fp32 accumulators in registers -> split-K partials (reduced in fixed order by wgrad_finalize_kernel).
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>

#include "umma_conv.cuh"
#include "umma_dev.cuh"

namespace ssnb {
namespace {

using namespace umma;
constexpr int MAX_STAGES = 8;
constexpr int BOX_BYTES = 64 * 128;                 // [64 px][64 ch] fp16: one pixel tile of one 64-channel atom
constexpr int PIPE_BYTES = 192 * 1024;              // operand staging, cut into p.stages stages of p.stage_bytes
constexpr int NUM_THREADS = 384;
constexpr int ONES_OFF = PIPE_BYTES + 1024;                // [16 rows][64 px] of fp16 ones (bias-gradient operand), 1 KiB aligned
constexpr int ONES_BYTES = 16 * 128;
constexpr int SMEM_BYTES = PIPE_BYTES + 1024 /*align slack*/ + 1024 /*barriers*/ + ONES_BYTES;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");

// D[64 co][NACC * 64] += dz^T x over the PX pixels of one stage: one m64n(64 NACC)k16 MMA per 16 pixel rows.  The x boxes of all
// taps of the CTA are consecutive 64-channel N atoms PX * 128 bytes apart (the LBO), so the dz rows are read from shared memory
// once per 16 pixels.
template <int NACC, int PX>
__device__ __forceinline__ void mma_px(float* acc, uint32_t dz, uint32_t x) {
#pragma unroll
  for (int k = 0; k < PX / MMA_K; ++k)
    wgmma<NACC * MMA_N, 1, 1>(acc, make_desc_sw128(dz + k * (MMA_K * 128), PX * 128), make_desc_sw128(x + k * (MMA_K * 128), PX * 128));
}

// NACC = taps_per_cta * block_n / 64 accumulator blocks of 64 columns per consumer warpgroup.  NSEG = 3 (SSNB_EXACT_TC): a
// stage holds the hi and lo planes of dz and x, [dz_hi | dz_lo | x_hi | x_lo], each fetched once, for half a pixel tile (32
// pixels), so that a stage is no larger than FAST's one-plane stage of a whole tile and the ring keeps 4 to 8 stages: with
// whole-tile four-plane stages (2 of 96 KiB) the weight gradient of the EXACT_TC step took 13.1 ms instead of 9.7.
template <int NACC, int NSEG>
__global__ void __launch_bounds__(NUM_THREADS, 1)
umma_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dz, const __grid_constant__ CUtensorMap tmap_x,
                  const __grid_constant__ CUtensorMap tmap_dz_lo, const __grid_constant__ CUtensorMap tmap_x_lo,
                  const __grid_constant__ UmmaWgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + PIPE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + MAX_STAGES;
  constexpr int PLANES = NSEG == 3 ? 2 : 1;
  constexpr int PX = NSEG == 3 ? 32 : 64;            // pixels per stage
  constexpr int SUB = 64 / PX;                       // stages per pixel tile
  constexpr int BOX = PX * 128;                      // one staged box: [PX px][64 ch]

  const int wg = threadIdx.x / 128;
  int id = blockIdx.x;
  const int tgrp = id % p.tap_groups; id /= p.tap_groups;
  const int nt = id % p.n_tiles; id /= p.n_tiles;
  const int mt = id;
  const int tap0 = tgrp * p.taps_per_cta;
  const int ntap = min(p.taps_per_cta, p.ntaps - tap0);        // taps handled by this CTA (share the dz tile)
  const int split = blockIdx.y;
  const int m0 = mt * BLOCK_M, n0 = nt * p.block_n;
  const int ptiles = p.tiles_w * p.tiles_h * p.tiles_f;
  const int pt0 = split * p.ptiles_per_split;
  const int pt1 = min(pt0 + p.ptiles_per_split, ptiles);
  const int nboxes_b = p.block_n / 64;
  const int nxb = p.taps_per_cta * nboxes_b;          // x box slots of a plane
  const int x_off = 2 * PLANES * BOX;                 // stage: [dz_hi 2][dz_lo 2][x_hi nxb][x_lo nxb] boxes
  // CTAs of the first input tile / tap group also reduce dz over pixels: db[co] = sum_p dz[p, co] = dz^T * 1
  const bool do_bias = p.bias_partial != nullptr && nt == 0 && tgrp == 0;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_dz)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_x)) : "memory");
    for (int i = 0; i < MAX_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (do_bias) {
    uint32_t* ones = reinterpret_cast<uint32_t*>(smem + ONES_OFF);
    for (int i = threadIdx.x; i < ONES_BYTES / 4; i += NUM_THREADS) ones[i] = 0x3C003C00u;     // half2(1, 1)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the tensor core
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");       // programmatic dependent launch: the prologue above overlapped the previous kernel's tail
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (wg == 0) {
    producer_regs();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      // pixel-tile coordinates advance by carries (no divisions in the loop)
      int tw = pt0 % p.tiles_w, th = (pt0 / p.tiles_w) % p.tiles_h, tf = pt0 / (p.tiles_w * p.tiles_h);
      for (int pt = pt0; pt < pt1; ++pt) {
#pragma unroll 1
        for (int h = 0; h < SUB; ++h) {
          // a half tile is the lower or upper half of the box in frames (bf > 1) or else in rows
          const int w0 = tw * p.bw, h0 = th * p.bh + h * p.sub_dh, f0 = tf * p.bf + h * p.sub_df;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + stage * p.stage_bytes;
          // the second 64-row dz box of a 128-row co tile lies wholly past Cout when Cout % 128 is in (0, 64]: not fetched
          // (recomputed per stage: the producer runs on 40 registers)
          const int ndz = m0 + 64 < p.Cout ? 2 : 1;
          mbar_expect_tx(&full_bar[stage], (uint32_t)(PLANES * (ndz + nboxes_b * ntap) * BOX));
#pragma unroll 1
          for (int b = 0; b < ndz; ++b) {
            tma_load_4d(st + b * BOX, &tmap_dz, &full_bar[stage], m0 + b * 64, w0, h0, f0);
            if (NSEG == 3) tma_load_4d(st + (2 + b) * BOX, &tmap_dz_lo, &full_bar[stage], m0 + b * 64, w0, h0, f0);
          }
#pragma unroll 1
          for (int t = 0; t < ntap; ++t) {
            const int xw = w0 * p.x_stride + p.tap_dx[tap0 + t], xh = h0 * p.x_stride + p.tap_dy[tap0 + t];
            for (int b = 0; b < nboxes_b; ++b) {
              uint8_t* dst = st + x_off + (t * nboxes_b + b) * BOX;
              tma_load_4d(dst, &tmap_x, &full_bar[stage], n0 + b * 64, xw, xh, f0);
              if (NSEG == 3) tma_load_4d(dst + nxb * BOX, &tmap_x_lo, &full_bar[stage], n0 + b * 64, xw, xh, f0);
            }
          }
          if (++stage == (uint32_t)p.stages) { stage = 0; phase ^= 1; }
        }
        if (++tw == p.tiles_w) { tw = 0; if (++th == p.tiles_h) { th = 0; ++tf; } }
      }
    }
  } else {
    consumer_regs();
    const int cw = wg - 1;
    const int warp = (threadIdx.x / 32) & 3, lane = threadIdx.x & 31;
    const int nacc = ntap * nboxes_b;                 // accumulator blocks in use (<= NACC)
    uint32_t stage = 0, phase = 0, prev = 0;
    const int nstages = (pt1 - pt0) * SUB;
    if (m0 + cw * 64 >= p.Cout) {
      // all 64 co rows of this warpgroup lie past Cout: no MMAs (they would multiply zero-filled rows), it only hands the
      // stages it would have read back to the producer
      for (int i = 0; i < nstages; ++i) {
        mbar_wait(&full_bar[stage], phase);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == (uint32_t)p.stages) { stage = 0; phase ^= 1; }
      }
      return;
    }
    float acc[NACC][32], accb[8];
#pragma unroll
    for (int j = 0; j < NACC; ++j)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) accb[i] = 0.f;
    const uint32_t ones = smem_u32(smem + ONES_OFF);
    bool first = true;
    for (int i = 0; i < nstages; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t st = smem_u32(smem + stage * p.stage_bytes);
      const uint32_t dz_hi = st + cw * BOX, x_hi = st + x_off;
      // A CTA of a short last tap group (nacc < NACC) multiplies stale atoms into accumulator blocks it never stores, which
      // keeps the MMA sequence free of predication.
      wgmma_fence();
      if constexpr (NSEG == 3) {                     // small terms first, into the same registers: lo.hi, hi.lo, hi.hi
        mma_px<NACC, PX>(&acc[0][0], dz_hi + 2 * BOX, x_hi);
        mma_px<NACC, PX>(&acc[0][0], dz_hi, x_hi + nxb * BOX);
      }
      mma_px<NACC, PX>(&acc[0][0], dz_hi, x_hi);
      if (do_bias) {                                 // column sums of dz (lo plane, then hi); the ones operand is K-major
#pragma unroll
        for (int q = PLANES - 1; q >= 0; --q)
#pragma unroll
          for (int k = 0; k < PX / MMA_K; ++k)
            wgmma<16, 1, 0>(accb, make_desc_sw128(dz_hi + q * 2 * BOX + k * (MMA_K * 128), PX * 128), make_desc_sw128(ones + k * MMA_K * 2));
      }
      wgmma_commit();
      // one group stays in flight: the previous stage's MMAs have retired, its smem slot goes back to the producer
      wgmma_wait<1>();
      if (!first && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      first = false;
      prev = stage;
      if (++stage == (uint32_t)p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (!first && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
    // fragments straight to the partials: register i of this thread is row 16 warp + lane/4 + 8 ((i/2)%2), column
    // 8 (i/4) + 2 (lane%4) + i%2 of its 64 x 64 block
    const int mrow = m0 + cw * 64 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
      if (j >= nacc) break;
      const int t = j / nboxes_b, b = j % nboxes_b;
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int m = mrow + 8 * ((i >> 1) & 1);
        const int c = n0 + b * 64 + 8 * (i >> 2) + 2 * (lane & 3);
        if (m < p.Cout && c < p.Cin)      // Cin is a multiple of 8
          *reinterpret_cast<float2*>(p.partial + (((long long)split * p.ntaps + tap0 + t) * p.Cout + m) * p.Cin + c) = make_float2(acc[j][i], acc[j][i + 1]);
      }
    }
    if (do_bias && (lane & 3) == 0) {
      if (mrow < p.Cout) p.bias_partial[(long long)split * p.Cout + mrow] = accb[0];
      if (mrow + 8 < p.Cout) p.bias_partial[(long long)split * p.Cout + mrow + 8] = accb[2];
    }
  }
}

// 64-pixel boxes whose rows are all real-or-zero-filled pixels (the pixel index is the reduction dim)
void wgrad_box(int W, int& bw, int& bh, int& bf) {
  if (W % 8 == 0) { bw = 8; bh = 8; bf = 1; }
  else if (W % 4 == 0) { bw = 4; bh = 4; bf = 4; }
  else if (W % 2 == 0) { bw = 2; bh = 2; bf = 16; }
  else { bw = 1; bh = 1; bf = 64; }
}

}  // namespace

int umma_wgrad_ptiles(int W, int H, int F) {
  int bw, bh, bf;
  wgrad_box(W, bw, bh, bf);
  return ((W + bw - 1) / bw) * ((H + bh - 1) / bh) * ((F + bf - 1) / bf);
}

int umma_wgrad_splits(int ctas, int ptiles, int num_sms, int waves) {
  // one CTA per SM is resident (192 KiB pipeline), so a second wave only runs after the first: ONE wave of CTAs with twice the
  // pixels each does the same work with half the split-K partial traffic (every CTA writes its whole 128 x taps*N fp32
  // accumulator: 100-250 KB) and no wave tail -- until a split gets longer than UMMA_WGRAD_MAX_PTILES tiles
  const int per_wave = std::max(1, waves * num_sms / ctas);
  const int need = (ptiles + UMMA_WGRAD_MAX_PTILES - 1) / UMMA_WGRAD_MAX_PTILES;
  return std::max(1, (need + per_wave - 1) / per_wave) * per_wave;
}

int umma_wgrad_bind(UmmaContext& ctx, UmmaWgradPlan& plan, View dz, View x, int F, int cin, int cout, int k, int pad,
                    float* partial, int max_splits, int x_stride) {
  int dy[UMMA_MAX_TAPS], dx[UMMA_MAX_TAPS];
  if (k * k > UMMA_MAX_TAPS) { set_thread_error("umma wgrad: too many taps"); return 1; }
  for (int r = 0; r < k; ++r)
    for (int s = 0; s < k; ++s) { dy[r * k + s] = r - pad; dx[r * k + s] = s - pad; }
  return umma_wgrad_bind_taps(ctx, plan, dz, x, F, cin, cout, k * k, dy, dx, partial, max_splits, x_stride);
}

int umma_wgrad_bind_taps(UmmaContext& ctx, UmmaWgradPlan& plan, View dz, View x, int F, int cin, int cout, int ntaps,
                         const int* tdy, const int* tdx, float* partial, int max_splits, int x_stride) {
  plan.enabled = false;
  if (int rc = umma_resolve_encode(ctx)) return rc;
  if (dz.H != (x.H + x_stride - 1) / x_stride || dz.W != (x.W + x_stride - 1) / x_stride) { set_thread_error("umma wgrad: geometry mismatch"); return 1; }
  if (cin % 8 || cout % 8 || dz.pitch % 8 || dz.coff % 8 || x.pitch % 8 || x.coff % 8 || ntaps > UMMA_MAX_TAPS) {
    set_thread_error("umma wgrad: unsupported channel alignment"); return 1; }
  UmmaWgradParams& p = plan.p;
  memset(&p, 0, sizeof(p));
  p.W = dz.W; p.H = dz.H; p.F = F; p.x_stride = x_stride;     // tiles enumerate dz (output) pixels
  wgrad_box(dz.W, p.bw, p.bh, p.bf);
  p.tiles_w = (dz.W + p.bw - 1) / p.bw; p.tiles_h = (dz.H + p.bh - 1) / p.bh; p.tiles_f = (F + p.bf - 1) / p.bf;
  p.ntaps = ntaps;
  for (int t = 0; t < ntaps; ++t) { p.tap_dy[t] = tdy[t]; p.tap_dx[t] = tdx[t]; }
  p.Cout = cout; p.Cin = cin;
  p.m_tiles = (cout + BLOCK_M - 1) / BLOCK_M;
  const int chunks = (cin + 63) / 64;
  p.n_tiles = (chunks + 3) / 4;
  p.block_n = ((chunks + p.n_tiles - 1) / p.n_tiles) * 64;
  // several taps per CTA share one dz tile: 2 dz boxes + taps * (block_n/64) <= 4 x boxes per plane, which also bounds the
  // register accumulators at 256 fp32 columns
  p.taps_per_cta = std::max(1, 4 / (p.block_n / 64));
  if (p.taps_per_cta > ntaps) p.taps_per_cta = ntaps;
  p.tap_groups = (ntaps + p.taps_per_cta - 1) / p.taps_per_cta;
  p.taps_per_cta = (ntaps + p.tap_groups - 1) / p.tap_groups;        // balance the groups (9 taps: 3+3+3 rather than 4+4+1)
  const int ptiles = p.tiles_w * p.tiles_h * p.tiles_f;
  const int ctas = p.m_tiles * p.n_tiles * p.tap_groups;
  const char* we = getenv("SSNB_WGRAD_WAVES");
  int splits = umma_wgrad_splits(ctas, ptiles, ctx.num_sms, we ? atoi(we) : 1);
  if (splits > max_splits) splits = max_splits;
  if (splits > ptiles) splits = ptiles;
  if (splits < 1) splits = 1;
  p.ptiles_per_split = (ptiles + splits - 1) / splits;
  p.splits = (ptiles + p.ptiles_per_split - 1) / p.ptiles_per_split;
  p.partial = partial; p.bias_partial = nullptr;
  p.nseg = (dz.lo_off && x.lo_off) ? 3 : 1;
  if ((dz.lo_off != 0) != (x.lo_off != 0)) { set_thread_error("umma wgrad: both operands or neither must carry LO planes"); return 1; }
  // a stage holds every operand box of one pixel tile (FAST) or both planes of each box of half a tile (EXACT_TC)
  const int sub = p.nseg == 3 ? 2 : 1;       // stages per pixel tile: the kernel's SUB
  const int sub_bh = p.bf > 1 ? p.bh : p.bh / sub, sub_bf = p.bf > 1 ? p.bf / sub : 1;
  p.sub_dh = sub == 1 ? 0 : p.bh - sub_bh; p.sub_df = sub == 1 ? 0 : p.bf - sub_bf;
  p.stage_bytes = (p.nseg == 3 ? 2 : 1) * (2 + p.taps_per_cta * (p.block_n / 64)) * BOX_BYTES / sub;
  p.stages = std::min(PIPE_BYTES / p.stage_bytes, MAX_STAGES);
  auto lo_ptr = [](const View& v) { return reinterpret_cast<__half*>(reinterpret_cast<char*>(v.base) + v.lo_off) + v.coff; };
  {
    cuuint64_t dims[4] = {(cuuint64_t)cout, (cuuint64_t)dz.W, (cuuint64_t)dz.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)dz.pitch * 2, (cuuint64_t)dz.W * dz.pitch * 2, (cuuint64_t)dz.H * dz.W * dz.pitch * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.bw, (cuuint32_t)sub_bh, (cuuint32_t)sub_bf};
    if (int rc = umma_encode_f16(ctx, &plan.tmap_dz, 4, reinterpret_cast<__half*>(dz.base) + dz.coff, dims, str, box)) return rc;
    plan.tmap_dz_lo = plan.tmap_dz;
    if (p.nseg == 3) if (int rc = umma_encode_f16(ctx, &plan.tmap_dz_lo, 4, lo_ptr(dz), dims, str, box)) return rc;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)x.W, (cuuint64_t)x.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)x.pitch * 2, (cuuint64_t)x.W * x.pitch * 2, (cuuint64_t)x.H * x.W * x.pitch * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(p.bw * x_stride), (cuuint32_t)(sub_bh * x_stride), (cuuint32_t)sub_bf};
    if (int rc = umma_encode_f16(ctx, &plan.tmap_x, 4, reinterpret_cast<__half*>(x.base) + x.coff, dims, str, box, x_stride)) return rc;
    plan.tmap_x_lo = plan.tmap_x;
    if (p.nseg == 3) if (int rc = umma_encode_f16(ctx, &plan.tmap_x_lo, 4, lo_ptr(x), dims, str, box, x_stride)) return rc;
  }
  plan.enabled = true;
  return 0;
}

namespace {
template <int NACC, int NSEG>
int launch_nacc(const UmmaWgradPlan& plan, const UmmaWgradParams& p, cudaStream_t s) {
  static bool attr_set[64] = {};          // function attributes are per device
  auto kern = umma_wgrad_kernel<NACC, NSEG>;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess) {
      set_thread_error("umma wgrad: cannot raise dynamic shared memory limit"); cudaGetLastError(); return 2; }
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3((unsigned)(p.m_tiles * p.n_tiles * p.tap_groups), (unsigned)p.splits);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = s;
  static const bool pdl = [] { const char* e = getenv("SSNB_PDL"); return !(e && e[0] == '0'); }();
  if (pdl) { attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1; cfg.attrs = attr; cfg.numAttrs = 1; }
  if (cudaLaunchKernelEx(&cfg, kern, plan.tmap_dz, plan.tmap_x, plan.tmap_dz_lo, plan.tmap_x_lo, p) != cudaSuccess) {
    set_thread_error(std::string("umma_wgrad_kernel launch: ") + cudaGetErrorString(cudaGetLastError())); return 2; }
  SSNB_LAUNCH_CHECK("umma_wgrad_kernel");
  return 0;
}
}  // namespace

int umma_wgrad_launch(UmmaContext&, const UmmaWgradPlan& plan, cudaStream_t s, float* bias_partial) {
  if (!plan.enabled) { set_thread_error("umma wgrad: plan not bound"); return 3; }
  UmmaWgradParams p = plan.p;
  p.bias_partial = bias_partial;
  t_tag.tiles = p.m_tiles * p.n_tiles * p.tap_groups; t_tag.block_n = p.splits;     // the launch log's grid: ctas x splits
  switch (p.taps_per_cta * (p.block_n / 64) * 4 + p.nseg) {
    case 5: return launch_nacc<1, 1>(plan, p, s);
    case 9: return launch_nacc<2, 1>(plan, p, s);
    case 13: return launch_nacc<3, 1>(plan, p, s);
    case 17: return launch_nacc<4, 1>(plan, p, s);
    case 7: return launch_nacc<1, 3>(plan, p, s);
    case 11: return launch_nacc<2, 3>(plan, p, s);
    case 15: return launch_nacc<3, 3>(plan, p, s);
    case 19: return launch_nacc<4, 3>(plan, p, s);
  }
  set_thread_error("umma wgrad: unsupported tile width"); return 3;
}

}  // namespace ssnb
