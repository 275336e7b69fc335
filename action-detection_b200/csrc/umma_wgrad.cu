// wgmma weight-gradient kernel (sm_90a).  dW[tap][co][ci] = sum_p dz[p, co] * x[p + shift(tap), ci]
// is a GEMM whose reduction runs over pixels, so both operands are MN-major in shared memory:
// a TMA box is [64 pixels][64 channels] (128-byte rows, SWIZZLE_128B) and the wgmma descriptors walk
// it with 8-pixel groups every 1024 B (SBO).
//
//   CTA = (co tile of 128, ci tile of block_n <= 256, taps, pixel split); K loop over 64-pixel boxes.
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
constexpr int BOX_BYTES = 64 * 128;                 // [64 px][64 ch] fp16
constexpr int A_BYTES = 2 * BOX_BYTES;              // 128 output channels
constexpr int STAGE_BYTES = A_BYTES + 4 * BOX_BYTES;        // 2 dz boxes + up to 4 x boxes (taps x 64-channel atoms)
constexpr int STAGES = 4;
constexpr int PIPE_BYTES = STAGES * STAGE_BYTES;            // 192 KiB of operand staging
constexpr int NUM_THREADS = 384;
constexpr int ONES_OFF = PIPE_BYTES + 1024;                // [16 rows][64 px] of fp16 ones (bias-gradient operand), 1 KiB aligned
constexpr int ONES_BYTES = 16 * 128;
constexpr int SMEM_BYTES = PIPE_BYTES + 1024 /*align slack*/ + 1024 /*barriers*/ + ONES_BYTES;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");

// NACC = taps_per_cta * block_n / 64 accumulator blocks of 64 columns per consumer warpgroup
template <int NACC>
__global__ void __launch_bounds__(NUM_THREADS, 1)
umma_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_dz, const __grid_constant__ CUtensorMap tmap_x,
                  const __grid_constant__ CUtensorMap tmap_dz_lo, const __grid_constant__ CUtensorMap tmap_x_lo,
                  const __grid_constant__ UmmaWgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + PIPE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + MAX_STAGES;

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
      const uint32_t tx_bytes = (uint32_t)(2 + nboxes_b * ntap) * BOX_BYTES;
      // pixel-tile coordinates advance by carries (no divisions in the loop)
      int tw = pt0 % p.tiles_w, th = (pt0 / p.tiles_w) % p.tiles_h, tf = pt0 / (p.tiles_w * p.tiles_h);
      for (int pt = pt0; pt < pt1; ++pt) {
        const int w0 = tw * p.bw, h0 = th * p.bh, f0 = tf * p.bf;
        // SSNB_EXACT_TC (nseg = 3): the tile is staged three times, (dz_lo, x_hi), (dz_hi, x_lo), (dz_hi, x_hi)
        for (int seg = 3 - p.nseg; seg < 3; ++seg) {
          const CUtensorMap* mdz = seg == 0 ? &tmap_dz_lo : &tmap_dz;
          const CUtensorMap* mx = seg == 1 ? &tmap_x_lo : &tmap_x;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full_bar[stage], tx_bytes);
          tma_load_4d(sa, mdz, &full_bar[stage], m0, w0, h0, f0);
          tma_load_4d(sa + BOX_BYTES, mdz, &full_bar[stage], m0 + 64, w0, h0, f0);
          for (int t = 0; t < ntap; ++t)
            for (int b = 0; b < nboxes_b; ++b)
              tma_load_4d(sb + (t * nboxes_b + b) * BOX_BYTES, mx, &full_bar[stage], n0 + b * 64,
                          w0 * p.x_stride + p.tap_dx[tap0 + t], h0 * p.x_stride + p.tap_dy[tap0 + t], f0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if (++tw == p.tiles_w) { tw = 0; if (++th == p.tiles_h) { th = 0; ++tf; } }
      }
    }
  } else {
    consumer_regs();
    const int cw = wg - 1;
    const int warp = (threadIdx.x / 32) & 3, lane = threadIdx.x & 31;
    const int nacc = ntap * nboxes_b;                 // accumulator blocks in use (<= NACC)
    float acc[NACC][32], accb[8];
#pragma unroll
    for (int j = 0; j < NACC; ++j)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) accb[i] = 0.f;
    const uint32_t ones = smem_u32(smem + ONES_OFF);
    uint32_t stage = 0, phase = 0, prev = 0;
    bool first = true;
    for (int pt = pt0; pt < pt1; ++pt)
    for (int seg = 3 - p.nseg; seg < 3; ++seg) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + cw * BOX_BYTES;
      const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES) + A_BYTES;
      // the x boxes of all taps of this CTA are consecutive 64-channel N atoms BOX_BYTES apart (the LBO), so ONE m64n(64 NACC)k16
      // MMA per 16 pixel rows takes them all and the dz rows are read from shared memory once.  A CTA of a short last tap
      // group (nacc < NACC) multiplies stale atoms into accumulator blocks it never stores, which keeps the MMA sequence free
      // of predication.
      const bool bias_mma = do_bias && seg != 1;     // column sums of dz: hi and lo planes once each (seg 1 re-stages dz_hi)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 64 / MMA_K; ++k)           // 16 pixel rows (2 groups of 8) per instruction
        wgmma<NACC * MMA_N, 1, 1>(&acc[0][0], make_desc_sw128(sa + k * (MMA_K * 128), BOX_BYTES), make_desc_sw128(sb + k * (MMA_K * 128), BOX_BYTES));
      if (bias_mma) {                                // the ones operand is K-major
#pragma unroll
        for (int k = 0; k < 64 / MMA_K; ++k)
          wgmma<16, 1, 0>(accb, make_desc_sw128(sa + k * (MMA_K * 128), BOX_BYTES), make_desc_sw128(ones + k * MMA_K * 2));
      }
      wgmma_commit();
      // one group stays in flight: the previous stage's MMAs have retired, its smem slot goes back to the producer
      wgmma_wait<1>();
      if (!first && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      first = false;
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
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
  // several taps per CTA share one dz tile: stage = 2 dz boxes + taps * (block_n/64) x boxes <= 6 boxes, which also
  // bounds the register accumulators at 256 fp32 columns
  p.stage_bytes = STAGE_BYTES; p.stages = STAGES;
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
  auto lo_ptr = [](const View& v) { return reinterpret_cast<__half*>(reinterpret_cast<char*>(v.base) + v.lo_off) + v.coff; };
  {
    cuuint64_t dims[4] = {(cuuint64_t)cout, (cuuint64_t)dz.W, (cuuint64_t)dz.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)dz.pitch * 2, (cuuint64_t)dz.W * dz.pitch * 2, (cuuint64_t)dz.H * dz.W * dz.pitch * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.bw, (cuuint32_t)p.bh, (cuuint32_t)p.bf};
    if (int rc = umma_encode_f16(ctx, &plan.tmap_dz, 4, reinterpret_cast<__half*>(dz.base) + dz.coff, dims, str, box)) return rc;
    plan.tmap_dz_lo = plan.tmap_dz;
    if (p.nseg == 3) if (int rc = umma_encode_f16(ctx, &plan.tmap_dz_lo, 4, lo_ptr(dz), dims, str, box)) return rc;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)x.W, (cuuint64_t)x.H, (cuuint64_t)F};
    cuuint64_t str[3] = {(cuuint64_t)x.pitch * 2, (cuuint64_t)x.W * x.pitch * 2, (cuuint64_t)x.H * x.W * x.pitch * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(p.bw * x_stride), (cuuint32_t)(p.bh * x_stride), (cuuint32_t)p.bf};
    if (int rc = umma_encode_f16(ctx, &plan.tmap_x, 4, reinterpret_cast<__half*>(x.base) + x.coff, dims, str, box, x_stride)) return rc;
    plan.tmap_x_lo = plan.tmap_x;
    if (p.nseg == 3) if (int rc = umma_encode_f16(ctx, &plan.tmap_x_lo, 4, lo_ptr(x), dims, str, box, x_stride)) return rc;
  }
  plan.enabled = true;
  return 0;
}

namespace {
template <int NACC>
int launch_nacc(const UmmaWgradPlan& plan, const UmmaWgradParams& p, cudaStream_t s) {
  static bool attr_set[64] = {};          // function attributes are per device
  auto kern = umma_wgrad_kernel<NACC>;
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
  switch (p.taps_per_cta * (p.block_n / 64)) {
    case 1: return launch_nacc<1>(plan, p, s);
    case 2: return launch_nacc<2>(plan, p, s);
    case 3: return launch_nacc<3>(plan, p, s);
    case 4: return launch_nacc<4>(plan, p, s);
  }
  set_thread_error("umma wgrad: unsupported tile width"); return 3;
}

}  // namespace ssnb
