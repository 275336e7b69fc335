// Dual TV-L1 optical flow for many frame pairs per call (ssnb_tvl1_flow), the rules of oracle/tvl1_oracle.py (R1 .. R9).
//
// Every launch covers all pairs of the call (blockIdx.z = pair, one thread per pixel of a 32 x 8 tile), so the ~2 x iterations
// x warps x levels dependent launches of a call are few compared with the pixels each one moves: at 340 x 256 and a few
// hundred pairs a primal or dual launch streams hundreds of MB, and the solver is bound by HBM, not by launch latency.
//
//   tvl1_init_kernel      pair -> first frame from the video offsets; zeroes the per-pair stopping state
//   tvl1_grey_kernel      R1, uint8 RGB -> fp32 grey, every frame once
//   tvl1_resize_kernel    R3, the pyramid (every frame) and the flow's upsampling (times 1 / scale_step)
//   tvl1_gradient_kernel  R4 of each pair's second frame
//   tvl1_warp_kernel      R5; resets the pair's iteration count and stop flag for the warp
//   tvl1_primal_kernel    R6; each CTA's squared update summed in double in a fixed tree, the pair's CTA partials summed in
//                         index order by the pair's last CTA (an arrival counter), which applies R8's test and counts
//   tvl1_dual_kernel      R7, only for pairs whose primal update ran in this iteration
//   flow_planes_kernel    R9
#include <climits>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int BX = 32, BY = 8, kThreads = BX * BY;
constexpr int kMaxSide = 8192, kMaxPairs = 32767, kMaxPlanes = 65535, kMaxLevels = 32;   // grid.z: pairs, 2 x pairs, frames

struct StopState {
  double* partial;     // [P, tiles] CTA sums of the squared update
  int* arrived;        // [P] CTAs of the pair done with this iteration (reset to 0 by the last one)
  int* iter;           // [P] iterations run in the current warp
  int* stopped;        // [P] the current warp of the pair has met the stopping rule
  int32_t* counts;     // [P, levels, warps] or nullptr
  double thr;          // epsilon^2 * level area
  int stopping, tiles, levels, warps, level, warp;
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__device__ __forceinline__ float cubic(float t) {
  t = fabsf(t);
  if (t <= 1.f) return t * t * (1.5f * t - 2.5f) + 1.f;
  if (t < 2.f) return t * (t * (-0.5f * t + 2.5f) - 4.f) + 2.f;
  return 0.f;
}

__global__ void tvl1_init_kernel(const int64_t* __restrict__ offsets, int n_videos, int P, int* __restrict__ pair_frame, int* __restrict__ arrived,
                                 int* __restrict__ iter, int* __restrict__ stopped) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  // video v owns pairs offsets[v] - v .. offsets[v + 1] - v - 2: the last video whose first pair is <= p
  int lo = 0, hi = n_videos - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] - mid <= p) lo = mid; else hi = mid - 1;
  }
  pair_frame[p] = p + lo;
  arrived[p] = 0;
  iter[p] = 0;
  stopped[p] = 0;
}

__global__ void tvl1_fill_kernel(float* __restrict__ x, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] = 0.f;
}

__global__ void tvl1_grey_kernel(const uint8_t* __restrict__ rgb, long long n, float* __restrict__ g) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint8_t* c = rgb + 3 * i;
    g[i] = (float)((c[0] * 9798 + c[1] * 19235 + c[2] * 3735 + (1 << 14)) >> 15);
  }
}

// blockIdx.z = plane; source h x w -> dst oh x ow
__global__ void tvl1_resize_kernel(const float* __restrict__ src, int h, int w, float* __restrict__ dst, int oh, int ow, float mul) {
  const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
  if (x >= ow || y >= oh) return;
  const float* s = src + (long long)blockIdx.z * h * w;
  // source coordinate and weights in double, each weight rounded once to fp32 (an fp32 coordinate near x = 300 would carry
  // 1.5e-5 px of rounding into the weights)
  const double sx = (x + 0.5) * ((double)w / ow) - 0.5, sy = (y + 0.5) * ((double)h / oh) - 0.5;
  const double fx = floor(sx), fy = floor(sy);
  const float ax = (float)(sx - fx), ay = (float)(sy - fy);
  const int x0 = clampi((int)fx, 0, w - 1), x1 = clampi((int)fx + 1, 0, w - 1);
  const int y0 = clampi((int)fy, 0, h - 1), y1 = clampi((int)fy + 1, 0, h - 1);
  const float r0 = s[(long long)y0 * w + x0] * (1.f - ax) + s[(long long)y0 * w + x1] * ax;
  const float r1 = s[(long long)y1 * w + x0] * (1.f - ax) + s[(long long)y1 * w + x1] * ax;
  dst[(long long)blockIdx.z * oh * ow + (long long)y * ow + x] = (r0 * (1.f - ay) + r1 * ay) * mul;
}

// I1 of pair p is plane (fr ? fr[p] + 1 : p) of I1
__global__ void tvl1_gradient_kernel(const float* __restrict__ I1, const int* __restrict__ fr, int h, int w, float* __restrict__ Ix,
                                     float* __restrict__ Iy) {
  const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y, p = blockIdx.z;
  if (x >= w || y >= h) return;
  const long long A = (long long)h * w;
  const float* I = I1 + (fr ? fr[p] + 1 : p) * A;
  const long long o = p * A + (long long)y * w + x;
  Ix[o] = 0.5f * (I[(long long)y * w + min(x + 1, w - 1)] - I[(long long)y * w + max(x - 1, 0)]);
  Iy[o] = 0.5f * (I[(long long)min(y + 1, h - 1) * w + x] - I[(long long)max(y - 1, 0) * w + x]);
}

__global__ void tvl1_warp_kernel(const float* __restrict__ I0, const float* __restrict__ I1, const int* __restrict__ fr, const float* __restrict__ Ix,
                                 const float* __restrict__ Iy, const float* __restrict__ u, int h, int w, float* __restrict__ Ixw, float* __restrict__ Iyw,
                                 float* __restrict__ grad, float* __restrict__ rho_c, int* __restrict__ iter, int* __restrict__ stopped) {
  const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y, p = blockIdx.z;
  if (iter && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0) { iter[p] = 0; stopped[p] = 0; }
  if (x >= w || y >= h) return;
  const long long A = (long long)h * w, o = (long long)y * w + x;
  const float* J = I1 + (fr ? fr[p] + 1 : p) * A;
  const float* gx = Ix + p * A;
  const float* gy = Iy + p * A;
  const float u1 = u[2 * p * A + o], u2 = u[(2 * p + 1) * A + o];
  // the sample point and each tap's offset in double, the offset rounded once to fp32: x + u1 in fp32 rounds to 2^-11 px near
  // x = 8191 (to 3e-5 px near x = 300), and every tap weight would carry that
  const double wx = fmin(fmax(x + (double)u1, -3.0), w + 2.0), wy = fmin(fmax(y + (double)u2, -3.0), h + 2.0);
  const int xmin = (int)ceil(wx - 2.0), xmax = (int)floor(wx + 2.0), ymin = (int)ceil(wy - 2.0), ymax = (int)floor(wy + 2.0);
  float s = 0.f, sx = 0.f, sy = 0.f, ws = 0.f;
  for (int cy = ymin; cy <= ymax; ++cy) {
    const float ky = cubic((float)(wy - cy));
    const long long row = (long long)clampi(cy, 0, h - 1) * w;
    for (int cx = xmin; cx <= xmax; ++cx) {
      const float k = ky * cubic((float)(wx - cx));
      const long long q = row + clampi(cx, 0, w - 1);
      s += k * J[q];
      sx += k * gx[q];
      sy += k * gy[q];
      ws += k;
    }
  }
  const float c = 1.f / ws;
  const float I1w = s * c, Ixv = sx * c, Iyv = sy * c;
  const long long po = p * A + o;
  Ixw[po] = Ixv;
  Iyw[po] = Iyv;
  grad[po] = Ixv * Ixv + Iyv * Iyv;
  rho_c[po] = I1w - Ixv * u1 - Iyv * u2 - I0[(fr ? fr[p] : p) * A + o];
}

// div(a, b) at (x, y) with the first column's / row's backward term dropped (R6)
__device__ __forceinline__ float divergence(const float* a, const float* b, int x, int y, int w) {
  const long long o = (long long)y * w + x;
  float d = a[o] + b[o];
  if (x > 0) d -= a[o - 1];
  if (y > 0) d -= b[o - w];
  return d;
}

__global__ void __launch_bounds__(kThreads) tvl1_primal_kernel(const float* __restrict__ Ixw, const float* __restrict__ Iyw, const float* __restrict__ grad,
                                                               const float* __restrict__ rho_c, const float* __restrict__ pd, const float* u_in, float* u_out,
                                                               int h, int w, float l_t, float theta, StopState st, int n) {
  const int p = blockIdx.z;
  if (st.partial && st.stopped[p]) return;
  const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y, t = threadIdx.y * BX + threadIdx.x;
  float e = 0.f;
  if (x < w && y < h) {
    const long long A = (long long)h * w, o = (long long)y * w + x, po = p * A + o;
    const float gxv = Ixw[po], gyv = Iyw[po], gv = grad[po];
    const float u1 = u_in[2 * p * A + o], u2 = u_in[(2 * p + 1) * A + o];
    const float rho = rho_c[po] + (gxv * u1 + gyv * u2);
    float d1 = 0.f, d2 = 0.f;
    if (rho < -l_t * gv) { d1 = l_t * gxv; d2 = l_t * gyv; }
    else if (rho > l_t * gv) { d1 = -l_t * gxv; d2 = -l_t * gyv; }
    else if (gv > 1.1920928955078125e-7f) { const float fi = -rho / gv; d1 = fi * gxv; d2 = fi * gyv; }
    const float* P4 = pd + 4 * p * A;
    const float n1 = u1 + d1 + theta * divergence(P4, P4 + A, x, y, w);
    const float n2 = u2 + d2 + theta * divergence(P4 + 2 * A, P4 + 3 * A, x, y, w);
    u_out[2 * p * A + o] = n1;
    u_out[(2 * p + 1) * A + o] = n2;
    e = (u1 - n1) * (u1 - n1) + (u2 - n2) * (u2 - n2);
  }
  if (!st.partial) return;
  __shared__ double red[kThreads];
  __shared__ int last;
  red[t] = (double)e;
  __syncthreads();
  for (int k = kThreads / 2; k > 0; k >>= 1) {
    if (t < k) red[t] += red[t + k];
    __syncthreads();
  }
  if (t == 0) {
    st.partial[(long long)p * st.tiles + blockIdx.y * gridDim.x + blockIdx.x] = red[0];
    __threadfence();
    last = atomicAdd(&st.arrived[p], 1) == st.tiles - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double s = 0.0;
  for (int i = t; i < st.tiles; i += kThreads) s += __ldcg(&st.partial[(long long)p * st.tiles + i]);
  red[t] = s;
  __syncthreads();
  for (int k = kThreads / 2; k > 0; k >>= 1) {
    if (t < k) red[t] += red[t + k];
    __syncthreads();
  }
  if (t == 0) {
    st.arrived[p] = 0;
    st.iter[p] = n + 1;
    if (st.counts) st.counts[((long long)p * st.levels + st.level) * st.warps + st.warp] = n + 1;
    if (st.stopping && red[0] <= st.thr) st.stopped[p] = 1;
  }
}

__global__ void __launch_bounds__(kThreads) tvl1_dual_kernel(const float* __restrict__ u, const float* p_in, float* p_out, int h, int w, float taut,
                                                             const int* __restrict__ iter, int n) {
  const int p = blockIdx.z;
  if (iter && iter[p] != n + 1) return;
  const int x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
  if (x >= w || y >= h) return;
  const long long A = (long long)h * w, o = (long long)y * w + x;
  const long long ox = (long long)y * w + min(x + 1, w - 1), oy = (long long)min(y + 1, h - 1) * w + x;
  for (int i = 0; i < 2; ++i) {
    const float* U = u + (2 * p + i) * A;
    const float ux = U[ox] - U[o], uy = U[oy] - U[o];
    const float ng = 1.f + taut * hypotf(ux, uy);
    const long long b = (4 * p + 2 * i) * A + o;
    p_out[b] = (p_in[b] + taut * ux) / ng;
    p_out[b + A] = (p_in[b + A] + taut * uy) / ng;
  }
}

__global__ void flow_planes_kernel(const float* __restrict__ flow, long long n, double bound, uint8_t* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double v = (double)flow[i];
    out[i] = v > bound ? 255 : (!(v >= -bound) ? 0 : (uint8_t)__double2int_rn(255.0 * (v + bound) / (2.0 * bound)));
  }
}

int blocks_for(long long n) { return (int)std::min<long long>((n + kThreads - 1) / kThreads, 148LL * 32); }
dim3 tiles(int h, int w, int n) { return dim3((unsigned)((w + BX - 1) / BX), (unsigned)((h + BY - 1) / BY), (unsigned)n); }

const char* check_params(const ssnb_tvl1_params* q) {
  if (!q) return "NULL params";
  if (!(q->tau > 0 && q->tau < 1e6) || !(q->theta > 0 && q->theta < 1e6)) return "tau and theta must be positive and finite";
  if (!(q->lambda >= 0 && q->lambda < 1e6)) return "lambda must be >= 0 and finite";
  if (!(q->epsilon >= 0 && q->epsilon < 1e6)) return "epsilon must be >= 0 and finite";
  if (!(q->scale_step > 0 && q->scale_step < 1)) return "scale_step must lie in (0, 1)";
  if (q->gamma != 0) return "gamma != 0 (the illumination term) is not implemented";
  if (q->nscales < 1 || q->nscales > kMaxLevels) return "nscales must be in 1..32";
  if (q->warps < 1 || q->warps > 1000) return "warps must be in 1..1000";
  if (q->iterations < 1 || q->iterations > 100000) return "iterations must be in 1..100000";
  return nullptr;
}

// R2: sizes finest first
void level_sizes(const ssnb_tvl1_params* q, int h, int w, std::vector<int>& hs, std::vector<int>& ws) {
  hs.assign(1, h);
  ws.assign(1, w);
  while ((int)hs.size() < q->nscales) {
    const int nh = (int)std::nearbyint(hs.back() * q->scale_step), nw = (int)std::nearbyint(ws.back() * q->scale_step);
    if (nh < 16 || nw < 16) break;
    hs.push_back(nh);
    ws.push_back(nw);
  }
}

struct Layout {
  std::vector<int> hs, ws;
  long long F = 0, P = 0;
  size_t pyr = 0, pair_frame = 0, ix = 0, iy = 0, wx = 0, wy = 0, grad = 0, rho = 0, pd = 0, u[2] = {0, 0}, partial = 0, arrived = 0,
         iter = 0, stopped = 0, total = 0;
  std::vector<size_t> level_off;   // byte offset of pyramid level l
  int tiles0 = 0;
};

const char* plan(const ssnb_tvl1_params* q, const int64_t* offsets, int V, int h, int w, Layout& L) {
  if (const char* bad = check_params(q)) return bad;
  if (h < 1 || w < 1 || h > kMaxSide || w > kMaxSide) return "height / width outside 1..8192";
  if (!offsets || V < 1) return "no video";
  if (offsets[0] != 0) return "offsets[0] must be 0";
  for (int v = 0; v < V; ++v)
    if (offsets[v + 1] < offsets[v] + 1) return "a video without frames (offsets must increase)";
  L.F = offsets[V];
  L.P = L.F - V;
  if (L.P < 1) return "no frame pair (every video has one frame)";
  if (L.P > kMaxPairs || L.F > kMaxPlanes) return "more than 32767 pairs or 65535 frames in one call";
  level_sizes(q, h, w, L.hs, L.ws);
  const long long A0 = (long long)h * w;
  size_t off = 0;
  auto take = [&](long long bytes) { const size_t o = off; off += ((size_t)bytes + 255) & ~(size_t)255; return o; };
  L.level_off.clear();
  long long pyr_floats = 0;
  for (size_t l = 0; l < L.hs.size(); ++l) {
    L.level_off.push_back((size_t)pyr_floats * 4);
    pyr_floats += L.F * L.hs[l] * L.ws[l];
  }
  L.pyr = take(pyr_floats * 4);
  L.pair_frame = take(L.P * 4);
  L.ix = take(L.P * A0 * 4); L.iy = take(L.P * A0 * 4);
  L.wx = take(L.P * A0 * 4); L.wy = take(L.P * A0 * 4); L.grad = take(L.P * A0 * 4); L.rho = take(L.P * A0 * 4);
  L.pd = take(4 * L.P * A0 * 4);
  const long long A1 = L.hs.size() > 1 ? (long long)L.hs[1] * L.ws[1] : 0;
  L.u[0] = take(2 * L.P * A1 * 4); L.u[1] = take(2 * L.P * A1 * 4);
  const dim3 g = tiles(h, w, 1);
  L.tiles0 = (int)(g.x * g.y);
  L.partial = take(L.P * L.tiles0 * 8);
  L.arrived = take(L.P * 4); L.iter = take(L.P * 4); L.stopped = take(L.P * 4);
  L.total = off;
  return nullptr;
}

}  // namespace
}  // namespace ssnb

using namespace ssnb;

extern "C" {

int ssnb_tvl1_levels(const ssnb_tvl1_params* prm, int height, int width) {
  if (check_params(prm) || height < 1 || width < 1 || height > kMaxSide || width > kMaxSide) return 0;
  std::vector<int> hs, ws;
  level_sizes(prm, height, width, hs, ws);
  return (int)hs.size();
}

size_t ssnb_tvl1_workspace_bytes(const ssnb_tvl1_params* prm, const int64_t* offsets, int n_videos, int height, int width) {
  Layout L;
  if (plan(prm, offsets, n_videos, height, width, L)) return 0;
  return L.total;
}

int ssnb_tvl1_flow(const ssnb_tvl1_params* prm, const uint8_t* frames, const int64_t* offsets, const int64_t* offsets_dev, int n_videos,
                   int height, int width, float* flow, int32_t* iterations, void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("tvl1_flow: " + m); return (int)SSNB_EINVAL; };
  Layout L;
  if (const char* bad = plan(prm, offsets, n_videos, height, width, L)) return fail(bad);
  if (!frames || !offsets_dev || !flow) return fail("NULL frames, offsets_dev or flow");
  if (!workspace || workspace_bytes < L.total) return fail("workspace too small (ssnb_tvl1_workspace_bytes)");
  char* ws = (char*)workspace;
  float* pyr = (float*)(ws + L.pyr);
  int* fr = (int*)(ws + L.pair_frame);
  float *Ix = (float*)(ws + L.ix), *Iy = (float*)(ws + L.iy), *Ixw = (float*)(ws + L.wx), *Iyw = (float*)(ws + L.wy);
  float *grad = (float*)(ws + L.grad), *rho = (float*)(ws + L.rho), *pd = (float*)(ws + L.pd);
  const int P = (int)L.P, levels = (int)L.hs.size();
  StopState st{(double*)(ws + L.partial), (int*)(ws + L.arrived), (int*)(ws + L.iter), (int*)(ws + L.stopped), iterations, 0.0,
               prm->fixed_iterations == 0, 0, levels, prm->warps, 0, 0};
  const float l_t = (float)(prm->lambda * prm->theta), taut = (float)(prm->tau / prm->theta), theta = (float)prm->theta;

  tvl1_init_kernel<<<(P + 255) / 256, 256, 0, s>>>(offsets_dev, n_videos, P, fr, st.arrived, st.iter, st.stopped);
  SSNB_LAUNCH_CHECK("tvl1_init_kernel");
  const long long A0 = (long long)height * width;
  tvl1_grey_kernel<<<blocks_for(L.F * A0), kThreads, 0, s>>>(frames, L.F * A0, pyr);
  SSNB_LAUNCH_CHECK("tvl1_grey_kernel");
  for (int l = 1; l < levels; ++l) {
    tvl1_resize_kernel<<<tiles(L.hs[l], L.ws[l], (int)L.F), dim3(BX, BY), 0, s>>>((float*)(ws + L.pyr + L.level_off[l - 1]), L.hs[l - 1], L.ws[l - 1],
                                                                                  (float*)(ws + L.pyr + L.level_off[l]), L.hs[l], L.ws[l], 1.f);
    SSNB_LAUNCH_CHECK("tvl1_resize_kernel");
  }
  for (int l = levels - 1; l >= 0; --l) {
    const int h = L.hs[l], w = L.ws[l];
    const long long A = (long long)h * w;
    float* u = l == 0 ? flow : (float*)(ws + L.u[l & 1]);
    const float* lev = (const float*)(ws + L.pyr + L.level_off[l]);
    if (l == levels - 1) {
      tvl1_fill_kernel<<<blocks_for(2 * P * A), kThreads, 0, s>>>(u, 2 * P * A);
      SSNB_LAUNCH_CHECK("tvl1_fill_kernel");
    }
    tvl1_fill_kernel<<<blocks_for(4 * P * A), kThreads, 0, s>>>(pd, 4 * P * A);
    SSNB_LAUNCH_CHECK("tvl1_fill_kernel");
    const dim3 grid = tiles(h, w, P), block(BX, BY);
    tvl1_gradient_kernel<<<grid, block, 0, s>>>(lev, fr, h, w, Ix, Iy);
    SSNB_LAUNCH_CHECK("tvl1_gradient_kernel");
    st.tiles = (int)(grid.x * grid.y);
    st.thr = prm->epsilon * prm->epsilon * (double)A;
    st.level = l;
    for (int wp = 0; wp < prm->warps; ++wp) {
      st.warp = wp;
      tvl1_warp_kernel<<<grid, block, 0, s>>>(lev, lev, fr, Ix, Iy, u, h, w, Ixw, Iyw, grad, rho, st.iter, st.stopped);
      SSNB_LAUNCH_CHECK("tvl1_warp_kernel");
      for (int n = 0; n < prm->iterations; ++n) {
        tvl1_primal_kernel<<<grid, block, 0, s>>>(Ixw, Iyw, grad, rho, pd, u, u, h, w, l_t, theta, st, n);
        SSNB_LAUNCH_CHECK("tvl1_primal_kernel");
        tvl1_dual_kernel<<<grid, block, 0, s>>>(u, pd, pd, h, w, taut, st.iter, n);
        SSNB_LAUNCH_CHECK("tvl1_dual_kernel");
      }
    }
    if (l > 0) {
      float* un = l - 1 == 0 ? flow : (float*)(ws + L.u[(l - 1) & 1]);
      tvl1_resize_kernel<<<tiles(L.hs[l - 1], L.ws[l - 1], 2 * P), block, 0, s>>>(u, h, w, un, L.hs[l - 1], L.ws[l - 1], (float)(1.0 / prm->scale_step));
      SSNB_LAUNCH_CHECK("tvl1_resize_kernel");
    }
  }
  return SSNB_OK;
}

int ssnb_tvl1_stage(int stage, const ssnb_tvl1_params* prm, int n, int height, int width, int out_height, int out_width, double mul,
                    const void* const* in, void* const* out, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("tvl1_stage: " + m); return (int)SSNB_EINVAL; };
  if (const char* bad = check_params(prm)) return fail(bad);
  if (n < 1 || n > kMaxPlanes) return fail("n must be in 1..65535");
  if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide) return fail("height / width outside 1..8192");
  static const int n_in[] = {1, 1, 1, 5, 6, 2}, n_out[] = {1, 1, 2, 4, 1, 1};
  if (stage < SSNB_TVL1_GREY || stage > SSNB_TVL1_DUAL) return fail("unknown stage");
  if (!in || !out) return fail("NULL in or out");
  for (int i = 0; i < n_in[stage]; ++i) if (!in[i]) return fail("NULL input operand");
  for (int i = 0; i < n_out[stage]; ++i) if (!out[i]) return fail("NULL output operand");
  const dim3 grid = tiles(height, width, n), block(BX, BY);
  const StopState none{};
  const float* const* f = (const float* const*)in;
  float* const* o = (float* const*)out;
  switch (stage) {
    case SSNB_TVL1_GREY: {
      const long long N = (long long)n * height * width;
      tvl1_grey_kernel<<<blocks_for(N), kThreads, 0, s>>>((const uint8_t*)in[0], N, o[0]);
      SSNB_LAUNCH_CHECK("tvl1_grey_kernel");
      break;
    }
    case SSNB_TVL1_RESIZE:
      if (out_height < 1 || out_width < 1 || out_height > kMaxSide || out_width > kMaxSide) return fail("out size outside 1..8192");
      if (!std::isfinite(mul)) return fail("mul must be finite");
      tvl1_resize_kernel<<<tiles(out_height, out_width, n), block, 0, s>>>(f[0], height, width, o[0], out_height, out_width, (float)mul);
      SSNB_LAUNCH_CHECK("tvl1_resize_kernel");
      break;
    case SSNB_TVL1_GRADIENT:
      tvl1_gradient_kernel<<<grid, block, 0, s>>>(f[0], nullptr, height, width, o[0], o[1]);
      SSNB_LAUNCH_CHECK("tvl1_gradient_kernel");
      break;
    case SSNB_TVL1_WARP:
      tvl1_warp_kernel<<<grid, block, 0, s>>>(f[0], f[1], nullptr, f[2], f[3], f[4], height, width, o[0], o[1], o[2], o[3], nullptr, nullptr);
      SSNB_LAUNCH_CHECK("tvl1_warp_kernel");
      break;
    case SSNB_TVL1_PRIMAL:
      tvl1_primal_kernel<<<grid, block, 0, s>>>(f[0], f[1], f[2], f[3], f[4], f[5], o[0], height, width, (float)(prm->lambda * prm->theta),
                                                (float)prm->theta, none, 0);
      SSNB_LAUNCH_CHECK("tvl1_primal_kernel");
      break;
    case SSNB_TVL1_DUAL:
      tvl1_dual_kernel<<<grid, block, 0, s>>>(f[0], f[1], o[0], height, width, (float)(prm->tau / prm->theta), nullptr, 0);
      SSNB_LAUNCH_CHECK("tvl1_dual_kernel");
      break;
  }
  return SSNB_OK;
}

int ssnb_flow_planes(const float* flow, int64_t pairs, int height, int width, double bound, uint8_t* planes, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  auto fail = [](const std::string& m) { set_thread_error("flow_planes: " + m); return (int)SSNB_EINVAL; };
  if (!flow || !planes) return fail("NULL flow or planes");
  if (pairs < 1 || height < 1 || width < 1 || height > kMaxSide || width > kMaxSide || pairs > (1LL << 40) / ((long long)height * width))
    return fail("empty or oversized flow");
  if (!(bound > 0 && bound < 1e30)) return fail("bound must be positive and finite");
  const long long N = 2 * pairs * height * width;
  flow_planes_kernel<<<blocks_for(N), kThreads, 0, s>>>(flow, N, bound, planes);
  SSNB_LAUNCH_CHECK("flow_planes_kernel");
  return SSNB_OK;
}

}  // extern "C"
