// SSNB_EXACT_TC glue: error-compensated fp16 operand planes of fp32 tensors.
//
// The reference computes every convolution in fp32 (model_zoo/bninception/layer_factory.py:25-39, no AMP in
// ssn_train.py:81).  tensor-core has no fp32 MMA; an fp32 value x is instead carried as TWO fp16 numbers
//     hi = fp16(x),  lo = fp16(x - float(hi))          (hi + lo == x to ~2^-22 relative, fp16 range permitting)
// and a product a*b is evaluated as a_lo*b_hi + a_hi*b_lo + a_hi*b_hi on the tensor cores with fp32 accumulation
// (umma_conv.cu / umma_wgrad.cu, nseg = 3).  The kernels here produce those planes for tensors that
// do not come out of a convolution epilogue (pool outputs, masked output gradients, weights); the network input's planes
// come from the space-to-depth conversions of s2d_glue.cu.
#include "common.cuh"

namespace ssnb {
namespace {

constexpr int TPB = 256;

// one thread = 8 channels of one pixel: 2 x 16-byte fp32 loads -> 16 bytes of hi + 16 bytes of lo
__global__ void split_view_kernel(const float* __restrict__ src, int spitch, int scoff, long long pixels, int C, float scale,
                                  __half* __restrict__ hi, int hpitch, int hcoff, long long lo_off, int* __restrict__ flag) {
  const int G = C / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pixels * G) return;
  const int g = (int)(i % G);
  const long long p = i / G;
  const float4* s4 = reinterpret_cast<const float4*>(src + p * spitch + scoff + g * 8);
  float4 a = __ldg(s4), b = __ldg(s4 + 1);
  a.x *= scale; a.y *= scale; a.z *= scale; a.w *= scale; b.x *= scale; b.y *= scale; b.z *= scale; b.w *= scale;
  if (flag) {
    const float m = fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))),
                          fmaxf(fmaxf(fabsf(b.x), fabsf(b.y)), fmaxf(fabsf(b.z), fabsf(b.w))));
    if (!(m <= HALF_MAX)) *flag = 1;                   // overflow or NaN under this loss scale
  }
  uint4 h, l;
  split2(a.x, a.y, h.x, l.x); split2(a.z, a.w, h.y, l.y); split2(b.x, b.y, h.z, l.z); split2(b.z, b.w, h.w, l.w);
  __half* hp = hi + p * hpitch + hcoff + g * 8;
  *reinterpret_cast<uint4*>(hp) = h;
  *reinterpret_cast<uint4*>(reinterpret_cast<char*>(hp) + lo_off) = l;
}

__global__ void split_all_kernel(const __grid_constant__ SplitTable t) {
  int ei = 0;
  while (ei + 1 < t.n && (int)blockIdx.x >= t.e[ei + 1].block0) ++ei;
  const SplitEntry& q = t.e[ei];
  const long long i = (long long)((int)blockIdx.x - q.block0) * blockDim.x + threadIdx.x;
  float sc = 1.0f;
  int e = 0;
  const float m = *q.absmax;
  if (m > 0.f && m < INFINITY) { frexpf(m, &e); sc = ldexpf(1.0f, 13 - e); }
  if (i == 0) *q.inv_scale = 1.0f / sc;
  if (i >= q.n) return;
#pragma unroll
  for (int l = 0; l < 2; ++l) {
    const float v = (l ? q.wd : q.wf)[i] * sc;
    __half* hi = l ? q.wd16 : q.wf16;
    const __half h = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(h));
    hi[i] = h;
    *reinterpret_cast<__half*>(reinterpret_cast<char*>(hi + i) + q.plane_bytes) = lo;
    __half* hb = l ? q.wd16_b : q.wf16_b;
    if (hb) {                                   // 1x1 member of a fused sibling block: wd[co][ci] rows stacked, wf[ci][co] as a column block
      const long long j = l ? i : (i / q.cout) * (long long)q.b_pitch + (i % q.cout);
      hb[j] = h;
      *reinterpret_cast<__half*>(reinterpret_cast<char*>(hb + j) + q.b_plane_bytes) = lo;
    }
  }
}

// diagnostic read-back: (hi + lo) * scale as NCHW fp32 (what the consuming tensor-core kernels see)
__global__ void planes_to_nchw_kernel(const __half* __restrict__ hi, long long lo_off, int F, int C, int H, int W, int pitch, int coff,
                                      float scale, float* __restrict__ dst) {
  const long long total = (long long)F * C * H * W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long yx = i % ((long long)H * W);
  const int c = (int)((i / ((long long)H * W)) % C);
  const long long f = i / ((long long)H * W * C);
  const __half* hp = hi + (f * H * W + yx) * pitch + coff + c;
  const __half* lp = reinterpret_cast<const __half*>(reinterpret_cast<const char*>(hp) + lo_off);
  dst[i] = (__half2float(*hp) + __half2float(*lp)) * scale;
}

}  // namespace

int launch_split_view(View src, int F, float scale, View planes, int* flag, cudaStream_t s) {
  if (src.C % 8 || src.pitch % 4 || src.coff % 4 || planes.pitch % 8 || planes.coff % 8 || planes.C != src.C || !planes.lo_off) {
    set_thread_error("split_view: channel counts / offsets must be multiples of 8 and the planes view must carry a LO plane"); return 1; }
  const long long px = (long long)F * src.H * src.W;
  const long long n = px * (src.C / 8);
  split_view_kernel<<<(unsigned)((n + TPB - 1) / TPB), TPB, 0, s>>>((const float*)src.base, src.pitch, src.coff, px, src.C, scale,
                                                                  (__half*)planes.base, planes.pitch, planes.coff, planes.lo_off, flag);
  SSNB_LAUNCH_CHECK("split_view_kernel");
  return 0;
}
int launch_split_all(const SplitTable& t, int total_blocks, cudaStream_t s) {
  if (t.n <= 0) return 0;
  split_all_kernel<<<(unsigned)total_blocks, TPB, 0, s>>>(t);
  SSNB_LAUNCH_CHECK("split_all_kernel");
  return 0;
}
int launch_planes_to_nchw(View planes, int F, float scale, float* dst, cudaStream_t s) {
  const long long n = (long long)F * planes.C * planes.H * planes.W;
  planes_to_nchw_kernel<<<(unsigned)((n + TPB - 1) / TPB), TPB, 0, s>>>((const __half*)planes.base, planes.lo_off, F, planes.C, planes.H, planes.W,
                                                                      planes.pitch, planes.coff, scale, dst);
  SSNB_LAUNCH_CHECK("planes_to_nchw_kernel");
  return 0;
}

}  // namespace ssnb
