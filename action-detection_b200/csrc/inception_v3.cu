// InceptionV3 test-time engine: graph table and forward schedule of the second backbone the reference offers (--arch
// InceptionV3: ssn_models.py:133-139, binary_model.py:175-178; graph model_zoo/bninception/inceptionv3.yaml, class
// model_zoo/bninception/pytorch_load.py:64-67).  Forward only, frozen BatchNorm folded into every convolution, in the
// three precisions of the BNInception engine: EXACT_FP32 on the SIMT kernels of simt_conv.cu, FAST_FP16 and EXACT_TC on the
// wgmma kernel of umma_conv.cu (every convolution, through its tap-table bind: valid stride-1 / stride-2 layers tile at the
// output's geometry with the A map at the input's dims, 1x3 / 3x1 / 1x7 / 7x1 and 25-tap 5x5 tables, and the 3- / 10-channel
// stem over an input zero-padded to 16 channels with its weights padded to match).  The graph records, workspace planner,
// weight pack, pools and value I/O are the BNInception engine's (graph.cuh); this file adds the block table, the stem
// padding and the tap-table binds.  Its handle and ABI section (ssnb_iv3_*) are its own.
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "graph.cuh"
#include "umma_conv.cuh"

namespace {

using namespace ssnb;

constexpr int kInput = 299;
// tensor-core modes: the stem's input channels as the wgmma kernel reads them (K % 8 == 0 and 32-byte pixels), zeros past
// in_channels in the input and in the packed weights
constexpr int kStemK = 16;

}  // namespace

struct ssnb_iv3 : ssnb::Graph<ssnb::GraphOp> {
  ssnb_iv3_config cfg;
  std::vector<UmmaConvPlan> plans;    // tensor-core modes: one forward plan per convolution (bound by ssnb_iv3_set_workspace)
  UmmaContext umma_ctx;
  size_t w0pad = 0;                   // tensor-core modes: the stem's weights zero-padded to kStemK input channels (fp32)
  size_t ws_bytes = 0;
  bool weights_ready = false;

  // input channels of convolution 0 as the kernels read them
  int stem_k() const { return tensor_cores() ? kStemK : convs[0].cin; }
};

namespace {

int fail(int code, const std::string& msg) { set_thread_error(msg); return code; }

// Builds the graph of inceptionv3.yaml in its layer order.  Convolution outputs that are branch ends of a block are
// channel slices of the block's concat buffer (`<block>_join`), in the yaml's concat order, so no concat runs.
struct Builder {
  ssnb_iv3* e;
  int H(int v) const { return e->bufs[e->vals[v].buf].H; }
  int W(int v) const { return e->bufs[e->vals[v].buf].W; }
  int C(int v) const { return e->vals[v].C; }
  // conv kh x kw / stride, pads (ph, pw); dst: -1 = a buffer of its own, else the concat buffer and channel offset
  int conv(const std::string& id, int in, int cout, int kh, int kw, int stride, int ph, int pw, int dst = -1, int coff = 0) {
    const int oh = conv_out(H(in), kh, stride, ph), ow = conv_out(W(in), kw, stride, pw);
    const int v = dst < 0 ? e->whole(id, oh, ow, cout) : e->add_value(id, dst, coff, cout);
    e->convs.push_back({id, C(in), cout, kh, kw, stride, ph, pw});
    GraphOp o; o.kind = OP_CONV; o.id = id; o.in = in; o.out = v; o.conv = (int)e->convs.size() - 1; o.stride = stride;
    e->ops.push_back(o);
    return v;
  }
  int pool(OpKind kind, const std::string& id, int in, int k, int s, int p, int dst = -1, int coff = 0) {
    const int oh = pool_out(H(in), k, s, p), ow = pool_out(W(in), k, s, p);
    const int v = dst < 0 ? e->whole(id, oh, ow, C(in)) : e->add_value(id, dst, coff, C(in));
    GraphOp o; o.kind = kind; o.id = id; o.in = in; o.out = v; o.k = k; o.stride = s; o.pad = p;
    e->ops.push_back(o);
    return v;
  }
  int join(const std::string& p, int HW, int C) { return e->add_buffer(p + "_join", HW, HW, C); }
  int join_val(const std::string& p, int buf) { return e->add_value(p + "_join", buf, 0, e->bufs[buf].C); }

  // 35x35 blocks mixed, mixed_1, mixed_2: 1x1 | 1x1 -> 5x5 | 1x1 -> 3x3 -> 3x3 | avg pool -> 1x1
  int block_a(const std::string& p, int x, int proj) {
    const int hw = H(x), j = join(p, hw, 64 + 64 + 96 + proj);
    conv(p + "_conv", x, 64, 1, 1, 1, 0, 0, j, 0);
    int t = conv(p + "_tower_conv", x, 48, 1, 1, 1, 0, 0);
    conv(p + "_tower_conv_1", t, 64, 5, 5, 1, 2, 2, j, 64);
    t = conv(p + "_tower_1_conv", x, 64, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_1_conv_1", t, 96, 3, 3, 1, 1, 1);
    conv(p + "_tower_1_conv_2", t, 96, 3, 3, 1, 1, 1, j, 128);
    t = pool(OP_AVGPOOL, p + "_tower_2_pool", x, 3, 1, 1);
    conv(p + "_tower_2_conv", t, proj, 1, 1, 1, 0, 0, j, 224);
    return join_val(p, j);
  }
  // 35 -> 17 (mixed_3): 3x3/2 | 1x1 -> 3x3 -> 3x3/2 | max pool
  int block_b(const std::string& p, int x) {
    const int hw = pool_out(H(x), 3, 2, 0), cx = C(x), j = join(p, hw, 384 + 96 + cx);
    conv(p + "_conv", x, 384, 3, 3, 2, 0, 0, j, 0);
    int t = conv(p + "_tower_conv", x, 64, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_conv_1", t, 96, 3, 3, 1, 1, 1);
    conv(p + "_tower_conv_2", t, 96, 3, 3, 2, 0, 0, j, 384);
    pool(OP_MAXPOOL, p + "_pool", x, 3, 2, 0, j, 480);
    return join_val(p, j);
  }
  // 17x17 blocks mixed_4 .. mixed_7 (c7 = 128, 160, 160, 192): 1x1 | 1x1 -> 7x1 -> 1x7 | 1x1 -> 1x7 -> 7x1 -> 1x7 -> 7x1 |
  // avg pool -> 1x1
  int block_c(const std::string& p, int x, int c7) {
    const int hw = H(x), j = join(p, hw, 4 * 192);
    conv(p + "_conv", x, 192, 1, 1, 1, 0, 0, j, 0);
    int t = conv(p + "_tower_conv", x, c7, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_conv_1", t, c7, 7, 1, 1, 3, 0);
    conv(p + "_tower_conv_2", t, 192, 1, 7, 1, 0, 3, j, 192);
    t = conv(p + "_tower_1_conv", x, c7, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_1_conv_1", t, c7, 1, 7, 1, 0, 3);
    t = conv(p + "_tower_1_conv_2", t, c7, 7, 1, 1, 3, 0);
    t = conv(p + "_tower_1_conv_3", t, c7, 1, 7, 1, 0, 3);
    conv(p + "_tower_1_conv_4", t, 192, 7, 1, 1, 3, 0, j, 384);
    t = pool(OP_AVGPOOL, p + "_tower_2_pool", x, 3, 1, 1);
    conv(p + "_tower_2_conv", t, 192, 1, 1, 1, 0, 0, j, 576);
    return join_val(p, j);
  }
  // 17 -> 8 (mixed_8): 1x1 -> 3x3/2 | 1x1 -> 7x1 -> 1x7 -> 3x3/2 | max pool
  int block_d(const std::string& p, int x) {
    const int hw = pool_out(H(x), 3, 2, 0), cx = C(x), j = join(p, hw, 320 + 192 + cx);
    int t = conv(p + "_tower_conv", x, 192, 1, 1, 1, 0, 0);
    conv(p + "_tower_conv_1", t, 320, 3, 3, 2, 0, 0, j, 0);
    t = conv(p + "_tower_1_conv", x, 192, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_1_conv_1", t, 192, 7, 1, 1, 3, 0);
    t = conv(p + "_tower_1_conv_2", t, 192, 1, 7, 1, 0, 3);
    conv(p + "_tower_1_conv_3", t, 192, 3, 3, 2, 0, 0, j, 320);
    pool(OP_MAXPOOL, p + "_pool", x, 3, 2, 0, j, 512);
    return join_val(p, j);
  }
  // 8x8 blocks mixed_9 (avg pool) and mixed_10 (max pool 3x3/1/1): 1x1 | 1x1 -> (3x1 | 1x3) | 1x1 -> 3x3 -> (3x1 | 1x3) |
  // pool -> 1x1
  int block_e(const std::string& p, int x, OpKind pool_kind) {
    const int hw = H(x), j = join(p, hw, 320 + 4 * 384 + 192);
    conv(p + "_conv", x, 320, 1, 1, 1, 0, 0, j, 0);
    int t = conv(p + "_tower_conv", x, 384, 1, 1, 1, 0, 0);
    conv(p + "_tower_mixed_conv", t, 384, 3, 1, 1, 1, 0, j, 320);
    conv(p + "_tower_mixed_conv_1", t, 384, 1, 3, 1, 0, 1, j, 704);
    t = conv(p + "_tower_1_conv", x, 448, 1, 1, 1, 0, 0);
    t = conv(p + "_tower_1_conv_1", t, 384, 3, 3, 1, 1, 1);
    conv(p + "_tower_1_mixed_conv", t, 384, 3, 1, 1, 1, 0, j, 1088);
    conv(p + "_tower_1_mixed_conv_1", t, 384, 1, 3, 1, 0, 1, j, 1472);
    t = pool(pool_kind, p + "_tower_2_pool", x, 3, 1, 1);
    conv(p + "_tower_2_conv", t, 192, 1, 1, 1, 0, 0, j, 1856);
    return join_val(p, j);
  }

  void build(int in_ch) {
    int x = e->add_value("data", e->add_buffer("data", kInput, kInput, e->tensor_cores() ? kStemK : in_ch), 0, in_ch);
    x = conv("conv", x, 32, 3, 3, 2, 0, 0);
    x = conv("conv_1", x, 32, 3, 3, 1, 0, 0);
    x = conv("conv_2", x, 64, 3, 3, 1, 1, 1);
    x = pool(OP_MAXPOOL, "pool", x, 3, 2, 0);
    x = conv("conv_3", x, 80, 1, 1, 1, 0, 0);
    x = conv("conv_4", x, 192, 3, 3, 1, 0, 0);
    x = pool(OP_MAXPOOL, "pool_1", x, 3, 2, 0);
    x = block_a("mixed", x, 32);
    x = block_a("mixed_1", x, 64);
    x = block_a("mixed_2", x, 64);
    x = block_b("mixed_3", x);
    x = block_c("mixed_4", x, 128);
    x = block_c("mixed_5", x, 160);
    x = block_c("mixed_6", x, 160);
    x = block_c("mixed_7", x, 192);
    x = block_d("mixed_8", x);
    x = block_e("mixed_9", x, OP_AVGPOOL);
    x = block_e("mixed_10", x, OP_MAXPOOL);
    // top_cls_pool (8x8 average) writes the caller's feat [F, 2048]; it has no workspace buffer
    GraphOp g; g.kind = OP_GPOOL; g.id = "top_cls_pool"; g.in = x; g.out = -1; g.k = H(x);
    e->ops.push_back(g);
  }
};

// the shared forward storage, then the stem's padded weights
void plan(ssnb_iv3* e) {
  size_t off = e->plan_storage(0, false, e->stem_k(), 0);
  if (e->tensor_cores()) {
    const Conv& c = e->convs[0];
    e->w0pad = off; off = align_up(off + (size_t)c.cout * kStemK * c.kh * c.kw * 4, 1024);
  }
  e->ws_bytes = align_up(off, 1024);
}

// NCHW fp32 frames -> NHWC T with CP >= C channels per pixel, zeros in channels C .. CP-1 (tensor-core modes: the stem's input)
template <typename T>
__global__ void nchw_to_nhwc_pad_kernel(const float* __restrict__ src, int F, int C, int HW, int CP, T* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)F * HW * CP) return;
  const int c = (int)(i % CP);
  const long long p = i / CP;
  const long long f = p / HW, hw = p % HW;
  dst[i] = from_f<T>(c < C ? src[(f * C + c) * HW + hw] : 0.f);
}
template <typename T> int launch_nchw_to_nhwc_pad(const float* src, int F, int C, int HW, int CP, T* dst, cudaStream_t s) {
  const long long n = (long long)F * HW * CP;
  nchw_to_nhwc_pad_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, F, C, HW, CP, dst);
  SSNB_LAUNCH_CHECK("nchw_to_nhwc_pad_kernel");
  return 0;
}
// reference weights [cout][cin][taps] -> [cout][cp][taps], zeros for the input channels cin .. cp-1
__global__ void pad_weights_kernel(const float* __restrict__ w, int cout, int cin, int taps, int cp, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)cout * cp * taps) return;
  const int t = (int)(i % taps), ci = (int)((i / taps) % cp);
  const long long co = i / ((long long)taps * cp);
  out[i] = ci < cin ? w[(co * cin + ci) * taps + t] : 0.f;
}
int launch_pad_weights(const float* w, int cout, int cin, int taps, int cp, float* out, cudaStream_t s) {
  const long long n = (long long)cout * cp * taps;
  pad_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w, cout, cin, taps, cp, out);
  SSNB_LAUNCH_CHECK("pad_weights_kernel");
  return 0;
}

// tensor-core modes: the forward plan of every convolution, taps (r - pad_h, s - pad_w) in the reference's [kh][kw] order.
// No tc_ok-style gate applies: every plan runs on umma_conv_kernel (EXACT_TC: split operands, fp32 epilogue, output planes),
// which tests/test_gpu_inception_v3.py checks launch by launch at the EXACT_TC and FAST bars.
int bind_plans(ssnb_iv3* e) {
  e->plans.assign(e->convs.size(), UmmaConvPlan());
  for (const GraphOp& o : e->ops) {
    if (o.kind != OP_CONV) continue;
    const Conv& c = e->convs[o.conv];
    const PackedConv& pk = e->packed[o.conv];
    const int ck = o.conv == 0 ? kStemK : c.cin;
    int dy[UMMA_MAX_TAPS], dx[UMMA_MAX_TAPS];
    for (int r = 0; r < c.kh; ++r)
      for (int q = 0; q < c.kw; ++q) { dy[r * c.kw + q] = r - c.ph; dx[r * c.kw + q] = q - c.pw; }
    View in = e->operand(o.in);
    in.C = ck;
    UmmaTcOpts tc;
    const UmmaTcOpts* opts = nullptr;
    if (e->exact_tc()) {
      tc.w_lo_off = (long long)pk.wplane; tc.out32 = (float*)e->view(o.out).base; tc.alpha = 1.0f;
      tc.alpha_dev = (const float*)(e->ws + pk.wmax) + 1;
      opts = &tc;
    }
    const __half* w = (const __half*)(e->ws + (e->exact_tc() ? pk.wd16 : pk.wd));
    if (int rc = umma_conv_bind_taps(e->umma_ctx, e->plans[o.conv], in, e->operand(o.out), e->F, ck, c.cout, c.kh * c.kw,
                                     dy, dx, w, (const float*)(e->ws + pk.bias), 1, opts, c.stride))
      return fail(rc, "bind(" + c.id + "): " + thread_error());
  }
  return SSNB_OK;
}

// op `o` over the first n frames
int run_op(ssnb_iv3* e, const GraphOp& o, float* feat, int n, cudaStream_t s) {
  if (o.kind == OP_CONV && e->tensor_cores()) {
    t_tag.phase = 0; t_tag.flop = e->conv_flops(o, n); t_tag.op = o.id.c_str();
    return umma_conv_launch(e->umma_ctx, e->plans[o.conv], s, false, n);
  }
  if (o.kind == OP_CONV) return e->simt_conv_fwd(o, 1, n, s);
  t_tag.phase = 0; t_tag.flop = 0.0; t_tag.op = o.id.c_str();
  if (o.kind != OP_GPOOL) return e->pool_fwd(o, n, s);
  if (!feat) return fail(SSNB_EINVAL, "top_cls_pool needs the feat output pointer");
  return e->gpool_fwd(o, n, feat, s);
}

// the forward of frames [0, n) after the caller's checks
int forward(ssnb_iv3* h, const float* input_nchw, int n, float* feat, cudaStream_t s) {
  const int dv = h->val_by_name["data"];
  const View d = h->view(dv);
  int rc;
  if (!h->tensor_cores()) {
    rc = h->value_write(dv, false, input_nchw, 1.0f, n, s);
  } else {      // every kStemK channels of a pixel written, the padding as zeros
    rc = h->fast() ? launch_nchw_to_nhwc_pad<__half>(input_nchw, n, d.C, d.H * d.W, d.pitch, (__half*)d.base, s)
                   : launch_nchw_to_nhwc_pad<float>(input_nchw, n, d.C, d.H * d.W, d.pitch, (float*)d.base, s);
    if (!rc && h->exact_tc()) {
      View x = d, xp = h->planes(dv);
      x.C = xp.C = d.pitch;
      rc = launch_split_view(x, n, 1.0f, xp, nullptr, s);
    }
  }
  if (rc) return fail(rc, "input layout: " + thread_error());
  for (const GraphOp& o : h->ops)
    if (int rc = run_op(h, o, feat, n, s)) return fail(rc, o.id + ": " + thread_error());
  return SSNB_OK;
}

// the graph of in_channels, planned for cfg
void build(ssnb_iv3* e, const ssnb_iv3_config& cfg) {
  e->cfg = cfg;
  e->F = cfg.frames; e->precision = cfg.precision; e->esz = e->fast() ? 2 : 4;
  Builder{e}.build(cfg.in_channels);
}

}  // namespace

extern "C" {

int ssnb_iv3_num_convs(void) { return 94; }

int ssnb_iv3_conv_info(int idx, int in_channels, char* name, int name_cap, int* cin, int* cout, int* kh, int* kw, int* stride, int* pad_h,
                       int* pad_w) {
  ssnb_iv3 e;
  build(&e, ssnb_iv3_config{in_channels, 1, SSNB_EXACT_FP32, 0});
  if (idx < 0 || idx >= (int)e.convs.size()) return fail(SSNB_EINVAL, "ssnb_iv3_conv_info: index out of range");
  const Conv& c = e.convs[idx];
  if (name && name_cap > 0) snprintf(name, name_cap, "%s", c.id.c_str());
  if (cin) *cin = c.cin;
  if (cout) *cout = c.cout;
  if (kh) *kh = c.kh;
  if (kw) *kw = c.kw;
  if (stride) *stride = c.stride;
  if (pad_h) *pad_h = c.ph;
  if (pad_w) *pad_w = c.pw;
  return SSNB_OK;
}

int ssnb_iv3_create(const ssnb_iv3_config* cfg, ssnb_iv3_handle* out) {
  if (!cfg || !out) return fail(SSNB_EINVAL, "ssnb_iv3_create: null argument");
  *out = nullptr;
  if (cfg->in_channels != 3 && cfg->in_channels != 10) return fail(SSNB_EINVAL, "ssnb_iv3_create: in_channels must be 3 (RGB) or 10 (Flow)");
  if (cfg->frames < 1) return fail(SSNB_EINVAL, "ssnb_iv3_create: frames must be >= 1");
  if (cfg->precision != SSNB_EXACT_FP32 && cfg->precision != SSNB_FAST_FP16 && cfg->precision != SSNB_EXACT_TC)
    return fail(SSNB_EINVAL, "ssnb_iv3_create: unknown precision");
  ssnb_iv3* e = new ssnb_iv3();
  build(e, *cfg);
  plan(e);
  *out = e;
  return SSNB_OK;
}

int ssnb_iv3_destroy(ssnb_iv3_handle h) { delete h; return SSNB_OK; }

size_t ssnb_iv3_workspace_bytes(ssnb_iv3_handle h) { return h ? h->ws_bytes : 0; }

int ssnb_iv3_set_workspace(ssnb_iv3_handle h, void* dev_ptr, size_t bytes) {
  if (!h) return fail(SSNB_EINVAL, "null handle");
  if (!dev_ptr || bytes < h->ws_bytes) return fail(SSNB_EINVAL, "ssnb_iv3_set_workspace: workspace too small");
  if (((uintptr_t)dev_ptr) % 1024) return fail(SSNB_EINVAL, "ssnb_iv3_set_workspace: workspace must be 1024-byte aligned");
  h->ws = (char*)dev_ptr;
  h->weights_ready = false;
  return h->tensor_cores() ? bind_plans(h) : SSNB_OK;
}

int ssnb_iv3_pack_weights(ssnb_iv3_handle h, const float* const* w, const float* const* b, const float* const* gamma, const float* const* beta,
                          const float* const* mean, const float* const* var, void* stream) {
  if (!h || !w || !b || !gamma || !beta || !mean || !var) return fail(SSNB_EINVAL, "ssnb_iv3_pack_weights: null argument");
  if (!h->ws) return fail(SSNB_ESTATE, "ssnb_iv3_pack_weights: set the workspace first");
  for (size_t i = 0; i < h->convs.size(); ++i)
    if (!w[i] || !b[i] || !gamma[i] || !beta[i] || !mean[i] || !var[i])
      return fail(SSNB_EINVAL, "ssnb_iv3_pack_weights: null tensor for " + h->convs[i].id);
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<const float*> ws(w, w + h->convs.size());
  if (h->tensor_cores()) {       // the stem's kernels over the zero-padded input channels
    const Conv& c = h->convs[0];
    if (int rc = launch_pad_weights(w[0], c.cout, c.cin, c.kh * c.kw, kStemK, (float*)(h->ws + h->w0pad), s))
      return fail(rc, "ssnb_iv3_pack_weights: " + thread_error());
    ws[0] = (const float*)(h->ws + h->w0pad);
  }
  if (int rc = h->pack_weights(ws.data(), b, gamma, beta, mean, var, h->stem_k(), [](size_t, PackEntry&, SplitEntry*) {},
                               "ssnb_iv3_pack_weights", s))
    return rc;
  h->weights_ready = true;
  return SSNB_OK;
}

int ssnb_iv3_forward(ssnb_iv3_handle h, const float* input_nchw, float* feat, void* stream) {
  if (!h || !input_nchw || !feat) return fail(SSNB_EINVAL, "ssnb_iv3_forward: null argument");
  if (!h->ws || !h->weights_ready) return fail(SSNB_ESTATE, "ssnb_iv3_forward: workspace / weights not set");
  return forward(h, input_nchw, h->F, feat, (cudaStream_t)stream);
}

int ssnb_iv3_forward_frames(ssnb_iv3_handle h, const float* input_nchw, int frames, float* feat, void* stream) {
  if (!h || !input_nchw || !feat) return fail(SSNB_EINVAL, "ssnb_iv3_forward_frames: null argument");
  if (frames < 1 || frames > h->F) return fail(SSNB_EINVAL, "ssnb_iv3_forward_frames: frames must be in 1 .. " + std::to_string(h->F));
  if (!h->ws || !h->weights_ready) return fail(SSNB_ESTATE, "ssnb_iv3_forward_frames: workspace / weights not set");
  return forward(h, input_nchw, frames, feat, (cudaStream_t)stream);
}

int ssnb_iv3_num_ops(ssnb_iv3_handle h) { return h ? (int)h->ops.size() : 0; }

int ssnb_iv3_op_info(ssnb_iv3_handle h, int op, char* kind, int kind_cap, char* in_name, int in_cap, char* out_name, int out_cap, int* conv,
                     int* k, int* stride, int* pad) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(SSNB_EINVAL, "ssnb_iv3_op_info: op out of range");
  const GraphOp& o = h->ops[op];
  if (kind && kind_cap > 0) snprintf(kind, kind_cap, "%s", kOpKindName[o.kind]);
  if (in_name && in_cap > 0) snprintf(in_name, in_cap, "%s", h->vals[o.in].name.c_str());
  if (out_name && out_cap > 0) snprintf(out_name, out_cap, "%s", o.out >= 0 ? h->vals[o.out].name.c_str() : "top_cls_global_pool");
  if (conv) *conv = o.conv;
  if (k) *k = o.k;
  if (stride) *stride = o.stride;
  if (pad) *pad = o.pad;
  return SSNB_OK;
}

int ssnb_iv3_value_info(ssnb_iv3_handle h, const char* name, int* c, int* hh, int* ww, char* buffer, int buffer_cap, int* coff) {
  if (!h) return fail(SSNB_EINVAL, "null handle");
  const int v = h->value_of(name);
  if (v < 0) return fail(SSNB_EINVAL, std::string("ssnb_iv3_value_info: unknown value ") + (name ? name : "(null)"));
  const Buffer& b = h->bufs[h->vals[v].buf];
  if (c) *c = h->vals[v].C;
  if (hh) *hh = b.H;
  if (ww) *ww = b.W;
  if (buffer && buffer_cap > 0) snprintf(buffer, buffer_cap, "%s", b.name.c_str());
  if (coff) *coff = h->vals[v].coff;
  return SSNB_OK;
}

int ssnb_iv3_value_write(ssnb_iv3_handle h, const char* name, const float* src_nchw, void* stream) {
  if (!h || !src_nchw || !h->ws) return fail(SSNB_EINVAL, "ssnb_iv3_value_write: null argument or no workspace");
  const int v = h->value_of(name);
  if (v < 0) return fail(SSNB_EINVAL, std::string("ssnb_iv3_value_write: unknown value ") + (name ? name : "(null)"));
  const int rc = h->value_write(v, false, src_nchw, 1.0f, h->F, (cudaStream_t)stream);
  return rc ? fail(rc, thread_error()) : SSNB_OK;
}

int ssnb_iv3_value_read(ssnb_iv3_handle h, const char* name, int planes, float* dst_nchw, void* stream) {
  if (!h || !dst_nchw || !h->ws) return fail(SSNB_EINVAL, "ssnb_iv3_value_read: null argument or no workspace");
  const int v = h->value_of(name);
  if (v < 0) return fail(SSNB_EINVAL, std::string("ssnb_iv3_value_read: unknown value ") + (name ? name : "(null)"));
  if (planes && !h->exact_tc()) return fail(SSNB_ESTATE, "ssnb_iv3_value_read: operand planes exist in EXACT_TC only");
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = planes ? h->planes_read(v, false, 1.0f, dst_nchw, s) : h->value_read(v, false, 1.0f, dst_nchw, s);
  return rc ? fail(rc, thread_error()) : SSNB_OK;
}

int ssnb_iv3_run_op(ssnb_iv3_handle h, int op, float* feat, void* stream) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(SSNB_EINVAL, "ssnb_iv3_run_op: op out of range");
  if (!h->ws || !h->weights_ready) return fail(SSNB_ESTATE, "ssnb_iv3_run_op: workspace / weights not set");
  if (int rc = run_op(h, h->ops[op], feat, h->F, (cudaStream_t)stream)) return fail(rc, h->ops[op].id + ": " + thread_error());
  return SSNB_OK;
}

}  // extern "C"
