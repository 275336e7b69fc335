// BNInception execution engine: graph table, workspace planner, forward/backward schedules and the
// backbone part of the C ABI (include/ssnb.h).  Replaces the reference's YAML-driven op
// interpreter (model_zoo/bninception/pytorch_load.py:8-61, layer_factory.py:25-83,
// bn_inception.yaml) and the autograd graph PyTorch builds from it.
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include <cuda_profiler_api.h>

#include "../../include/ssnb.h"
#include "common.cuh"
#include "graph.cuh"
#include "umma_conv.cuh"

namespace ssnb {

std::atomic<long long> g_launches{0};
static thread_local std::string t_error;
void set_thread_error(const std::string& s) { t_error = s; }
const std::string& thread_error() { return t_error; }

// ---- per-launch timing session (see common.cuh) ---------------------------------------------------
thread_local bool t_timing = false;
thread_local LaunchTag t_tag;
struct TimingMark { const char* what; LaunchTag tag; std::string op; cudaEvent_t ev; };
static thread_local std::vector<TimingMark> t_marks;
static thread_local std::vector<cudaEvent_t> t_event_pool;
static thread_local std::string t_report;
static cudaEvent_t timing_event() {
  if (!t_event_pool.empty()) { cudaEvent_t e = t_event_pool.back(); t_event_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
void timing_mark(const char* what, cudaStream_t s) {
  TimingMark m{what, t_tag, t_tag.op ? t_tag.op : "", timing_event()};
  m.tag.op = nullptr;
  if (m.ev && cudaEventRecord(m.ev, s) == cudaSuccess) t_marks.push_back(m);
  else cudaGetLastError();
  // FLOPs, name and tiles belong to the one launch they were set for
  t_tag.flop = 0.0; t_tag.op = nullptr; t_tag.tiles = 0; t_tag.block_n = 0;
}

// closes the session and waits for its last launch; false if the events cannot be read
static bool timing_close() {
  t_timing = false;
  if (t_marks.empty()) return false;
  if (cudaEventSynchronize(t_marks.back().ev) != cudaSuccess) { cudaGetLastError(); return false; }
  return true;
}

// ---- graph table ---------------------------------------------------------------------------------
struct BlockSpec { const char* name; int c1, c3r, c3, cdr, cd1, cd2; int pool_max; int cproj; int stride; };
// bn_inception.yaml:30-551
static const BlockSpec kBlocks[10] = {
    {"3a", 64, 64, 64, 64, 96, 96, 0, 32, 1},      {"3b", 64, 64, 96, 64, 96, 96, 0, 64, 1},
    {"3c", 0, 128, 160, 64, 96, 96, 1, 0, 2},      {"4a", 224, 64, 96, 96, 128, 128, 0, 128, 1},
    {"4b", 192, 96, 128, 96, 128, 128, 0, 128, 1}, {"4c", 160, 128, 160, 128, 160, 160, 0, 128, 1},
    {"4d", 96, 128, 192, 160, 192, 192, 0, 128, 1}, {"4e", 0, 128, 192, 192, 256, 256, 1, 0, 2},
    {"5a", 352, 192, 320, 160, 224, 224, 0, 128, 1}, {"5b", 352, 192, 320, 192, 224, 224, 1, 128, 1}};

// every convolution is square: k x k, stride, padding pad on all sides
static std::vector<Conv> conv_table(int in_ch) {
  std::vector<Conv> v;
  auto add = [&](const std::string& id, int cin, int cout, int k, int stride, int pad) { v.push_back({id, cin, cout, k, k, stride, pad, pad}); };
  add("conv1_7x7_s2", in_ch, 64, 7, 2, 3);
  add("conv2_3x3_reduce", 64, 64, 1, 1, 0);
  add("conv2_3x3", 64, 192, 3, 1, 1);
  int cx = 192;
  for (const BlockSpec& b : kBlocks) {
    std::string p = std::string("inception_") + b.name + "_";
    if (b.c1) add(p + "1x1", cx, b.c1, 1, 1, 0);
    add(p + "3x3_reduce", cx, b.c3r, 1, 1, 0);
    add(p + "3x3", b.c3r, b.c3, 3, b.stride, 1);
    add(p + "double_3x3_reduce", cx, b.cdr, 1, 1, 0);
    add(p + "double_3x3_1", b.cdr, b.cd1, 3, 1, 1);
    add(p + "double_3x3_2", b.cd1, b.cd2, 3, b.stride, 1);
    if (b.cproj) add(p + "pool_proj", cx, b.cproj, 1, 1, 0);
    cx = b.c1 + b.c3 + b.cd2 + (b.cproj ? b.cproj : cx);
  }
  return v;
}

// ---- planned objects -----------------------------------------------------------------------------
// the forward fields (graph.cuh) and what the training schedule and the tensor-core binding add
struct Op : GraphOp {
  int grad_accumulate = 0;  // backward: dIn += (another consumer wrote first)
  int wsplits = 1, wrows = 0;
  int tsplits = 1;                // upper bound of the split count the tensor-core weight-gradient planner may pick (sizes `partial`)
  size_t partial_off = 0, bias_partial_off = 0;   // this layer's split-K partials (own region: finalised in one batch)
  UmmaConvPlan umma;        // tensor-core forward plan (FAST mode, stride-1 layers)
  UmmaConvPlan umma_dgrad;  // tensor-core data-gradient plan
  UmmaWgradPlan umma_wgrad; // tensor-core weight-gradient plan
  int pool_consumer = -1;   // conv whose only consumer is a k3/s2 max pool: that pool's op index (backward gather is folded in)
  bool folded_into_conv = false;   // max pool whose backward runs inside its producer conv's mask+bias pass
  bool dgrad_masks = false; // this op's data gradient is the LAST writer of d(in): it applies the ReLU mask of in
  bool bias_in_wgrad = false;// conv: bias gradient comes out of the tensor-core weight-gradient kernel (ones operand)
  bool dy_premasked = false;// conv: d(out) arrives already masked, the backward pass only needs the bias column sums
  bool raw = false;         // conv whose BatchNorm runs unfused in training mode: no fold, no ReLU in the epilogue, no ReLU mask in backward
  int fuse_role = 0;        // sibling 1x1 fusion: 1 = leader (launches the fused kernels), 2 = follower
  int fuse_block = -1;
};
// the 1x1 convolutions of one inception block that read the block input (1x1, 3x3_reduce, double_3x3_reduce)
struct FusedBlock {
  int op1 = -1, op_r3 = -1, op_rd = -1;   // op indices (op1 = -1 for 3c/4e)
  int c1 = 0, c3r = 0, cdr = 0, cx = 0;
  size_t w_fwd = 0, bias = 0, w_dg = 0;   // stacked forward weights/bias, K-concatenated data-gradient weights
  size_t w_fwd_plane = 0, w_dg_plane = 0, wmax = 0;   // EXACT_TC: LO plane distance of both; shared (absmax, 1/scale) slot of the three layers
  UmmaConvPlan fwd, dgrad;
  bool enabled = false;
};

}  // namespace ssnb

using namespace ssnb;

struct ssnb_engine : ssnb::Graph<ssnb::Op> {
  ssnb_config cfg;
  size_t up_plane = 0, s2d_plane = 0, s2d_w_plane = 0;
  int* tc_flag = nullptr;           // device int: set when a split pass saw |x * grad_scale| beyond the fp16 range
  size_t tc_flag_off = 0;
  // tensor-core modes: the backward's gradient exponent, [0] = 2^k, [1] = 2^-k (launch_grad_exponent, at the start of every
  // backward).  Every gradient buffer holds dz * 2^k (FAST: times grad_scale as well); the global pool's backward multiplies
  // by 2^k and every kernel that writes a gradient the caller sees (dW, db, dgamma, dbeta) by 2^-k
  float* gscale = nullptr;           // in the flag's 256-byte slot, 16 bytes after the flag
  bool bn1_train = false;           // bn_mode='partial': the first BatchNorm2d in training mode (bn_train.cu)
  const float *bn1_gamma = nullptr, *bn1_beta = nullptr; float *bn1_rmean = nullptr, *bn1_rvar = nullptr, *bn1_dgamma = nullptr, *bn1_dbeta = nullptr;
  float bn1_momentum = 0.1f, bn1_eps = 1e-5f;
  size_t bn_stat_off = 0, bn_partial_off = 0;
  std::vector<FusedBlock> fused;
  size_t ws_bytes = 0, partial_off = 0, partial_bytes = 0, bpartial_off = 0;
  size_t s2d_off = 0, s2d_w_off = 0, up_off = 0;   // tensor-core modes: space-to-depth input + weights, zero-upsampled dz
  bool fold_pools = true;                            // SSNB_DISABLE_FUSION=1 also keeps the max-pool backward separate
  bool s2d_ready = false;                            // backbone_fwd converted the input directly
  int Cs = 0;                                        // channels of the space-to-depth input (4*Cin rounded up to 8)
  int conv1_tsplits = 128;                           // tensor-core modes: bound of conv1's weight-gradient split count (sizes its partials)
  bool weights_ready = false;
  std::vector<float*> dw, db;
  std::vector<int> pending_finalize;  // conv ops whose partials wait for the batched finalize of this backward
  int grad_accumulate = 0;          // 1: dw/db += (autograd-style accumulation into existing .grad), 0: overwrite
  std::string error;
  long long launches0 = 0;
  UmmaContext umma_ctx;

  int fail(int code, const std::string& msg) { error = msg; return code; }
  const float* grad_scale_dev() const { return tensor_cores() ? gscale : nullptr; }      // 2^k (nullptr: 1)
  const float* grad_unscale_dev() const { return tensor_cores() ? gscale + 1 : nullptr; }  // 2^-k
  int nplanes() const { return exact_tc() ? 2 : 1; }                     // fp16 operand planes per tensor-core operand
  // tensor-core weight operands of a convolution: forward [tap][co][ci], data gradient [tap][ci][co]
  const __half* w_fwd(const PackedConv& p) const { return (const __half*)(ws + (exact_tc() ? p.wd16 : p.wd)); }
  const __half* w_dgrad(const PackedConv& p) const { return (const __half*)(ws + (exact_tc() ? p.wf16 : p.wf)); }
  // EXACT_TC bind options (nullptr in FAST): LO weight plane `w_lo_off` bytes after the HI plane, fp32 result `out32`, result
  // scale alpha times 1 / the weights' power-of-two plane scale, which the split pass writes to the second float of `wmax`
  const UmmaTcOpts* tc_opts(UmmaTcOpts& t, size_t w_lo_off, void* out32, float alpha, size_t wmax) const {
    if (!exact_tc()) return nullptr;
    t.w_lo_off = (long long)w_lo_off; t.out32 = (float*)out32; t.alpha = alpha; t.alpha_dev = (const float*)(ws + wmax) + 1;
    return &t;
  }
};

namespace ssnb {

// profiling aid: SSNB_PROFILE_FWD_OPS / SSNB_PROFILE_BWD_OPS = comma-separated op ids; the engine brackets those ops of a whole
// forward / backward pass with cudaProfilerStart/Stop (use with `ncu --profile-from-start off`)
static bool profiled_op(const char* env, const std::string& id) {
  const char* e = getenv(env);
  if (!e || !*e) return false;
  const std::string list = std::string(",") + e + ",";
  return list.find("," + id + ",") != std::string::npos;
}
// diagnostic switch `name` set to 1
static bool env_on(const char* name) {
  const char* v = getenv(name);
  return v && v[0] == '1';
}
// SM count of the current device (the H100 SXM's 132 where none is visible: planning without a GPU)
static int device_sms() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) {
    cudaGetLastError();
    return 132;
  }
  return sms;
}

static void build_graph(ssnb_engine* e) {
  const int cin = e->cfg.in_channels;
  e->convs = conv_table(cin);
  int ci = 0;
  auto conv_op = [&](int in, int out) {
    const Conv& c = e->convs[ci];
    Op o; o.kind = OP_CONV; o.id = c.id; o.in = in; o.out = out; o.conv = ci;
    o.k = c.kh; o.stride = c.stride; o.pad = c.ph;
    e->ops.push_back(o);
    ++ci;
  };
  auto pool_op = [&](OpKind kind, const std::string& id, int in, int out, int k, int s, int p) {
    Op o; o.kind = kind; o.id = id; o.in = in; o.out = out; o.k = k; o.stride = s; o.pad = p;
    e->ops.push_back(o);
  };
  int x = e->whole("data", 224, 224, cin);
  int v;
  if (e->bn1_train) {
    const int raw = e->whole("conv1_7x7_s2_raw", 112, 112, 64); conv_op(x, raw); e->ops.back().raw = true;
    v = e->whole("conv1_7x7_s2_bn", 112, 112, 64);
    pool_op(OP_BN1, "conv1_7x7_s2_bn", raw, v, 0, 1, 0); x = v;
  } else {
    v = e->whole("conv1_7x7_s2_bn", 112, 112, 64); conv_op(x, v); x = v;
  }
  v = e->whole("pool1_3x3_s2", 56, 56, 64); pool_op(OP_MAXPOOL, "pool1_3x3_s2", x, v, 3, 2, 0); x = v;
  v = e->whole("conv2_3x3_reduce_bn", 56, 56, 64); conv_op(x, v); x = v;
  v = e->whole("conv2_3x3_bn", 56, 56, 192); conv_op(x, v); x = v;
  v = e->whole("pool2_3x3_s2", 28, 28, 192); pool_op(OP_MAXPOOL, "pool2_3x3_s2", x, v, 3, 2, 0); x = v;
  int H = 28, cx = 192;
  for (const BlockSpec& b : kBlocks) {
    const std::string p = std::string("inception_") + b.name + "_";
    const int OHW = (b.stride == 2) ? pool_out(H, 3, 2, 0) : H;
    const int ctot = b.c1 + b.c3 + b.cd2 + (b.cproj ? b.cproj : cx);
    const int cat = e->add_buffer(p + "output", OHW, OHW, ctot);
    const int red = e->add_buffer(p + "reduce", H, H, b.c3r + b.cdr);
    int off = 0;
    if (b.c1) { v = e->add_value(p + "1x1_bn", cat, off, b.c1); conv_op(x, v); off += b.c1; }
    int r3 = e->add_value(p + "3x3_reduce_bn", red, 0, b.c3r); conv_op(x, r3);
    v = e->add_value(p + "3x3_bn", cat, off, b.c3); conv_op(r3, v); off += b.c3;
    int rd = e->add_value(p + "double_3x3_reduce_bn", red, b.c3r, b.cdr); conv_op(x, rd);
    int d1 = e->whole(p + "double_3x3_1_bn", H, H, b.cd1); conv_op(rd, d1);
    v = e->add_value(p + "double_3x3_2_bn", cat, off, b.cd2); conv_op(d1, v); off += b.cd2;
    if (b.stride == 2) {
      v = e->add_value(p + "pool", cat, off, cx);
      pool_op(OP_MAXPOOL, p + "pool", x, v, 3, 2, 0);
    } else {
      int pl = e->whole(p + "pool", H, H, cx);
      pool_op(b.pool_max ? OP_MAXPOOL : OP_AVGPOOL, p + "pool", x, pl, 3, 1, 1);
      v = e->add_value(p + "pool_proj_bn", cat, off, b.cproj); conv_op(pl, v);
    }
    x = e->add_value(p + "output", cat, 0, ctot);
    H = OHW; cx = ctot;
  }
  // global_pool writes the caller's feat tensor; it has no workspace buffer
  Op g; g.kind = OP_GPOOL; g.id = "global_pool"; g.in = x; g.out = -1; g.k = 7;
  e->ops.push_back(g);
}

// The fixed-size slots first (their sizes are multiples of 1024, so every region behind them keeps its alignment), then the
// shared forward storage (graph.cuh) with one extra (absmax, 1 / scale) slot per fused sibling block, then the training and
// tensor-core regions of this engine.
static void plan(ssnb_engine* e) {
  const size_t F = (size_t)e->F;
  size_t off = 0;
  e->tc_flag_off = off; off = align_up(off + 256, 1024);      // gradient overflow flag (every mode), gradient exponent
  if (e->bn1_train) { e->bn_stat_off = off; off = align_up(off + 4 * 64 * 4, 1024); e->bn_partial_off = off; off = align_up(off + (size_t)1200 * 2 * 64 * 4, 1024); }
  off = e->plan_storage(off, e->cfg.training != 0, e->convs[0].cin, 16);
  // backward bookkeeping: accumulate flags + split-K sizing
  size_t pmax = 0;
  if (e->cfg.training) {
    std::vector<char> written(e->vals.size(), 0);
    for (int i = (int)e->ops.size() - 1; i >= 0; --i) {
      Op& o = e->ops[i];
      o.grad_accumulate = written[o.in];
      written[o.in] = 1;
      if (o.kind == OP_CONV) {
        const Conv& c = e->convs[o.conv];
        const Buffer& ob = e->bufs[e->vals[o.out].buf];
        const long long M = (long long)F * ob.H * ob.W;
        const int taps = c.kh * c.kw;
        const bool flat = c.cin < 16;
        const long long tiles = (long long)((c.cout + 63) / 64) * (flat ? (taps * c.cin + 63) / 64 : ((c.cin + 63) / 64) * taps);
        long long splits = (592 + tiles - 1) / tiles;
        if (splits > 128) splits = 128;
        while (splits > 1 && M / splits < 256) --splits;
        long long rows = (M + splits - 1) / splits;
        rows = (rows + 15) / 16 * 16;
        splits = (M + rows - 1) / rows;
        o.wsplits = (int)splits; o.wrows = (int)rows;
        // tensor-core path: one CTA per SM is resident, so the planner wants num_sms / (M tiles x N tiles x tap groups) pixel
        // splits, and whole waves more where a split would sum more than UMMA_WGRAD_MAX_PTILES pixel tiles; the SIMT
        // heuristic above used to cap it and left most SMs idle on most 3x3 layers
        {
          const int chunks = (c.cin + 63) / 64, n_tiles = (chunks + 3) / 4, block_n = ((chunks + n_tiles - 1) / n_tiles) * 64;
          const int tpc = std::max(1, 4 / (block_n / 64));
          const int ctas = ((c.cout + 127) / 128) * n_tiles * ((taps + tpc - 1) / tpc);
          o.tsplits = std::max(o.wsplits, std::min(128, umma_wgrad_splits(ctas, umma_wgrad_ptiles(ob.W, ob.H, e->F), device_sms())));
        }
        if (e->tensor_cores()) splits = std::max<long long>(splits, o.tsplits);
        const size_t need = (size_t)splits * taps * c.cout * c.cin * 4;
        if (need > pmax) pmax = need;
      }
    }
  }
  if (e->tensor_cores()) {
    for (int i = 0; i < (int)e->ops.size(); ++i) {
      const Op& o = e->ops[i];
      if (o.kind != OP_CONV || o.k != 1) continue;
      const std::string& id = o.id;
      const std::string suf = "_3x3_reduce";
      if (id.size() < suf.size() || id.compare(id.size() - suf.size(), suf.size(), suf) != 0 || id.find("double") != std::string::npos) continue;
      const std::string pre = id.substr(0, id.size() - suf.size() + 1);      // "inception_3a_"
      FusedBlock fb; fb.op_r3 = i;
      for (int j = 0; j < (int)e->ops.size(); ++j) {
        if (e->ops[j].id == pre + "1x1") fb.op1 = j;
        if (e->ops[j].id == pre + "double_3x3_reduce") fb.op_rd = j;
      }
      if (fb.op_rd < 0) continue;
      fb.cx = e->convs[o.conv].cin; fb.c3r = e->convs[o.conv].cout; fb.cdr = e->convs[e->ops[fb.op_rd].conv].cout;
      fb.c1 = fb.op1 >= 0 ? e->convs[e->ops[fb.op1].conv].cout : 0;
      const int n = fb.c1 + fb.c3r + fb.cdr, kf = (fb.c1 + 63) / 64 * 64 + fb.c3r + fb.cdr;
      fb.w_fwd_plane = align_up((size_t)n * fb.cx * 2, 1024); fb.w_dg_plane = align_up((size_t)fb.cx * kf * 2, 1024);
      if (e->exact_tc()) fb.w_fwd_plane = fb.w_dg_plane = std::max(fb.w_fwd_plane, fb.w_dg_plane);     // one LO-plane distance for both (split_all_kernel)
      fb.w_fwd = off; off += e->nplanes() * fb.w_fwd_plane;
      fb.bias = off; off = align_up(off + (size_t)n * 4, 256);
      fb.w_dg = off; off += e->nplanes() * fb.w_dg_plane;
      if (e->exact_tc()) {       // the three layers share ONE power-of-two plane scale (their operands are stacked / K-concatenated in one launch)
        if (e->fused.size() >= 16) continue;
        fb.wmax = e->wmax_off + (e->convs.size() + e->fused.size()) * 8;
        for (int j : {fb.op1, fb.op_r3, fb.op_rd}) if (j >= 0) e->packed[e->ops[j].conv].wmax = fb.wmax;
      }
      e->fused.push_back(fb);
    }
  }
  if (e->tensor_cores()) {
    // convolutions whose only consumer is a k3/s2/pad0 max pool: that pool's backward gather is folded into their mask pass,
    // whose vector width must divide the channel count
    for (int i = 0; i < (int)e->ops.size(); ++i) {
      Op& po = e->ops[i];
      if (po.kind != OP_MAXPOOL || po.k != 3 || po.stride != 2 || po.pad != 0) continue;
      int producer = -1, consumers = 0;
      for (int j = 0; j < (int)e->ops.size(); ++j) {
        if (e->ops[j].out == po.in && e->ops[j].kind == OP_CONV) producer = j;
        if (e->ops[j].in == po.in) ++consumers;
      }
      if (producer >= 0 && consumers == 1 && e->vals[po.in].C % (e->fast() ? VEC_WIDTH<__half> : VEC_WIDTH<float>) == 0) { e->ops[producer].pool_consumer = i; po.folded_into_conv = true; }
    }
    // fp16 operand regions: one plane in FAST (the next region starts 1024-aligned behind it), hi + lo planes `plane`
    // bytes apart in EXACT_TC
    auto operand_region = [&](size_t bytes, size_t& plane) {
      const size_t at = off;
      if (e->exact_tc()) { plane = align_up(bytes, 1024); off += 2 * plane; }
      else off = align_up(off + bytes, 1024);
      return at;
    };
    e->Cs = (4 * e->cfg.in_channels + 7) / 8 * 8;
    // conv1's weight gradient (4 taps over the 4*Cs-channel space-to-depth input, one M tile): 128 splits, or as many whole
    // waves as keep a split at most UMMA_WGRAD_MAX_PTILES pixel tiles long where 128 would not
    {
      const int chunks = (4 * e->Cs + 63) / 64, n_tiles = (chunks + 3) / 4, block_n = ((chunks + n_tiles - 1) / n_tiles) * 64;
      const int tpc = std::min(4, std::max(1, 4 / (block_n / 64)));
      const int ptiles = umma_wgrad_ptiles(112, 112, e->F);
      if ((ptiles + UMMA_WGRAD_MAX_PTILES - 1) / UMMA_WGRAD_MAX_PTILES > 128)
        e->conv1_tsplits = umma_wgrad_splits(n_tiles * ((4 + tpc - 1) / tpc), ptiles, device_sms());
    }
    e->s2d_off = operand_region(F * 112 * 112 * 4 * e->Cs * 2, e->s2d_plane);      // packed: 4 horizontal neighbours per pixel
    e->s2d_w_off = operand_region((size_t)16 * 64 * e->Cs * 2, e->s2d_w_plane);
    if (e->cfg.training) {
      size_t up = 0;
      for (const Op& o : e->ops)
        if (o.kind == OP_CONV && o.stride == 2 && o.conv != 0) {
          const Buffer& ib = e->bufs[e->vals[o.in].buf];
          up = std::max(up, F * ib.H * ib.W * (size_t)e->convs[o.conv].cout * 2);
        }
      e->up_off = operand_region(up, e->up_plane);
      pmax = std::max(pmax, (size_t)e->conv1_tsplits * 16 * 64 * e->Cs * 4);
    }
  }
  e->partial_off = off; e->partial_bytes = pmax; off = align_up(off + pmax, 1024);
  if (e->cfg.training)
    for (Op& o : e->ops)
      if (o.kind == OP_CONV) {
        const Conv& c = e->convs[o.conv];
        const int nsplit = e->tensor_cores() ? std::max(o.wsplits, o.tsplits) : o.wsplits;
        size_t need = (size_t)nsplit * c.kh * c.kw * c.cout * c.cin * 4;
        if (o.conv == 0 && e->tensor_cores()) need = std::max(need, (size_t)e->conv1_tsplits * 16 * 64 * e->Cs * 4);
        o.partial_off = off; off = align_up(off + need, 1024);
        o.bias_partial_off = off; off = align_up(off + (size_t)std::max(nsplit, 128) * c.cout * 4, 256);
      }
  e->bpartial_off = off; off = align_up(off + (size_t)1024 * 512 * 4, 1024);   // column-sum partials: <= 1024 CTAs x 512 channels
  e->ws_bytes = off;
}

// ---- op execution --------------------------------------------------------------------------------
#define DISPATCH(e, call_f, call_h) ((e)->fast() ? (call_h) : (call_f))

// timing tags (common.cuh): the next launch is in pass `phase`, `flop` the algorithmic FLOPs of the convolution op `op`
static inline void tag_next(int phase, double flop, const char* op = nullptr) { t_tag.phase = phase; t_tag.flop = flop; t_tag.op = op; }
// a fused sibling launch is named after its convolutions, "a+b+c"
static thread_local std::string t_fused_name;
static const char* fused_name(const ssnb_engine* e, const FusedBlock& fb) {
  if (!t_timing) return nullptr;
  t_fused_name.clear();
  for (int j : {fb.op1, fb.op_r3, fb.op_rd})
    if (j >= 0) t_fused_name += (t_fused_name.empty() ? "" : "+") + e->ops[j].id;
  return t_fused_name.c_str();
}

// the forward of op `o` over the first n frames (n = F but for ssnb_backbone_fwd_frames, which bn1_train engines refuse)
static int run_fwd(ssnb_engine* e, const Op& o, float* feat, int n, cudaStream_t s) {
  tag_next(0, 0.0);
  if (o.kind == OP_CONV && o.umma.enabled) {
    // tensor-core convolution (EXACT_TC: reads the input's hi/lo planes, writes fp32 + the output's planes); conv1 runs as a
    // 4x4 stride-1 convolution over the space-to-depth input
    if (o.conv == 0 && !e->s2d_ready) {
      const View in = e->view(o.in, false);
      __half* s2d = (__half*)(e->ws + e->s2d_off);
      if (int rc = launch_nhwc_to_s2d(in, n, s2d, (long long)e->s2d_plane, e->Cs, s)) return rc;
    }
    tag_next(0, e->conv_flops(o, n), o.id.c_str());
    return umma_conv_launch(e->umma_ctx, o.umma, s, false, n);
  }
  if (o.kind == OP_BN1) {
    if (!e->bn1_gamma || !e->bn1_beta) { set_thread_error("bn1_train engine: call ssnb_set_bn1 first"); return SSNB_ESTATE; }
    return launch_bn_train_fwd(e->view(o.in, false), e->view(o.out, false), e->exact_tc() ? e->planes(o.out, false) : View(), e->F, e->bn1_gamma,
                               e->bn1_beta, e->bn1_eps, e->bn1_momentum, e->bn1_rmean, e->bn1_rvar, (float*)(e->ws + e->bn_stat_off),
                               (float*)(e->ws + e->bn_partial_off), 1200, s);
  }
  if (o.kind == OP_MAXPOOL || o.kind == OP_AVGPOOL) return e->pool_fwd(o, n, s);     // EXACT_TC: and the output's operand planes
  if (o.kind == OP_GPOOL) {
    if (!feat) return e->fail(SSNB_EINVAL, "global_pool needs the feat output pointer");
    return e->gpool_fwd(o, n, feat, s);
  }
  // SIMT convolution; the raw conv1 of a bn1_train engine has no ReLU
  if (int rc = e->simt_conv_fwd(o, o.raw ? 0 : 1, n, s)) return rc;
  if (!e->exact_tc() || !e->bufs[e->vals[o.out].buf].plane) return 0;     // EXACT_TC: the output's operand planes
  return launch_split_view(e->view(o.out), n, 1.0f, e->planes(o.out), nullptr, s);
}

// SIMT convolution backward (EXACT_FP32, and layers or passes without a tensor-core plan), reading the masked fp32 / fp16
// dz = d(out): weight gradient into the layer's split-K partials + finalize; data gradient into d(in)
static int simt_wgrad(ssnb_engine* e, const Op& o, cudaStream_t s) {
  const Conv& c = e->convs[o.conv];
  const View x = e->view(o.in, false), dz = e->view(o.out, true);
  float* partial = (float*)(e->ws + o.partial_off);
  WgradArgs w;
  w.dz = dz.base; w.OH = dz.H; w.OW = dz.W; w.Cout = dz.C; w.dz_pitch = dz.pitch; w.dz_coff = dz.coff;
  w.x = x.base; w.IH = x.H; w.IW = x.W; w.Cin = x.C; w.x_pitch = x.pitch; w.x_coff = x.coff;
  w.partial = partial; w.F = e->F; w.k = c.kh; w.stride = c.stride; w.pad = c.ph;
  w.rows_per_split = o.wrows; w.splits = o.wsplits;
  tag_next(2, e->conv_flops(o, e->F), o.id.c_str());
  if (int rc = DISPATCH(e, launch_wgrad<float>(w, s), launch_wgrad<__half>(w, s))) return rc;
  const float out_scale = e->fast() ? 1.0f / e->cfg.grad_scale : 1.0f;      // FAST stores gradients times the loss scale
  return launch_wgrad_finalize(partial, o.wsplits, c.kh * c.kw, c.cout, c.cin, (const float*)(e->ws + e->packed[o.conv].scale), out_scale,
                               e->dw[o.conv], e->grad_accumulate, s, nullptr, nullptr, nullptr, e->grad_unscale_dev());
}
static int simt_dgrad(ssnb_engine* e, const Op& o, cudaStream_t s) {
  const Conv& c = e->convs[o.conv];
  const View dz = e->view(o.out, true), dx = e->view(o.in, true);
  ConvArgs a;
  a.src = dz.base; a.SH = dz.H; a.SW = dz.W; a.Csrc = dz.C; a.src_pitch = dz.pitch; a.src_coff = dz.coff;
  a.dst = dx.base; a.DH = dx.H; a.DW = dx.W; a.Cdst = dx.C; a.dst_pitch = dx.pitch; a.dst_coff = dx.coff;
  a.wgt = e->ws + e->packed[o.conv].wd; a.bias = nullptr;
  a.F = e->F; a.kh = a.kw = c.kh; a.stride = c.stride; a.pad_h = a.pad_w = c.ph; a.relu = 0; a.accumulate = o.grad_accumulate; a.dgrad = 1;
  tag_next(1, e->conv_flops(o, e->F), o.id.c_str());
  return DISPATCH(e, launch_conv<float>(a, s), launch_conv<__half>(a, s));
}

static int run_bwd(ssnb_engine* e, const Op& o, const float* dfeat, cudaStream_t s, bool skip_dgrad = false, bool full = false) {
  const int F = e->F;
  const float gs = e->fast() ? e->cfg.grad_scale : 1.0f;
  int rc = 0;
  tag_next(3, 0.0);
  if (o.kind == OP_GPOOL) {
    if (!dfeat) return e->fail(SSNB_EINVAL, "global_pool backward needs dfeat");
    const View din = e->view(o.in, true);
    const void* ym = (full && e->fold_pools && o.dgrad_masks) ? e->view(o.in, false).base : nullptr;
    const float* gsd = e->grad_scale_dev();
    return DISPATCH(e, launch_gpool_bwd<float>(dfeat, gs, gsd, din, F, ym, s), launch_gpool_bwd<__half>(dfeat, gs, gsd, din, F, ym, s));
  }
  if (o.kind == OP_BN1) {
    return launch_bn_train_bwd(e->view(o.in, false), e->view(o.out, true), e->view(o.out, false), e->view(o.in, true),
                               e->exact_tc() ? e->planes(o.in, true) : View(), e->cfg.grad_scale, e->tc_flag, F, e->bn1_gamma, (float*)(e->ws + e->bn_stat_off),
                               (float*)(e->ws + e->bn_partial_off), 1200, e->bn1_dgamma, e->bn1_dbeta, e->grad_unscale_dev(), e->grad_accumulate, s);
  }
  if (o.kind == OP_MAXPOOL) {
    if (full && e->fold_pools && o.folded_into_conv) return 0;      // gathered by the producer conv's mask+bias pass (tensor-core modes)
    const View din = e->view(o.in, true), dout = e->view(o.out, true);
    const uint8_t* am = (const uint8_t*)(e->ws + o.argmax_off);
    return DISPATCH(e, launch_maxpool_bwd_vec<float>(din, dout, F, o.k, o.stride, o.pad, am, o.grad_accumulate, s),
                    launch_maxpool_bwd_vec<__half>(din, dout, F, o.k, o.stride, o.pad, am, o.grad_accumulate, s));
  }
  if (o.kind == OP_AVGPOOL) {
    const View din = e->view(o.in, true), dout = e->view(o.out, true);
    return DISPATCH(e, launch_avgpool3_vec<float>(dout, din, View(), F, o.grad_accumulate, s),
                    launch_avgpool3_vec<__half>(dout, din, View(), F, o.grad_accumulate, s));
  }
  // convolution: dz = dy * (y > 0); db, dW from dz; dx = dgrad(dz)
  const Conv& c = e->convs[o.conv];
  const View x = e->view(o.in, false), y = e->view(o.out, false), dy = e->view(o.out, true);
  const float* scale = (const float*)(e->ws + e->packed[o.conv].scale);
  float* bpartial = (float*)(e->ws + e->bpartial_off);
  float* dbp = (e->db.size() && e->db[o.conv]) ? e->db[o.conv] : nullptr;
  const bool want_w = e->dw.size() && e->dw[o.conv];
  const bool want_x = e->vals[o.in].name != "data" && !skip_dgrad;
  // the tensor-core products read dz times the loss scale (FAST: the fp16 storage, EXACT_TC: the planes); EXACT has no
  // tensor-core plans
  const float gst = e->cfg.grad_scale;
  const float* us = e->grad_unscale_dev();
  const bool tc_w = want_w && o.umma_wgrad.enabled, tc_x = want_x && o.umma_dgrad.enabled;
  const bool pre = full && e->fold_pools && o.dy_premasked;      // the last writer of dy masked it (EXACT_TC: and wrote its planes)
  const bool bias_w = pre && o.bias_in_wgrad && dbp && tc_w;     // ... and the bias column sums ride on the weight-gradient MMAs
  // the only consumer is a max pool whose backward gather is folded into this mask pass (the pooled input's dy is never materialised)
  const Op* pool = (full && e->fold_pools && o.pool_consumer >= 0) ? &e->ops[o.pool_consumer] : nullptr;
  const int max_ctas = (1024 * 512 - 64) / y.C;
  // 1. one pass over dy: ReLU mask + bias-gradient column sums.  FAST masks the fp16 dy in place.  EXACT_TC reads the fp32 dy,
  //    writes the hi/lo planes of dz * grad_scale and writes the masked fp32 dz back only when a SIMT kernel will read it;
  //    EXACT writes no planes and masks the fp32 dy in place for its SIMT kernels.
  const View dpool = pool ? e->view(pool->out, true) : View();
  const uint8_t* pam = pool ? (const uint8_t*)(e->ws + pool->argmax_off) : nullptr;
  if (e->fast()) {
    if (pool) rc = launch_pool_mask_bias_vec<__half>(dy, y, dpool, View(), 1.0f, 1, nullptr, F, pool->k, pool->stride, pool->pad, pam,
                                                    scale, 1.0f / gst, us, bpartial, max_ctas, dbp, e->grad_accumulate, s);
    else if (!bias_w) rc = launch_mask_bias_vec<__half>(dy, pre ? View() : y, View(), 1.0f, 1, nullptr, F, scale, 1.0f / gst, us, bpartial, max_ctas, dbp,
                                                       e->grad_accumulate, s);
  } else {
    const bool need_f32 = (want_w && !tc_w) || (want_x && !tc_x);
    const View pl = (tc_w || tc_x) ? e->planes(o.out, true) : View();
    if (o.raw) {         // the training-mode BatchNorm behind this convolution produced dz (and its planes): only the bias sums are left
      if (dbp) rc = launch_mask_bias_vec<float>(dy, View(), View(), gst, 0, nullptr, F, scale, 1.0f, us, bpartial, max_ctas, dbp, e->grad_accumulate, s);
    } else if (pre) {    // bias sums of the already masked fp32 dz only: no planes, nothing written back
      if (!bias_w && dbp) rc = launch_mask_bias_vec<float>(dy, y, View(), gst, 0, nullptr, F, scale, 1.0f, us, bpartial, max_ctas, dbp, e->grad_accumulate, s);
    } else if (pool) {
      rc = launch_pool_mask_bias_vec<float>(dy, y, dpool, pl, gst, need_f32 ? 1 : 0, e->tc_flag, F, pool->k, pool->stride, pool->pad, pam,
                                            scale, 1.0f, us, bpartial, max_ctas, dbp, e->grad_accumulate, s);
    } else {
      rc = launch_mask_bias_vec<float>(dy, y, pl, gst, (need_f32 || !full) ? 1 : 0, e->tc_flag, F, scale, 1.0f, us, bpartial, max_ctas, dbp,
                                       e->grad_accumulate, s);
    }
  }
  if (rc) return rc;
  // 2. a stride-2 data gradient reads dz zero-upsampled to the input resolution, every operand plane
  if (tc_x && c.stride == 2 && o.conv != 0) {
    View dz = e->operand(o.out, true);
    for (int p = 0; p < e->nplanes(); ++p, dz.base = (char*)dz.base + dz.lo_off)
      if ((rc = launch_upsample2_zero(dz, (__half*)(e->ws + e->up_off + p * e->up_plane), x.H, x.W, F, s))) return rc;
  }
  // 3. weight gradient.  The wgmma partials of a whole backward are finalised in one batch at its end; conv1's space-to-depth
  //    partials and those of a single op (ssnb_run_op) right away.
  if (tc_w) {
    float* partial = (float*)(e->ws + o.partial_off);
    float* bp = bias_w ? (float*)(e->ws + o.bias_partial_off) : nullptr;
    tag_next(2, e->conv_flops(o, F), o.id.c_str());
    if ((rc = umma_wgrad_launch(e->umma_ctx, o.umma_wgrad, s, bp))) return rc;
    if (full && o.conv != 0) e->pending_finalize.push_back((int)(&o - e->ops.data()));
    else if (o.conv == 0) rc = launch_wgrad_finalize_s2d(partial, o.umma_wgrad.p.splits, c.cout, c.cin, e->Cs, scale, 1.0f / gst, us, e->dw[o.conv],
                                                         e->grad_accumulate, s);
    else rc = launch_wgrad_finalize(partial, o.umma_wgrad.p.splits, c.kh * c.kw, c.cout, c.cin, scale, 1.0f / gst, e->dw[o.conv], e->grad_accumulate, s,
                                    nullptr, nullptr, e->tc_flag, us);
    if (rc) return rc;
  } else if (want_w && (rc = simt_wgrad(e, o, s))) return rc;
  // 4. data gradient; as the last writer of d(in) the wgmma epilogue applies in's ReLU mask
  if (tc_x) {
    tag_next(1, e->conv_flops(o, F), o.id.c_str());
    return umma_conv_launch(e->umma_ctx, o.umma_dgrad, s, full && e->fold_pools && o.dgrad_masks);
  }
  return want_x ? simt_dgrad(e, o, s) : 0;
}

int engine_tail_view(ssnb_handle h, View* v, int* F, int* fp16) {
  if (!h->ws || !h->weights_ready) return h->fail(SSNB_ESTATE, "workspace/weights not set");
  *v = h->view(h->ops.back().in, false);
  *F = h->F; *fp16 = h->fast() ? 1 : 0;
  return 0;
}

}  // namespace ssnb

// ---- C ABI -----------------------------------------------------------------------------------------
extern "C" {

const char* ssnb_version(void) { return "libssn_b200 0.3 (sm_90a)"; }

const char* ssnb_last_error(ssnb_handle h) { return h ? h->error.c_str() : ssnb::thread_error().c_str(); }

int ssnb_num_convs(void) { return 69; }

int ssnb_conv_info(int idx, int in_channels, char* name, int name_cap, int* cin, int* cout, int* k, int* stride, int* pad) {
  std::vector<Conv> t = conv_table(in_channels);
  if (idx < 0 || idx >= (int)t.size()) { set_thread_error("ssnb_conv_info: index out of range"); return SSNB_EINVAL; }
  if (name && name_cap > 0) { snprintf(name, name_cap, "%s", t[idx].id.c_str()); }
  if (cin) *cin = t[idx].cin; if (cout) *cout = t[idx].cout; if (k) *k = t[idx].kh;
  if (stride) *stride = t[idx].stride; if (pad) *pad = t[idx].ph;
  return SSNB_OK;
}

int ssnb_create(const ssnb_config* cfg, ssnb_handle* out) {
  if (!cfg || !out) { set_thread_error("ssnb_create: null argument"); return SSNB_EINVAL; }
  if (cfg->frames <= 0 || cfg->in_channels <= 0 || cfg->in_channels > 64) { set_thread_error("ssnb_create: bad frames/in_channels"); return SSNB_EINVAL; }
  if (cfg->precision != SSNB_EXACT_FP32 && cfg->precision != SSNB_FAST_FP16 && cfg->precision != SSNB_EXACT_TC) { set_thread_error("ssnb_create: unknown precision"); return SSNB_EINVAL; }
  ssnb_engine* e = new ssnb_engine();
  e->cfg = *cfg;
  if (!(e->cfg.grad_scale > 0.f)) e->cfg.grad_scale = 1.0f;
  e->F = cfg->frames;
  e->precision = cfg->precision;
  e->bn1_train = cfg->bn1_train != 0;
  if (e->bn1_train && e->fast()) { delete e; set_thread_error("ssnb_create: bn1_train (bn_mode='partial') needs EXACT_FP32 or EXACT_TC"); return SSNB_ENOSUPPORT; }
  e->esz = e->fast() ? 2 : 4;
  build_graph(e);
  if ((int)e->convs.size() != 69) { delete e; set_thread_error("internal: conv table size"); return SSNB_ESTATE; }
  umma_context_init(e->umma_ctx);
  plan(e);
  e->launches0 = g_launches.load();
  *out = e;
  return SSNB_OK;
}

int ssnb_destroy(ssnb_handle h) {
  if (!h) return SSNB_OK;
  umma_context_destroy(h->umma_ctx);
  delete h;
  return SSNB_OK;
}

size_t ssnb_workspace_bytes(ssnb_handle h) { return h ? h->ws_bytes : 0; }

int ssnb_set_workspace(ssnb_handle h, void* dev_ptr, size_t bytes) {
  if (!h) return SSNB_EINVAL;
  if (!dev_ptr || bytes < h->ws_bytes) return h->fail(SSNB_EINVAL, "workspace too small");
  if (((uintptr_t)dev_ptr) % 1024) return h->fail(SSNB_EINVAL, "workspace must be 1024-byte aligned");
  h->ws = (char*)dev_ptr;
  h->weights_ready = false;
  if (cudaMemset(h->ws + h->bpartial_off, 0, 256) != cudaSuccess) { cudaGetLastError(); /* no device (CPU-only planning) */ }
  h->tc_flag = (int*)(h->ws + h->tc_flag_off);
  if (cudaMemset(h->tc_flag, 0, 256) != cudaSuccess) cudaGetLastError();
  h->gscale = (float*)(h->ws + h->tc_flag_off + 16);
  const float one[2] = {1.0f, 1.0f};          // k = 0 until the first backward (ssnb_run_op / ssnb_value_write before any)
  if (cudaMemcpy(h->gscale, one, sizeof one, cudaMemcpyHostToDevice) != cudaSuccess) cudaGetLastError();
  // Bind the tensor-core plans (tensor maps need final addresses).  The diagnostic switches are read here, once per engine:
  // SSNB_DISABLE_UMMA=1 keeps every convolution on the SIMT kernels (FAST: fp16; EXACT_TC: fp32, the EXACT_FP32 arithmetic
  // that tools/umma_diag.py diffs the tensor-core launches against), SSNB_DISABLE_UMMA_WGRAD=1 only the weight gradients, and
  // SSNB_DISABLE_FUSION=1 turns off sibling fusion, last-writer masking and the max-pool backward folding.
  const bool training = h->cfg.training != 0;
  const bool use_tc = h->tensor_cores() && !env_on("SSNB_DISABLE_UMMA");
  const bool use_wgrad = use_tc && training && !env_on("SSNB_DISABLE_UMMA_WGRAD");
  const bool fuse = !env_on("SSNB_DISABLE_FUSION");
  const float gs = h->cfg.grad_scale;
  for (Op& o : h->ops) {
    o.umma.enabled = o.umma_dgrad.enabled = o.umma_wgrad.enabled = false;
    o.fuse_role = 0; o.fuse_block = -1; o.dgrad_masks = o.dy_premasked = o.bias_in_wgrad = false;
  }
  for (FusedBlock& fb : h->fused) fb.enabled = false;
  // FAST folds the max-pool backward into its producer on the SIMT kernels as well; EXACT_TC only in the tensor-core training schedule
  h->fold_pools = fuse && (h->fast() || (use_tc && training));
  // Where EXACT_TC runs a convolution.  umma_conv_kernel's split-operand epilogue covers the plans with UmmaConvParams::tc_ok:
  // stride-1 tiles of 1, 4 or 9 taps over images at least 7 pixels wide with 32-byte aligned outputs.  conv1's forward, the
  // per-layer data gradients and both fused sibling launches run on the tensor cores only when tc_ok holds, and otherwise on
  // the fp32 SIMT kernels.  The per-layer forward is not gated: the stride-2 3x3 forwards (tc_ok = 0, element-stride A
  // boxes) run on umma_conv_kernel as well.  Stride-2 data gradients are stride-1 convolutions of the zero-upsampled dz and
  // pass tc_ok.  In the default schedule every gated plan passes, so no convolution of EXACT_TC runs on the SIMT kernels.
  // FAST runs every plan it binds.
  auto tc_gate = [&](UmmaConvPlan& p) {
    if (h->exact_tc() && !p.p.tc_ok) p.enabled = false;
    return p.enabled;
  };
  for (Op& o : h->ops) {
    if (o.kind != OP_CONV || !use_tc) continue;
    const Conv& c = h->convs[o.conv];
    const PackedConv& pk = h->packed[o.conv];
    UmmaTcOpts tf, tg;
    int rc = 0;
    if (o.conv == 0) {
      // conv1 7x7/2: four vertical taps over the packed space-to-depth input (r = 2*dr + a - 1, s = 2*ds + b - 1)
      const int Ck = 4 * h->Cs;
      View xs; xs.base = h->ws + h->s2d_off; xs.H = 112; xs.W = 112; xs.C = Ck; xs.pitch = Ck; xs.coff = 0; xs.lo_off = (long long)h->s2d_plane;
      int dy[4], dx[4];
      for (int t = 0; t < 4; ++t) { dy[t] = t - 2; dx[t] = 0; }
      rc = umma_conv_bind_taps(h->umma_ctx, o.umma, xs, h->operand(o.out, false), h->F, Ck, c.cout, 4, dy, dx, (const __half*)(h->ws + h->s2d_w_off),
                               (const float*)(h->ws + pk.bias), o.raw ? 0 : 1, h->tc_opts(tf, h->s2d_w_plane, h->view(o.out, false).base, 1.0f, pk.wmax));
      if (rc) return h->fail(rc, "conv1 bind: " + ssnb::thread_error());
      tc_gate(o.umma);
      if (use_wgrad && (rc = umma_wgrad_bind_taps(h->umma_ctx, o.umma_wgrad, h->operand(o.out, true), xs, h->F, Ck, c.cout, 4, dy, dx,
                                                  (float*)(h->ws + o.partial_off), h->conv1_tsplits)))
        return h->fail(rc, "conv1 wgrad bind: " + ssnb::thread_error());
      continue;
    }
    if (c.cin % 8 != 0 || c.kh * c.kw > UMMA_MAX_TAPS) continue;
    rc = umma_conv_bind_fwd(h->umma_ctx, o.umma, h->operand(o.in, false), h->operand(o.out, false), h->F, c.cin, c.cout, c.kh, c.ph,
                            c.stride, h->w_fwd(pk), (const float*)(h->ws + pk.bias), h->tc_opts(tf, pk.wplane, h->view(o.out, false).base, 1.0f, pk.wmax));
    if (rc) return h->fail(rc, "bind_fwd(" + c.id + "): " + ssnb::thread_error());
    if (!training) continue;
    // data gradient: stride-2 layers read the zero-upsampled dz at input resolution.  EXACT_TC writes the fp32 d(in) only:
    // its consumer masks and splits it.
    const View in = h->view(o.in, false);
    View dz = h->operand(o.out, true);
    if (c.stride == 2) { dz.base = h->ws + h->up_off; dz.H = in.H; dz.W = in.W; dz.C = c.cout; dz.pitch = c.cout; dz.coff = 0; dz.lo_off = (long long)h->up_plane; }
    View dx = h->view(o.in, true);
    const UmmaTcOpts* og = h->tc_opts(tg, pk.wplane, dx.base, 1.0f / gs, pk.wmax);
    if (og) dx.base = nullptr;
    rc = umma_conv_bind_dgrad(h->umma_ctx, o.umma_dgrad, dz, dx, h->F, c.cin, c.cout, c.kh, c.ph, h->w_dgrad(pk), o.grad_accumulate, og);
    if (rc) return h->fail(rc, "bind_dgrad(" + c.id + "): " + ssnb::thread_error());
    tc_gate(o.umma_dgrad);
    // weight gradient: stride-2 layers read dz at its own (output) resolution, the x boxes step over the input with element stride 2
    if (use_wgrad && (rc = umma_wgrad_bind(h->umma_ctx, o.umma_wgrad, h->operand(o.out, true), h->operand(o.in, false), h->F, c.cin, c.cout,
                                           c.kh, c.ph, (float*)(h->ws + o.partial_off), o.tsplits, c.stride)))
      return h->fail(rc, "wgrad_bind(" + c.id + "): " + ssnb::thread_error());
  }
  // horizontal fusion of the sibling 1x1 convolutions of each inception block: ONE forward launch (stacked weights; the first
  // c1 columns land in the concat buffer, the rest in the shared reduce buffer) and ONE data-gradient launch (K-concatenated
  // dz from two sources) instead of three read-modify-write passes over the block input's gradient
  for (size_t bi = 0; bi < h->fused.size() && use_tc && fuse; ++bi) {
    FusedBlock& fb = h->fused[bi];
    const Op& o3 = h->ops[fb.op_r3]; const Op& od = h->ops[fb.op_rd];
    if (!o3.umma.enabled || !od.umma.enabled) continue;
    const int nr = fb.c3r + fb.cdr;                  // both reduce outputs: adjacent slices of one buffer
    const View x = h->operand(o3.in, false);
    View red = h->operand(o3.out, false); red.C = nr;
    UmmaTcOpts tf, tg;
    int rc;
    if (fb.op1 >= 0) {
      const int v1 = h->ops[fb.op1].out;
      const UmmaTcOpts* of = h->tc_opts(tf, fb.w_fwd_plane, h->view(v1, false).base, 1.0f, fb.wmax);
      tf.out32_2 = (float*)h->view(o3.out, false).base;
      rc = umma_conv_bind_fused_fwd(h->umma_ctx, fb.fwd, x, h->operand(v1, false), red, h->F, fb.cx, fb.c1, nr, (const __half*)(h->ws + fb.w_fwd),
                                    (const float*)(h->ws + fb.bias), of);
    } else {
      rc = umma_conv_bind_fwd(h->umma_ctx, fb.fwd, x, red, h->F, fb.cx, nr, 1, 0, 1, (const __half*)(h->ws + fb.w_fwd), (const float*)(h->ws + fb.bias),
                              h->tc_opts(tf, fb.w_fwd_plane, h->view(o3.out, false).base, 1.0f, fb.wmax));
    }
    if (rc) return h->fail(rc, "fused fwd bind(" + o3.id + "): " + ssnb::thread_error());
    if (!tc_gate(fb.fwd)) continue;
    if (training) {
      View dred = h->operand(o3.out, true); dred.C = nr;
      const View d1 = fb.op1 >= 0 ? h->operand(h->ops[fb.op1].out, true) : dred;
      View dx = h->view(o3.in, true);
      const UmmaTcOpts* og = h->tc_opts(tg, fb.w_dg_plane, dx.base, 1.0f / gs, fb.wmax);
      if (og) dx.base = nullptr;
      rc = umma_conv_bind_fused_dgrad(h->umma_ctx, fb.dgrad, d1, dred, dx, h->F, fb.cx, fb.c1, nr, (const __half*)(h->ws + fb.w_dg), od.grad_accumulate, og);
      if (rc) return h->fail(rc, "fused dgrad bind(" + o3.id + "): " + ssnb::thread_error());
      if (!tc_gate(fb.dgrad)) continue;
      // EXACT_TC: zero the K padding of the concatenated data-gradient weights once (both planes); split_all_kernel never
      // writes it.  FAST assembles these weights by copies and zeroes them on every pack.
      if (h->exact_tc() && cudaMemset(h->ws + fb.w_dg, 0, 2 * fb.w_dg_plane) != cudaSuccess) cudaGetLastError();
    }
    fb.enabled = true;
    const int leader = fb.op1 >= 0 ? fb.op1 : fb.op_r3;
    for (int j : {fb.op1, fb.op_r3, fb.op_rd})
      if (j >= 0) { h->ops[j].fuse_block = (int)bi; h->ops[j].fuse_role = (j == leader) ? 1 : 2; }
  }
  // ReLU-mask fusion: the consumer with the smallest forward index is the LAST writer of a value's gradient in the reverse
  // schedule (sibling followers are folded into their leader).  When that writer is a tensor-core data gradient, its epilogue
  // applies dz = dy * (y > 0) (EXACT_TC: and emits the gradient's operand planes dz * grad_scale), so the producing
  // convolutions run neither a mask pass nor a split pass, and their bias gradients ride on the weight-gradient MMAs (ones operand).
  if (use_tc && training && fuse) {
    std::vector<int> first_consumer(h->vals.size(), -1);
    for (int i = 0; i < (int)h->ops.size(); ++i)
      if (first_consumer[h->ops[i].in] < 0) first_consumer[h->ops[i].in] = i;
    for (size_t v = 0; v < h->vals.size(); ++v) {
      const int fc = first_consumer[v];
      if (fc < 0 || h->vals[v].name == "data") continue;
      if (h->exact_tc() && !h->bufs[h->vals[v].buf].plane) continue;      // no operand planes to emit
      bool conv_made = false;                    // only buffers that hold convolution outputs have a ReLU to differentiate
      for (const Op& q : h->ops) conv_made = conv_made || (q.kind == OP_CONV && h->vals[q.out].buf == h->vals[v].buf);
      if (!conv_made) continue;
      Op& c = h->ops[fc];
      UmmaConvPlan* dg = nullptr;
      if (c.kind == OP_CONV && c.fuse_role == 1 && h->fused[c.fuse_block].enabled) dg = &h->fused[c.fuse_block].dgrad;
      else if (c.kind == OP_CONV && c.fuse_role == 0 && c.umma_dgrad.enabled) dg = &c.umma_dgrad;
      if (dg) {
        c.dgrad_masks = true;
        if (h->exact_tc()) {
          if (int rc = umma_conv_set_mask_tc(h->umma_ctx, *dg, h->view((int)v, false), h->planes((int)v, true), gs, h->tc_flag))
            return h->fail(rc, "mask bind(" + h->vals[v].name + "): " + ssnb::thread_error());
        } else {
          umma_conv_set_mask(*dg, h->view((int)v, false));
        }
      } else if (c.kind == OP_GPOOL && h->fast()) {
        c.dgrad_masks = true;       // FAST only: gpool_bwd<float> writes no operand planes, so EXACT_TC keeps the producers' split pass
      }
    }
    for (Op& o : h->ops) {
      if (o.kind != OP_CONV) continue;
      int w = o.out;
      if (first_consumer[w] < 0) {               // a slice of a concat buffer: gradients are written through the whole-buffer value
        const Value& ov = h->vals[o.out];
        for (size_t v = 0; v < h->vals.size(); ++v)
          if (h->vals[v].buf == ov.buf && h->vals[v].coff == 0 && h->vals[v].C == h->bufs[ov.buf].C && first_consumer[v] >= 0) { w = (int)v; break; }
      }
      if (first_consumer[w] >= 0 && h->ops[first_consumer[w]].dgrad_masks) o.dy_premasked = true;
      o.bias_in_wgrad = o.dy_premasked && o.conv != 0 && o.umma_wgrad.enabled;
    }
  }
  return SSNB_OK;
}

int ssnb_pack_weights(ssnb_handle h, const float* const* w, const float* const* b, const float* const* gamma,
                      const float* const* beta, const float* const* mean, const float* const* var, void* stream) {
  if (!h || !h->ws) return h ? h->fail(SSNB_ESTATE, "set_workspace first") : SSNB_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  // the members of each fused sibling block: their rows in its stacked forward weights, their columns in its K-concatenated
  // data-gradient weights
  struct Member { int block = -1, row = 0, col = 0; };
  std::vector<Member> member(h->convs.size());
  for (size_t bi = 0; bi < h->fused.size(); ++bi) {
    const FusedBlock& fb = h->fused[bi];
    if (!fb.enabled) continue;
    const int k1p = (fb.c1 + 63) / 64 * 64;
    int row = 0, col = 0;
    for (int j : {fb.op1, fb.op_r3, fb.op_rd}) {
      if (j < 0) continue;
      const int ci = h->ops[j].conv;
      member[ci].block = (int)bi; member[ci].row = row; member[ci].col = col;
      row += h->convs[ci].cout;
      col += (j == fb.op1) ? k1p : h->convs[ci].cout;
    }
  }
  // bn1_train: conv1 is not folded.  EXACT_TC: the layers of a fused sibling block share one absmax slot, and the fold and
  // split launches also write the block's fused operands
  auto adjust = [&](size_t i, PackEntry& q, SplitEntry* e) {
    q.nofold = (h->bn1_train && i == 0) ? 1 : 0;
    const Member& mb = member[i];
    if (!h->exact_tc() || mb.block < 0) return;
    const FusedBlock& fb = h->fused[mb.block];
    q.bias_b = (float*)(h->ws + fb.bias) + mb.row;
    const int kf = (fb.c1 + 63) / 64 * 64 + fb.c3r + fb.cdr;
    e->wd16_b = (__half*)(h->ws + fb.w_fwd) + (size_t)mb.row * fb.cx;      // stacked forward rows [n][cx]
    e->wf16_b = (__half*)(h->ws + fb.w_dg) + mb.col;                         // column block of [cx][kf]
    e->b_pitch = kf;
    // both fused buffers are written through ONE plane distance per entry: the kernel applies it to wd16_b and wf16_b alike,
    // so the two buffers are planned with equal plane sizes (max of the two)
    e->b_plane_bytes = (long long)std::max(fb.w_fwd_plane, fb.w_dg_plane);
  };
  if (int rc = h->pack_weights(w, b, gamma, beta, mean, var, h->convs[0].cin, adjust, "pack_weights", s)) return h->fail(rc, ssnb::thread_error());
  if (h->ops.size() && h->ops[0].umma.enabled) {      // conv1's space-to-depth weights, every operand plane
    const PackedConv& p = h->packed[0];
    for (int pl = 0; pl < h->nplanes(); ++pl) {
      int rc = launch_pack_conv1_s2d((const __half*)((const char*)h->w_fwd(p) + pl * p.wplane), h->convs[0].cout, h->convs[0].cin, h->Cs,
                                     (__half*)(h->ws + h->s2d_w_off + pl * h->s2d_w_plane), s);
      if (rc) return h->fail(rc, "pack conv1 s2d: " + ssnb::thread_error());
    }
  }
  for (FusedBlock& fb : h->fused) {
    if (!fb.enabled || !h->fast()) continue;          // EXACT_TC: split_all_kernel wrote the fused operands directly
    // forward: rows of wd ([co][ci]) stacked; bias stacked.  data gradient: wf ([ci][co]) concatenated along K,
    // the 1x1 part padded to a multiple of 64 so each K chunk has a single activation source.
    const int k1p = (fb.c1 + 63) / 64 * 64, kf = k1p + fb.c3r + fb.cdr;
    __half* wfwd = (__half*)(h->ws + fb.w_fwd); float* bias = (float*)(h->ws + fb.bias); __half* wdg = (__half*)(h->ws + fb.w_dg);
    if (cudaMemsetAsync(wdg, 0, (size_t)fb.cx * kf * 2, s) != cudaSuccess) return h->fail(SSNB_ECUDA, "fused pack: memset");
    int row = 0, col = 0;
    for (int j : {fb.op1, fb.op_r3, fb.op_rd}) {
      if (j < 0) { continue; }
      const int ci = h->ops[j].conv, co = h->convs[ci].cout;
      cudaError_t e1 = cudaMemcpyAsync(wfwd + (size_t)row * fb.cx, h->ws + h->packed[ci].wd, (size_t)co * fb.cx * 2, cudaMemcpyDeviceToDevice, s);
      cudaError_t e2 = cudaMemcpyAsync(bias + row, h->ws + h->packed[ci].bias, (size_t)co * 4, cudaMemcpyDeviceToDevice, s);
      cudaError_t e3 = cudaMemcpy2DAsync(wdg + col, (size_t)kf * 2, h->ws + h->packed[ci].wf, (size_t)co * 2, (size_t)co * 2, fb.cx,
                                         cudaMemcpyDeviceToDevice, s);
      if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) return h->fail(SSNB_ECUDA, "fused pack: copy failed");
      row += co;
      col += (j == fb.op1) ? k1p : co;
    }
  }
  h->weights_ready = true;
  return SSNB_OK;
}

int ssnb_set_bn1(ssnb_handle h, const float* gamma, const float* beta, float* running_mean, float* running_var, float* dgamma, float* dbeta,
                 float momentum, float eps) {
  if (!h) return SSNB_EINVAL;
  if (!h->bn1_train) return h->fail(SSNB_ESTATE, "engine created without bn1_train");
  if (!gamma || !beta) return h->fail(SSNB_EINVAL, "set_bn1: gamma / beta are required");
  h->bn1_gamma = gamma; h->bn1_beta = beta; h->bn1_rmean = running_mean; h->bn1_rvar = running_var; h->bn1_dgamma = dgamma; h->bn1_dbeta = dbeta;
  h->bn1_momentum = momentum; h->bn1_eps = eps;
  return SSNB_OK;
}

// the forward of frames [0, n) after the caller's checks
static int backbone_fwd(ssnb_handle h, const float* input_nchw, int n, float* feat, cudaStream_t s) {
  const View d = h->view(h->val_by_name["data"], false);
  int rc;
  h->s2d_ready = h->tensor_cores() && h->ops[0].umma.enabled;
  if (h->s2d_ready) rc = launch_nchw_to_s2d(input_nchw, n, d.C, d.H, d.W, (__half*)(h->ws + h->s2d_off), (long long)h->s2d_plane, h->Cs, s);
  else rc = h->value_write(h->val_by_name["data"], false, input_nchw, 1.0f, n, s);
  if (rc) { h->s2d_ready = false; return h->fail(rc, "input layout: " + ssnb::thread_error()); }
  for (size_t i = 0; i < h->ops.size(); ++i) {
    const Op& o = h->ops[i];
    if (o.fuse_role == 2) continue;                       // computed by its block's fused launch
    const bool prof = profiled_op("SSNB_PROFILE_FWD_OPS", o.id);
    if (prof) cudaProfilerStart();
    int r;
    if (o.fuse_role == 1) {
      const FusedBlock& fb = h->fused[o.fuse_block];
      double fl = 0.0;
      for (int j : {fb.op1, fb.op_r3, fb.op_rd}) if (j >= 0) fl += h->conv_flops(h->ops[j], n);
      tag_next(0, fl, fused_name(h, fb));
      r = umma_conv_launch(h->umma_ctx, fb.fwd, s, false, n);
    } else r = run_fwd(h, o, feat, n, s);
    if (prof) cudaProfilerStop();
    if (r) { h->s2d_ready = false; return h->fail(r, "fwd " + o.id + ": " + ssnb::thread_error()); }
  }
  h->s2d_ready = false;
  return SSNB_OK;
}

int ssnb_backbone_fwd(ssnb_handle h, const float* input_nchw, float* feat, void* stream) {
  if (!h || !input_nchw || !feat) return h ? h->fail(SSNB_EINVAL, "null argument") : SSNB_EINVAL;
  if (!h->ws || !h->weights_ready) return h->fail(SSNB_ESTATE, "workspace/weights not set");
  return backbone_fwd(h, input_nchw, h->F, feat, (cudaStream_t)stream);
}

int ssnb_backbone_fwd_frames(ssnb_handle h, const float* input_nchw, int frames, float* feat, void* stream) {
  if (!h || !input_nchw || !feat) return h ? h->fail(SSNB_EINVAL, "null argument") : SSNB_EINVAL;
  if (frames < 1 || frames > h->F) return h->fail(SSNB_EINVAL, "backbone_fwd_frames: frames must be in 1 .. " + std::to_string(h->F));
  // a training engine keeps the activations of all F frames for its backward; bn_mode='partial' takes batch statistics over F
  if (h->cfg.training) return h->fail(SSNB_ESTATE, "backbone_fwd_frames: runs forward-only engines (training = 0)");
  if (h->bn1_train) return h->fail(SSNB_ENOSUPPORT, "backbone_fwd_frames: bn1_train engines run their planned frame count only");
  if (!h->ws || !h->weights_ready) return h->fail(SSNB_ESTATE, "workspace/weights not set");
  return backbone_fwd(h, input_nchw, frames, feat, (cudaStream_t)stream);
}

int ssnb_bind_grads(ssnb_handle h, float* const* dw, float* const* db) {
  if (!h) return SSNB_EINVAL;
  h->dw.assign(h->convs.size(), nullptr); h->db.assign(h->convs.size(), nullptr);
  for (size_t i = 0; i < h->convs.size(); ++i) { if (dw) h->dw[i] = dw[i]; if (db) h->db[i] = db[i]; }
  return SSNB_OK;
}

int ssnb_backbone_bwd(ssnb_handle h, const float* dfeat, float* const* dw, float* const* db, void* stream) {
  return ssnb_backbone_bwd_range(h, dfeat, dw, db, -1, 0, stream);
}

int ssnb_backbone_bwd_range(ssnb_handle h, const float* dfeat, float* const* dw, float* const* db, int op_hi, int op_lo, void* stream) {
  if (!h || (!dfeat && (op_hi < 0 || op_hi >= (int)h->ops.size() - 1))) return h ? h->fail(SSNB_EINVAL, "null argument") : SSNB_EINVAL;
  if (!h->cfg.training) return h->fail(SSNB_ESTATE, "engine created without training=1");
  if (!h->ws || !h->weights_ready) return h->fail(SSNB_ESTATE, "workspace/weights not set");
  ssnb_bind_grads(h, dw, db);
  h->pending_finalize.clear();
  cudaStream_t s = (cudaStream_t)stream;
  // ops [first, last] of the reverse schedule; the global pool's backward (the first of them) reads the caller's dfeat
  auto run_range = [&](int hi, int lo) -> int {
    for (int i = hi; i >= lo; --i) {
      const Op& o = h->ops[i];
      const bool prof = profiled_op("SSNB_PROFILE_BWD_OPS", o.id);
      if (prof) cudaProfilerStart();
      int rc = run_bwd(h, o, dfeat, s, o.fuse_role != 0, true);   // siblings: mask/bias/wgrad only ...
      if (!rc && o.fuse_role == 1) {                                   // ... one fused data gradient
        const FusedBlock& fb = h->fused[o.fuse_block];
        double fl = 0.0;
        for (int j : {fb.op1, fb.op_r3, fb.op_rd}) if (j >= 0) fl += h->conv_flops(h->ops[j], h->F);
        tag_next(1, fl, fused_name(h, fb));
        rc = umma_conv_launch(h->umma_ctx, fb.dgrad, s, h->fold_pools && o.dgrad_masks);
      }
      if (prof) cudaProfilerStop();
      if (rc) return h->fail(rc, "bwd " + o.id + ": " + ssnb::thread_error());
    }
    return 0;
  };
  auto finalize = [&]() -> int {
    const float gs = h->tensor_cores() ? h->cfg.grad_scale : 1.0f;
    FinalizeTable t; t.n = 0; t.total_blocks = 0; t.flag = h->tc_flag; t.unscale = h->grad_unscale_dev();
    auto flush = [&]() -> int { int rc = launch_wgrad_finalize_all(t, 1.0f / gs, h->grad_accumulate, s); t.n = 0; t.total_blocks = 0; return rc; };
    for (int oi : h->pending_finalize) {
      const Op& o = h->ops[oi];
      const Conv& c = h->convs[o.conv];
      FinalizeEntry& q = t.e[t.n];
      q.partial = (const float*)(h->ws + o.partial_off); q.mult = (const float*)(h->ws + h->packed[o.conv].scale); q.dw = h->dw[o.conv];
      const bool bias_w = o.dy_premasked && o.bias_in_wgrad && h->db.size() && h->db[o.conv];
      q.bias_partial = bias_w ? (const float*)(h->ws + o.bias_partial_off) : nullptr; q.db = bias_w ? h->db[o.conv] : nullptr;
      q.splits = o.umma_wgrad.p.splits; q.taps = c.kh * c.kw; q.Cout = c.cout; q.Cin = c.cin; q.block0 = t.total_blocks; q.pad_ = 0;
      t.total_blocks += (int)(((long long)q.taps * q.Cout * q.Cin + 255) / 256);
      if (++t.n == FIN_MAX) if (int rc = flush()) { h->pending_finalize.clear(); return h->fail(rc, "finalize: " + ssnb::thread_error()); }
    }
    h->pending_finalize.clear();
    if (int rc = flush()) return h->fail(rc, "finalize: " + ssnb::thread_error());
    return 0;
  };
  const int last = (int)h->ops.size() - 1;
  if (op_hi < 0 || op_hi > last) op_hi = last;
  if (op_lo < 0 || op_lo > op_hi) return h->fail(SSNB_EINVAL, "backbone_bwd_range: bad op range");
  // the range that starts at the global pool reads dfeat: choose the gradient exponent of this backward from it first
  if (op_hi == last && h->tensor_cores()) {
    if (int rc = launch_grad_exponent(dfeat, (long long)h->F * h->vals[h->ops[last].in].C, h->cfg.grad_scale,
                                      h->bufs[h->vals[h->ops[last].in].buf].H * h->bufs[h->vals[h->ops[last].in].buf].W, h->gscale, h->tc_flag, s))
      return h->fail(rc, "gradient exponent: " + ssnb::thread_error());
  }
  if (int rc = run_range(op_hi, op_lo)) return rc;
  return finalize();
}

int ssnb_set_grad_accumulate(ssnb_handle h, int accumulate) {
  if (!h) return SSNB_EINVAL;
  h->grad_accumulate = accumulate ? 1 : 0;
  return SSNB_OK;
}

int ssnb_num_ops(ssnb_handle h) { return h ? (int)h->ops.size() : 0; }

int ssnb_op_info(ssnb_handle h, int op, char* kind, int kind_cap, char* in_name, int in_cap, char* out_name, int out_cap) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return SSNB_EINVAL;
  const Op& o = h->ops[op];
  if (kind) snprintf(kind, kind_cap, "%s", kOpKindName[o.kind]);
  if (in_name) snprintf(in_name, in_cap, "%s", h->vals[o.in].name.c_str());
  if (out_name) snprintf(out_name, out_cap, "%s", o.out >= 0 ? h->vals[o.out].name.c_str() : "feat");
  return SSNB_OK;
}

int ssnb_value_shape(ssnb_handle h, const char* name, int* c, int* hh, int* ww) {
  if (!h || !name) return SSNB_EINVAL;
  const int v = h->value_of(name);
  if (v < 0) return h->fail(SSNB_EINVAL, std::string("unknown value ") + name);
  const View w = h->view(v, false);
  if (c) *c = w.C; if (hh) *hh = w.H; if (ww) *ww = w.W;
  return SSNB_OK;
}

// the gradient exponent's 2^k (which = 0) or 2^-k (which = 1) on the host, after the work queued on `stream` (1 in EXACT_FP32)
static float host_gscale(ssnb_handle h, int which, cudaStream_t s) {
  float v = 1.0f;
  if (!h->tensor_cores() || cudaMemcpyAsync(&v, h->gscale + which, sizeof v, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess) { cudaGetLastError(); return 1.0f; }
  return v;
}

int ssnb_value_write(ssnb_handle h, const char* name, int grad, const float* src_nchw, void* stream) {
  if (!h || !name || !src_nchw || !h->ws) return SSNB_EINVAL;
  const int v = h->value_of(name);
  if (v < 0) return h->fail(SSNB_EINVAL, std::string("unknown value ") + name);
  if (grad && !h->cfg.training) return h->fail(SSNB_ESTATE, "no gradient buffers");
  // a gradient is stored in the units of the last backward: times 2^k (FAST: and grad_scale)
  const float sc = grad ? (h->fast() ? h->cfg.grad_scale : 1.0f) * host_gscale(h, 0, (cudaStream_t)stream) : 1.0f;
  const int rc = h->value_write(v, grad != 0, src_nchw, sc, h->F, (cudaStream_t)stream);
  return rc ? h->fail(rc, ssnb::thread_error()) : SSNB_OK;
}

int ssnb_value_read(ssnb_handle h, const char* name, int grad, float* dst_nchw, void* stream) {
  if (!h || !name || !dst_nchw || !h->ws) return SSNB_EINVAL;
  const int v = h->value_of(name);
  if (v < 0) return h->fail(SSNB_EINVAL, std::string("unknown value ") + name);
  if ((grad & 1) && !h->cfg.training) return h->fail(SSNB_ESTATE, "no gradient buffers");     // grad = 2: an activation's planes
  if (grad & 2) {       // diagnostic: read hi + lo of the value's EXACT_TC operand planes (bit 0: gradient planes, un-scaled)
    if (!h->exact_tc() || !h->bufs[h->vals[v].buf].plane) return h->fail(SSNB_ESTATE, "value has no operand planes");
    const float sc = (grad & 1) ? host_gscale(h, 1, (cudaStream_t)stream) / h->cfg.grad_scale : 1.0f;
    const int rc = h->planes_read(v, (grad & 1) != 0, sc, dst_nchw, (cudaStream_t)stream);
    return rc ? h->fail(rc, ssnb::thread_error()) : SSNB_OK;
  }
  const float sc = grad ? host_gscale(h, 1, (cudaStream_t)stream) / (h->fast() ? h->cfg.grad_scale : 1.0f) : 1.0f;
  const int rc = h->value_read(v, grad != 0, sc, dst_nchw, (cudaStream_t)stream);
  return rc ? h->fail(rc, ssnb::thread_error()) : SSNB_OK;
}

int ssnb_run_op(ssnb_handle h, int op, int backward, void* stream) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return SSNB_EINVAL;
  if (!h->ws || !h->weights_ready) return h->fail(SSNB_ESTATE, "workspace/weights not set");
  const Op& o = h->ops[op];
  if (o.kind == OP_GPOOL) return h->fail(SSNB_ENOSUPPORT, "run_op: global_pool runs through backbone_fwd/bwd");
  int rc = backward ? run_bwd(h, o, nullptr, (cudaStream_t)stream) : run_fwd(h, o, nullptr, h->F, (cudaStream_t)stream);
  return rc ? h->fail(rc, o.id + ": " + ssnb::thread_error()) : SSNB_OK;
}

int ssnb_grad_overflow(ssnb_handle h, int clear) {
  // did a gradient leave the fp16 range under the loss scale since the last clear?  EXACT_TC: an operand plane saw
  // |dz * grad_scale| > 65504 or NaN; FAST: a weight-gradient sum came out inf / NaN (fp16 gradient storage overflowed).
  // Synchronises the device (one 4-byte read).
  if (!h) return -1;
  if (!h->tc_flag) return 0;
  int v = 0;
  if (cudaMemcpy(&v, h->tc_flag, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); return -1; }
  if (v && clear) cudaMemset(h->tc_flag, 0, sizeof(int));
  return v ? 1 : 0;
}

int ssnb_timing_begin(void* stream) {
  for (TimingMark& m : ssnb::t_marks) ssnb::t_event_pool.push_back(m.ev);
  ssnb::t_marks.clear();
  ssnb::t_tag = LaunchTag();
  ssnb::t_timing = true;
  ssnb::timing_mark("(begin)", (cudaStream_t)stream);
  return SSNB_OK;
}

const char* ssnb_timing_report(void) {
  // closes the session, waits for the last launch and aggregates by (kernel, phase): "kernel\tphase\tlaunches\tms\tflop\n"
  ssnb::t_report.clear();
  if (!ssnb::timing_close()) return ssnb::t_report.c_str();
  struct Agg { int n = 0; double ms = 0, flop = 0; };
  std::map<std::pair<std::string, int>, Agg> agg;
  for (size_t i = 1; i < ssnb::t_marks.size(); ++i) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ssnb::t_marks[i - 1].ev, ssnb::t_marks[i].ev) != cudaSuccess) { cudaGetLastError(); continue; }
    Agg& a = agg[{ssnb::t_marks[i].what, ssnb::t_marks[i].tag.phase}];
    a.n += 1; a.ms += ms; a.flop += ssnb::t_marks[i].tag.flop;
  }
  char line[256];
  for (const auto& kv : agg) {
    snprintf(line, sizeof line, "%s\t%d\t%d\t%.6f\t%.0f\n", kv.first.first.c_str(), kv.first.second, kv.second.n, kv.second.ms, kv.second.flop);
    ssnb::t_report += line;
  }
  return ssnb::t_report.c_str();
}

const char* ssnb_timing_launches(void) {
  // closes the session (if still open) and lists its launches in order: "kernel\tphase\top\tms\tflop\ttiles\tblock_n\n"
  ssnb::t_report.clear();
  if (!ssnb::timing_close()) return ssnb::t_report.c_str();
  char line[512];
  for (size_t i = 1; i < ssnb::t_marks.size(); ++i) {
    const ssnb::TimingMark& m = ssnb::t_marks[i];
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ssnb::t_marks[i - 1].ev, m.ev) != cudaSuccess) { cudaGetLastError(); continue; }
    snprintf(line, sizeof line, "%s\t%d\t%s\t%.6f\t%.0f\t%d\t%d\n", m.what, m.tag.phase, m.op.empty() ? "-" : m.op.c_str(), ms, m.tag.flop,
             m.tag.tiles, m.tag.block_n);
    ssnb::t_report += line;
  }
  return ssnb::t_report.c_str();
}

int64_t ssnb_launch_count(ssnb_handle h) { return h ? (int64_t)(g_launches.load() - h->launches0) : 0; }
int64_t ssnb_global_launch_count(void) { return (int64_t)g_launches.load(); }

}  // extern "C"
