// Host-side graph core of the backbone engines (BNInception in engine.cu, InceptionV3 in inception_v3.cu): the graph
// records, graph building, operand views, the forward-storage planner, the weight pack, the forward of the ops that do not
// run on the tensor cores, and value I/O.  Each engine adds the graph table and the schedule only it has.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "../../include/ssnb.h"
#include "common.cuh"

namespace ssnb {

// one convolution + BatchNorm (+ ReLU); `id` is the graph's name of the blob it writes
struct Conv { std::string id; int cin, cout, kh, kw, stride, ph, pw; };
// activation (off) and gradient (goff) storage; EXACT_TC: fp16 hi / lo operand planes of both (lo = hi + plane)
struct Buffer { std::string name; int H, W, C; size_t off = 0, goff = 0, hoff = 0, ghoff = 0, plane = 0; };
// channels [coff, coff + C) of a buffer: a whole buffer, or one branch of a concat buffer
struct Value { std::string name; int buf, coff, C; };
// OP_BN1 (BNInception only): training-mode BatchNorm + ReLU behind conv1 (bn_mode='partial')
enum OpKind { OP_CONV = 0, OP_MAXPOOL = 1, OP_AVGPOOL = 2, OP_GPOOL = 3, OP_BN1 = 4 };
const char* const kOpKindName[] = {"conv", "maxpool", "avgpool", "gpool", "bn"};
// the forward fields of an op; `out` = -1 for the global pool, which writes the caller's feat
struct GraphOp { OpKind kind; std::string id; int in, out; int conv = -1, k = 0, stride = 1, pad = 0; size_t argmax_off = 0; };
// EXACT_TC: fp16 hi planes of wf / wd (lo = hi + wplane); wmax: [0] max |folded weight|, [1] 1 / the power-of-two plane scale
struct PackedConv { size_t wf, wd, bias, scale; size_t wf16 = 0, wd16 = 0, wplane = 0, wmax = 0; };

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int conv_out(int h, int k, int s, int p) { return (h + 2 * p - k) / s + 1; }
// Caffe's ceil mode (layer_factory.py:46-50): the last window must start inside the input or its left padding
inline int pool_out(int h, int k, int s, int p) {
  int o = (h + 2 * p - k + s - 1) / s + 1;
  if ((o - 1) * s >= h + p) --o;
  return o;
}

template <class Op>
struct Graph {
  int F = 0, precision = SSNB_EXACT_FP32;
  size_t esz = 4;                     // bytes of an activation: 2 in FAST, 4 otherwise
  std::vector<Conv> convs;
  std::vector<Buffer> bufs;
  std::vector<Value> vals;
  std::map<std::string, int> val_by_name;
  std::vector<Op> ops;
  std::vector<PackedConv> packed;
  size_t wmax_off = 0, wmax_slots = 0;  // EXACT_TC: the contiguous (absmax, 1 / scale) slots, zeroed before every pack
  char* ws = nullptr;

  bool fast() const { return precision == SSNB_FAST_FP16; }          // fp16 storage, fp16 operands
  bool exact_tc() const { return precision == SSNB_EXACT_TC; }       // fp32 storage, convolutions on split (hi/lo fp16) operand planes
  bool tensor_cores() const { return precision != SSNB_EXACT_FP32; } // either of the two: the wgmma schedule

  // ---- graph building ----
  int add_buffer(const std::string& name, int H, int W, int C) { bufs.push_back({name, H, W, C}); return (int)bufs.size() - 1; }
  int add_value(const std::string& name, int buf, int coff, int C) {
    vals.push_back({name, buf, coff, C});
    val_by_name[name] = (int)vals.size() - 1;
    return (int)vals.size() - 1;
  }
  int whole(const std::string& name, int H, int W, int C) { return add_value(name, add_buffer(name, H, W, C), 0, C); }
  int value_of(const char* name) const {
    if (!name) return -1;
    auto it = val_by_name.find(name);
    return it == val_by_name.end() ? -1 : it->second;
  }

  // ---- views of a value (activation or gradient) ----
  View view(int v, bool grad = false) const {
    const Value& x = vals[v];
    const Buffer& b = bufs[x.buf];
    View w;
    w.base = ws + (grad ? b.goff : b.off);
    w.H = b.H; w.W = b.W; w.C = x.C; w.pitch = b.C; w.coff = x.coff;
    return w;
  }
  // EXACT_TC: the value's fp16 hi / lo operand planes
  View planes(int v, bool grad = false) const {
    const Buffer& b = bufs[vals[v].buf];
    View w = view(v, grad);
    w.base = ws + (grad ? b.ghoff : b.hoff); w.lo_off = (long long)b.plane;
    return w;
  }
  // what the tensor-core kernels read and write: the fp16 storage (FAST) or the operand planes (EXACT_TC)
  View operand(int v, bool grad = false) const { return exact_tc() ? planes(v, grad) : view(v, grad); }

  // ---- forward-storage planner ----
  // From `off`: activations (and their gradients when training), EXACT_TC operand planes of every buffer whose channels
  // are a multiple of 8, the arg-max bytes of every max pool, the packed weights of every convolution (k0: convolution
  // 0's input channels as the kernels read them), and in EXACT_TC one (absmax, 1 / scale) slot per convolution plus
  // `extra_slots`.  Returns the end of what it planned.
  size_t plan_storage(size_t off, bool training, int k0, int extra_slots) {
    const size_t N = (size_t)F;
    for (Buffer& b : bufs) { b.off = off; off = align_up(off + N * b.H * b.W * b.C * esz, 1024); }
    if (training)
      for (Buffer& b : bufs) { b.goff = off; off = align_up(off + N * b.H * b.W * b.C * esz, 1024); }
    if (exact_tc())
      for (Buffer& b : bufs) {
        if (b.C % 8) continue;        // BNInception's 3- / 10-channel input has no planes: conv1 reads its own packed copy
        b.plane = align_up(N * b.H * b.W * b.C * 2, 1024);
        b.hoff = off; off += 2 * b.plane;
        if (training) { b.ghoff = off; off += 2 * b.plane; }
      }
    for (Op& o : ops)
      if (o.kind == OP_MAXPOOL) {     // the vectorised max pool records its arg-max (one byte per output element)
        const View out = view(o.out);
        o.argmax_off = off; off = align_up(off + N * out.H * out.W * out.C, 1024);
      }
    packed.resize(convs.size());
    for (size_t i = 0; i < convs.size(); ++i) {
      const Conv& c = convs[i];
      const size_t n = (size_t)c.cout * (i == 0 ? k0 : c.cin) * c.kh * c.kw;
      PackedConv& p = packed[i];
      p.wf = off; off = align_up(off + n * esz, 1024);
      p.wd = off; off = align_up(off + n * esz, 1024);
      p.bias = off; off = align_up(off + c.cout * 4, 256);
      p.scale = off; off = align_up(off + c.cout * 4, 256);
      if (exact_tc()) {
        p.wplane = align_up(n * 2, 1024);
        p.wf16 = off; off += 2 * p.wplane;
        p.wd16 = off; off += 2 * p.wplane;
      }
    }
    if (exact_tc()) {
      wmax_off = off; wmax_slots = convs.size() + extra_slots;
      for (size_t i = 0; i < convs.size(); ++i) packed[i].wmax = off + i * 8;
      off = align_up(off + wmax_slots * 8, 1024);
    }
    return off;
  }

  // ---- weight pack ----
  // BatchNorm fold and re-layout of every convolution (k0 as in plan_storage), PACK_MAX layers per launch; EXACT_TC: every
  // fold launch first (layers may share an absmax slot), then the hi / lo splits.  adjust(i, pack_entry, split_entry) sets
  // what only one engine needs on convolution i's entries (split_entry is null outside EXACT_TC).  On failure the thread's
  // error reads "<what>: ..." / "<what> split: ...".
  template <class Adjust>
  int pack_weights(const float* const* w, const float* const* b, const float* const* gamma, const float* const* beta,
                   const float* const* mean, const float* const* var, int k0, Adjust&& adjust, const std::string& what, cudaStream_t s) {
    if (exact_tc() && cudaMemsetAsync(ws + wmax_off, 0, wmax_slots * 8, s) != cudaSuccess) {
      set_thread_error(what + ": memset failed");
      return SSNB_ECUDA;
    }
    std::vector<PackTable> pt;
    std::vector<SplitTable> st;
    std::vector<int> pblocks, sblocks;
    for (size_t i = 0; i < convs.size(); ++i) {
      const Conv& c = convs[i];
      const PackedConv& p = packed[i];
      const int ck = i == 0 ? k0 : c.cin, taps = c.kh * c.kw;
      if (i % PACK_MAX == 0) {
        pt.emplace_back(); pt.back().n = 0; pt.back().pad_ = 0; pblocks.push_back(0);
        st.emplace_back(); st.back().n = 0; st.back().pad_ = 0; sblocks.push_back(0);
      }
      PackEntry& q = pt.back().e[pt.back().n++];
      q.w = w[i]; q.b = b[i]; q.gamma = gamma[i]; q.beta = beta[i]; q.mean = mean[i]; q.var = var[i];
      q.wf = ws + p.wf; q.wd = ws + p.wd; q.bias = (float*)(ws + p.bias); q.scale = (float*)(ws + p.scale);
      q.absmax = exact_tc() ? (float*)(ws + p.wmax) : nullptr;
      q.cout = c.cout; q.cin = ck; q.taps = taps; q.block0 = pblocks.back();
      q.nofold = 0; q.pad_[0] = q.pad_[1] = q.pad_[2] = 0; q.bias_b = nullptr;
      pblocks.back() += pack_ctas(c.cout, ck, taps);
      SplitEntry* se = nullptr;
      if (exact_tc()) {               // hi / lo planes of both layouts with the layer's power-of-two scale (tc_glue.cu)
        const long long n = (long long)c.cout * ck * taps;
        se = &st.back().e[st.back().n++];
        se->wf = (const float*)(ws + p.wf); se->wd = (const float*)(ws + p.wd);
        se->wf16 = (__half*)(ws + p.wf16); se->wd16 = (__half*)(ws + p.wd16); se->plane_bytes = (long long)p.wplane; se->n = n;
        se->absmax = (const float*)(ws + p.wmax); se->inv_scale = (float*)(ws + p.wmax) + 1; se->block0 = sblocks.back(); se->pad_ = 0;
        se->wd16_b = nullptr; se->wf16_b = nullptr; se->b_plane_bytes = 0; se->b_pitch = 0; se->cout = c.cout;
        sblocks.back() += (int)((n + 255) / 256);
      }
      adjust(i, q, se);
    }
    for (size_t k = 0; k < pt.size(); ++k)
      if (int rc = fast() ? launch_pack_all<__half>(pt[k], pblocks[k], s) : launch_pack_all<float>(pt[k], pblocks[k], s)) {
        set_thread_error(what + ": " + thread_error());
        return rc;
      }
    if (exact_tc())
      for (size_t k = 0; k < st.size(); ++k)
        if (int rc = launch_split_all(st[k], sblocks[k], s)) {
          set_thread_error(what + " split: " + thread_error());
          return rc;
        }
    return SSNB_OK;
  }

  // ---- forward of the ops that do not run on the tensor cores ----
  // The forward helpers below run the first n <= F frames of the plan: every launch covers frames [0, n) only, and a frame's
  // arithmetic does not depend on n.
  // algorithmic FLOPs of convolution op `o` over n frames (timing tags)
  double conv_flops(const GraphOp& o, int n) const {
    const Conv& c = convs[o.conv];
    const View out = view(o.out);
    return 2.0 * n * out.H * out.W * (double)c.cout * c.cin * c.kh * c.kw;
  }
  // vectorised max pool / 3x3 average pool; EXACT_TC also writes the output's operand planes (the next convolution's A operand)
  int pool_fwd(const GraphOp& o, int n, cudaStream_t s) const {
    const View in = view(o.in), out = view(o.out);
    const View pl = exact_tc() && bufs[vals[o.out].buf].plane ? planes(o.out) : View();
    uint8_t* am = (uint8_t*)(ws + o.argmax_off);
    if (o.kind == OP_MAXPOOL)
      return fast() ? launch_maxpool_fwd_vec<__half>(in, out, pl, n, o.k, o.stride, o.pad, am, s)
                    : launch_maxpool_fwd_vec<float>(in, out, pl, n, o.k, o.stride, o.pad, am, s);
    return fast() ? launch_avgpool3_vec<__half>(in, out, pl, n, 0, s) : launch_avgpool3_vec<float>(in, out, pl, n, 0, s);
  }
  // global average pool of op `o`'s input into feat [n, C]
  int gpool_fwd(const GraphOp& o, int n, float* feat, cudaStream_t s) const {
    return fast() ? launch_gpool_fwd<__half>(view(o.in), n, feat, s) : launch_gpool_fwd<float>(view(o.in), n, feat, s);
  }
  // SIMT convolution forward of op `o` from the packed fp32 / fp16 weights; relu = 0 leaves the result un-clamped
  int simt_conv_fwd(const GraphOp& o, int relu, int n, cudaStream_t s) const {
    const Conv& c = convs[o.conv];
    const View in = view(o.in), out = view(o.out);
    ConvArgs a;
    a.src = in.base; a.SH = in.H; a.SW = in.W; a.Csrc = in.C; a.src_pitch = in.pitch; a.src_coff = in.coff;
    a.dst = out.base; a.DH = out.H; a.DW = out.W; a.Cdst = out.C; a.dst_pitch = out.pitch; a.dst_coff = out.coff;
    a.wgt = ws + packed[o.conv].wf; a.bias = (const float*)(ws + packed[o.conv].bias);
    a.F = n; a.kh = c.kh; a.kw = c.kw; a.stride = c.stride; a.pad_h = c.ph; a.pad_w = c.pw; a.relu = relu; a.accumulate = 0; a.dgrad = 0;
    t_tag.phase = 0; t_tag.flop = conv_flops(o, n); t_tag.op = o.id.c_str();
    return fast() ? launch_conv<__half>(a, s) : launch_conv<float>(a, s);
  }

  // ---- value I/O (NCHW fp32 on the caller's side) ----
  // frames [0, n) of the value's storage = src * scale; EXACT_TC refreshes an activation's operand planes (a padded input:
  // every channel of the pixel, the padding included)
  int value_write(int v, bool grad, const float* src, float scale, int n, cudaStream_t s) const {
    const View w = view(v, grad);
    int rc = fast() ? launch_nchw_to_nhwc<__half>(src, n, w.C, w.H, w.W, w, scale, s)
                    : launch_nchw_to_nhwc<float>(src, n, w.C, w.H, w.W, w, scale, s);
    if (!rc && exact_tc() && !grad && bufs[vals[v].buf].plane) {
      View x = w, xp = planes(v);
      if (w.C % 8) x.C = xp.C = w.pitch;
      rc = launch_split_view(x, n, 1.0f, xp, nullptr, s);
    }
    return rc;
  }
  // dst = the value's storage * scale
  int value_read(int v, bool grad, float scale, float* dst, cudaStream_t s) const {
    return fast() ? launch_nhwc_to_nchw<__half>(view(v, grad), F, scale, dst, s) : launch_nhwc_to_nchw<float>(view(v, grad), F, scale, dst, s);
  }
  // EXACT_TC: dst = (hi + lo of the value's operand planes) * scale
  int planes_read(int v, bool grad, float scale, float* dst, cudaStream_t s) const {
    return launch_planes_to_nchw(planes(v, grad), F, scale, dst, s);
  }
};

}  // namespace ssnb
