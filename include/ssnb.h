/* ssnb.h — C ABI of libssn_b200.so: the H100-native SSN forward/backward hot path.
 *
 * The reference (yjxiong/action-detection) has no FFI: its hot path is Python calling stock
 * PyTorch ops.  This ABI is what a binding for that path binds instead; each entry names the
 * reference interface it replaces (file:line relative to the reference root).  Plain pointers
 * and sizes only — no torch types.  All device pointers are CUDA device memory owned by the
 * caller; `stream` is a cudaStream_t passed as void*.  Every function returns 0 on success and a
 * non-zero code otherwise (never throws, never aborts); ssnb_last_error() returns the message.
 * All work is enqueued on `stream`; no call synchronises the device.
 */
#ifndef SSNB_H
#define SSNB_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ssnb_engine* ssnb_handle;

enum { SSNB_OK = 0, SSNB_EINVAL = 1, SSNB_ECUDA = 2, SSNB_ESTATE = 3, SSNB_ENOSUPPORT = 4 };

/* precision modes of the backbone */
enum {
  SSNB_EXACT_FP32 = 0, /* fp32 storage, fp32 SIMT FMA: end-to-end parity mode */
  SSNB_FAST_FP16 = 1,  /* fp16 storage, wgmma f16 MMA with fp32 register accumulators */
  SSNB_EXACT_TC = 2    /* fp32 storage; every convolution product as error-compensated split fp16 operands
                          (x = hi + lo, three wgmma MMAs a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, fp32 accumulate):
                          fp32-grade results (layer_factory.py:25-39 computes in fp32) on the tensor cores */
};

typedef struct {
  int32_t in_channels; /* 3 (RGB) or 10 (Flow 2x5), ssn_models.py:260 sample_len */
  int32_t frames;      /* F = proposals * segments processed per call */
  int32_t precision;   /* SSNB_EXACT_FP32 | SSNB_FAST_FP16 | SSNB_EXACT_TC */
  int32_t training;    /* 1: keep activations + allocate gradient buffers */
  float grad_scale;    /* loss scale (FAST: fp16 gradient storage; EXACT_TC: the fp16 operand planes of the output gradients).
                          Not needed for range: every backward of the tensor-core modes also multiplies the gradient by 2^k,
                          k chosen on the device from max |dfeat|, and divides dW / db / dgamma / dbeta by it again */
  int32_t bn1_train;   /* 1: the FIRST BatchNorm2d (conv1's) runs in training mode -- batch statistics, running-stat update, gradients for
                          its weight / bias: bn_mode='partial' (ssn_models.py:95-105,156-174).  EXACT_FP32 / EXACT_TC only. */
  int32_t reserved[2];
} ssnb_config;

/* ---- engine lifetime ---------------------------------------------------------------------- */
int ssnb_create(const ssnb_config* cfg, ssnb_handle* out);
int ssnb_destroy(ssnb_handle h);
/* h may be NULL: returns the calling thread's last error from a handle-less function. */
const char* ssnb_last_error(ssnb_handle h);
const char* ssnb_version(void);

/* ---- BNInception backbone: replaces model_zoo.BNInception (pytorch_load.py:8-61) as used by
 *      SSN.train_forward / test_forward (ssn_models.py:266, :298) ------------------------------ */
/* the 69 convolutions in graph order (bn_inception.yaml); lets the host check its own table */
int ssnb_num_convs(void);
int ssnb_conv_info(int idx, int in_channels, char* name, int name_cap, int* cin, int* cout, int* k,
                   int* stride, int* pad);
/* caller-owned scratch (activations, gradients, packed weights, split-K partials) */
size_t ssnb_workspace_bytes(ssnb_handle h);
int ssnb_set_workspace(ssnb_handle h, void* dev_ptr, size_t bytes);
/* Fold frozen BatchNorm2d (ssn_models.py:156-174) into each conv and re-layout for the kernels.
 * Arrays of ssnb_num_convs() device pointers in graph order, reference shapes: w [cout,cin,k,k],
 * b/gamma/beta/mean/var [cout].  Call after every optimizer step. */
int ssnb_pack_weights(ssnb_handle h, const float* const* w, const float* const* b, const float* const* gamma,
                      const float* const* beta, const float* const* mean, const float* const* var, void* stream);
/* bn1_train engines: the first BatchNorm2d's tensors (device pointers, 64 floats each).  gamma / beta / running stats are read
 * (running stats also updated) by ssnb_backbone_fwd; dgamma / dbeta (may be NULL) are written by ssnb_backbone_bwd
 * (added to when grad accumulation is on).  conv1's weights are then packed WITHOUT a BatchNorm fold. */
int ssnb_set_bn1(ssnb_handle h, const float* gamma, const float* beta, float* running_mean, float* running_var, float* dgamma,
                 float* dbeta, float momentum, float eps);
/* input [F, C, 224, 224] fp32 NCHW (the reference's frame tensor after input.view(-1, C, H, W),
 * ssn_models.py:266) -> feat [F, 1024] fp32 (global_pool output, fc replaced by Identity/Dropout) */
int ssnb_backbone_fwd(ssnb_handle h, const float* input_nchw, float* feat, void* stream);
/* The same forward over the first `frames` frames of the plan, 1 <= frames <= F: input [frames, C, 224, 224] -> feat
 * [frames, 1024], rows bitwise those of an engine planned for `frames`, on this engine's workspace and with the launches of
 * `frames` frames (no row of a frame >= frames is read from the input or written to feat).  frames == F is ssnb_backbone_fwd.
 * Forward-only engines: SSNB_EINVAL for frames outside 1 .. F, SSNB_ESTATE for a training engine, SSNB_ENOSUPPORT for a
 * bn1_train engine, each before any launch.  Binds nothing, so a call can be captured in a CUDA graph. */
int ssnb_backbone_fwd_frames(ssnb_handle h, const float* input_nchw, int frames, float* feat, void* stream);
/* dfeat [F,1024] fp32 -> dw[i] [cout,cin,k,k], db[i] [cout] fp32 in reference layout (what autograd
 * leaves in Conv2d.weight.grad / .bias.grad; BN params are frozen and get none).  Overwrites. */
int ssnb_backbone_bwd(ssnb_handle h, const float* dfeat, float* const* dw, float* const* db, void* stream);
/* The same backward in pieces, for overlapping the gradient exchange with it: runs the reverse schedule for ops
 * op_hi .. op_lo (indices of ssnb_op_info; op_hi < 0 = the last op, the global pool, which reads dfeat) and finalises the
 * weight / bias gradients of exactly those ops, so after the call dw[i] / db[i] of their convolutions are complete and a
 * bucket all-reduce can be issued on another stream while the next range runs.  Ranges must be issued from the top down. */
int ssnb_backbone_bwd_range(ssnb_handle h, const float* dfeat, float* const* dw, float* const* db, int op_hi, int op_lo,
                            void* stream);
/* 0 (default): ssnb_backbone_bwd overwrites dw/db; 1: it adds to them (what autograd's AccumulateGrad does
 * with Conv2d.weight.grad), so the caller can hand in the live .grad tensors */
int ssnb_set_grad_accumulate(ssnb_handle h, int accumulate);
/* bind the gradient outputs used by ssnb_run_op(backward=1) without running the whole backward */
int ssnb_bind_grads(ssnb_handle h, float* const* dw, float* const* db);

/* introspection for per-layer parity tests: named values are the reference's blob names
 * ("data", "conv1_7x7_s2_bn", "pool1_3x3_s2", "inception_3a_output", ...). */
int ssnb_num_ops(ssnb_handle h);
int ssnb_op_info(ssnb_handle h, int op, char* kind, int kind_cap, char* in_name, int in_cap, char* out_name, int out_cap);
int ssnb_value_shape(ssnb_handle h, const char* name, int* c, int* hh, int* ww);
int ssnb_value_write(ssnb_handle h, const char* name, int grad, const float* src_nchw, void* stream);
int ssnb_value_read(ssnb_handle h, const char* name, int grad, float* dst_nchw, void* stream);
int ssnb_run_op(ssnb_handle h, int op, int backward, void* stream);
/* Loss-scale guard: 1 when a gradient left the fp16 range since the last clear (dfeat held an inf / NaN; EXACT_TC: an operand
 * plane saw |dz * grad_scale * 2^k| > 65504 or NaN; FAST: a weight-gradient sum came out inf / NaN), 0 otherwise, -1 on error.
 * Synchronises the device: poll it every N steps and skip / rescale like a dynamic loss scaler would. */
int ssnb_grad_overflow(ssnb_handle h, int clear);

/* Per-launch device timing for the roofline figures (bench.py): ssnb_timing_begin opens a session on the calling thread
 * (every library launch then records a CUDA event on its stream); ssnb_timing_report closes it, waits for the last
 * launch and returns lines "kernel\tphase\tlaunches\tms\talgorithmic_flop\n" aggregated by kernel and pass
 * (phase 0 forward, 1 data gradient, 2 weight gradient, 3 other).  The string is owned by the library (thread-local). */
int ssnb_timing_begin(void* stream);
const char* ssnb_timing_report(void);
/* The same session launch by launch, in launch order: "kernel\tphase\top\tms\talgorithmic_flop\ttiles\tblock_n\n" with op the
 * engine's op name ("a+b+c" for a fused sibling launch, "-" for untagged glue) and tiles / block_n the tile count and tile
 * width of a umma_conv_kernel launch, the CTAs per pixel split and the split count (grid x and y) of a umma_wgrad_kernel
 * launch (0 otherwise).  Closes the session if it is still open; may follow ssnb_timing_report. */
const char* ssnb_timing_launches(void);
/* per-kernel-family launch counters since creation (bench.py's gpu_launches claim) */
int64_t ssnb_launch_count(ssnb_handle h);
int64_t ssnb_global_launch_count(void);

/* ---- STPP: replaces StructuredTemporalPyramidPooling.forward (ops/ssn_ops.py:39-70) ----------
 * ft [n*n_seg, D]; scaling [n,2]; parts: n_parts entries (lo, hi, norm, scale_col) over segment
 * indices (host mirrors the tick arithmetic of :49-53); course = mean over [course_lo, course_hi).
 * out: course_ft [n,D], stpp_ft [n, n_parts*D].
 * n_parts == 0 (0..32 parts): the course mean only (BinaryClassifier, binary_model.py:229-230); the part arrays, scaling,
 * stpp_ft / d_stpp are not read or written and may be NULL (ssnb_stpp_bwd then needs d_course). */
int ssnb_stpp_fwd(const float* ft, const float* scaling, int n, int n_seg, int D, int n_parts, const int* part_lo,
                  const int* part_hi, const int* part_norm, const int* part_scale_col, int course_lo, int course_hi,
                  float* course_ft, float* stpp_ft, void* stream);
int ssnb_stpp_bwd(const float* d_course, const float* d_stpp, const float* scaling, int n, int n_seg, int D,
                  int n_parts, const int* part_lo, const int* part_hi, const int* part_norm,
                  const int* part_scale_col, int course_lo, int course_hi, float* d_ft, void* stream);
/* fused tail of the backbone: 7x7 global average pool (bn_inception.yaml:552) + optional dropout
 * mask + STPP, reading the engine's 5b output directly.  feat [F,1024] is also written. */
int ssnb_gpool_stpp_fwd(ssnb_handle h, const float* drop_mask, const float* scaling, int n_seg, int n_parts,
                        const int* part_lo, const int* part_hi, const int* part_norm, const int* part_scale_col,
                        int course_lo, int course_hi, float* feat, float* course_ft, float* stpp_ft, void* stream);

/* ---- STPPReorgainzed.forward (ops/ssn_ops.py:109-170), standalong_classifier + regression ----
 * scores [T, D] with D = act_len + M*comp_len + M*reg_len; ticks [N,4] int32; scaling [N,2];
 * stage_parts: 3 stages, parts-per-level lists flattened: level_counts[3] + levels[].
 * One fp64 exclusive column scan of scores (workspace: (T+1)*D doubles, ssnb_stpp_reorg_workspace_bytes)
 * + one gather per proposal: every part costs two loads instead of its row count (1000 heavily overlapping proposals/video). */
size_t ssnb_stpp_reorg_workspace_bytes(int T, int D);
int ssnb_stpp_reorg_prefix(const float* scores, int T, int D, const int32_t* ticks, const float* scaling, int N, int act_len,
                           int comp_len, int reg_len, const int* level_counts, const int* levels, float* out_act,
                           float* out_comp, float* out_reg, void* workspace, void* stream);
/* ---- the per-video tail of ssn_test.py's worker loop (ssn_test.py:87-92) for V videos in one call: STPPReorgainzed.forward
 *      (ops/ssn_ops.py:109-170) of every video, then the regression de-normalisation by the checkpoint's reg_stats ----------
 * Video v owns ticks tick_offsets[v] .. tick_offsets[v+1]-1 of the packed score table scores [sum T, D] (fp32, D = act_len +
 * M*comp_len + M*reg_len) and proposal rows offsets[v] .. offsets[v+1]-1 of ticks [sum N, 4] int32 and scaling [sum N, 2]
 * fp32 (ssnb_test_proposals' ticks32 / scaling32 in its row layout).  Writes act [sum N, act_len], comp [sum N, comp_len] and
 * reg [sum N, reg_len] in the same row order, the layout ssnb_detect_batch reads.  Each video's rows are bitwise what
 * ssnb_stpp_reorg_prefix gives for that video alone, which is this call with V = 1 (same kernels: one fp64 exclusive column
 * scan per video segment, one gather per proposal).  A video with N_v = 0 writes nothing; one with T_v = 0 pools empty
 * slices (NaN), as the reference's slices of an empty table do.
 * reg_stats: NULL, or HOST double [4] = {mean loc, mean size, std loc, std size} (the [2, 2] reg_stats, means then stds):
 * reg[:, 2k] = fp32(fp32(x * (float)std loc) + (float)mean loc), reg[:, 2k+1] likewise with the size pair, each op rounded
 * on its own as torch runs ssn_test.py:90-92 (reg_len must be even).
 * tick_offsets and offsets (int64 [V+1], [0] = 0, non-decreasing) are HOST memory: validated, they size the call;
 * tick_offsets_dev / offsets_dev hold the same values on the device.  Workspace: (sum T + V) * D doubles, the per-video
 * prefix tables (ssnb_stpp_reorg_batch_workspace_bytes; 0 for arguments the call rejects).  At K = 100 and (1,(1,2),1),
 * D = 1601: 12.8 KB of workspace per tick beside the 6.4 KB of scores.  Bad arguments are refused before any launch.
 * Kernels only: no host synchronisation, allocation or host copy (graph-capturable). */
size_t ssnb_stpp_reorg_batch_workspace_bytes(const int64_t* tick_offsets, int n_videos, int D);
int ssnb_stpp_reorg_batch(const float* scores, int D, const int64_t* tick_offsets, const int64_t* tick_offsets_dev, const int32_t* ticks,
                          const float* scaling, const int64_t* offsets, const int64_t* offsets_dev, int n_videos, int act_len, int comp_len,
                          int reg_len, const int* level_counts, const int* levels, const double* reg_stats, float* out_act, float* out_comp,
                          float* out_reg, void* workspace, size_t workspace_bytes, void* stream);

/* ---- heads: activity_fc / completeness_fc / regressor_fc (ssn_models.py:272-283) ------------- */
int ssnb_linear_fwd(const float* x, const float* w, const float* b, int n, int in_dim, int out_dim, float* y,
                    void* stream);
/* Test-time scores of one chunk of a video with the 10-crop mean folded into the folded FC (replaces
 * `rst, _ = net(input); sc = rst.view(num_crop, -1, D).mean(0)`, ssn_test.py:83-84, with test_fc from
 * SSN.prepare_test_fc, ssn_models.py:176-201): feat [crops*nt, in_dim] crop-major -> y [nt, out_dim]. */
int ssnb_test_fc_cropmean(const float* feat, const float* w, const float* b, int crops, int nt, int in_dim, int out_dim,
                          float* y, void* stream);
/* dy [n,out] -> dx [n,in] (may be NULL), dw [out,in], db [out]; overwrite */
int ssnb_linear_bwd(const float* x, const float* w, const float* dy, int n, int in_dim, int out_dim, float* dx,
                    float* dw, float* db, void* stream);

/* ---- losses ------------------------------------------------------------------------------------
 * OHEMHingeLoss.forward/backward (ops/ssn_ops.py:180-213): pred [m,K], labels [m] int64 1-based
 * (0 wraps to class K-1); groups of group_size rows; keep_num = int(group_size*ratio) computed by
 * the caller.  loss[1]; kept [m] uint8 marks the rows whose gradient is written; slopes has room for
 * 2*m floats (slopes [m] followed by the per-row hinge losses [m]). */
int ssnb_ohem_hinge_fwd(const float* pred, const int64_t* labels, int m, int K, int is_positive, int group_size,
                        int keep_num, float* loss, uint8_t* kept, float* slopes, void* stream);
int ssnb_ohem_hinge_bwd(const int64_t* labels, const uint8_t* kept, const float* slopes, const float* grad_out,
                        int m, int K, float* grad_pred, void* stream);
/* ClassWiseRegressionLoss.forward (ops/ssn_ops.py:251-258) and its gradient */
int ssnb_classwise_reg_fwd(const float* pred, const int64_t* labels, const float* targets, int n, int K, float* loss,
                           void* stream);
int ssnb_classwise_reg_bwd(const float* pred, const int64_t* labels, const float* targets, const float* grad_out,
                           int n, int K, float* grad_pred, void* stream);

/* Fused classifier + multi-task loss forward AND backward in one kernel (ssn_models.py:272-289 +
 * ssn_train.py:210-214): three heads, row selection by prop_type, CE + w_comp*completeness(OHEM) +
 * w_reg*class-wise smooth-L1, and all gradients (d course_ft, d stpp_ft, dW, db of the heads). */
typedef struct {
  int32_t n;             /* proposals (videos * props_per_video) */
  int32_t props_per_video;
  int32_t num_class;     /* K */
  int32_t feat_dim;      /* 1024 */
  int32_t feat_mult;     /* M */
  int32_t fg_per_video;  /* sample_split (ssn_train.py:189) */
  int32_t comp_group;    /* fg + incomplete per video (ssn_train.py:190) */
  int32_t global_videos; /* videos in the GLOBAL batch: completeness denominator (SURVEY §8e) */
  int32_t keep_neg;      /* int((comp_group - fg_per_video) * ohem_ratio), host-computed (ops/ssn_ops.py:191) */
  float comp_denom;      /* (pos_cnt + int(neg_cnt * ohem_ratio)) of the GLOBAL batch (ops/ssn_ops.py:236-239)
                            divided by the number of data-parallel ranks, so that rank-averaged losses and
                            gradients equal the global-batch ones (SURVEY §8e) */
  float comp_w, reg_w;   /* 0.1, 0.1 (ssn_opts.py:35-37) */
  float loss_scale;      /* multiplies every gradient (1/world_size for data parallel) */
} ssnb_heads_cfg;
size_t ssnb_heads_loss_workspace_bytes(const ssnb_heads_cfg* cfg);
/* prop_type/target int64 [n]; reg_target [n,2].  outputs: raw_act [n,K+1], raw_comp [n,K],
 * raw_reg [n,2K] (all rows, unselected), losses[4] = {act, comp, reg, total}. */
int ssnb_heads_loss_fwd_bwd(const ssnb_heads_cfg* cfg, const float* course_ft, const float* stpp_ft,
                            const float* act_w, const float* act_b, const float* comp_w, const float* comp_b,
                            const float* reg_w, const float* reg_b, const int64_t* prop_type, const int64_t* target,
                            const float* reg_target, float* raw_act, float* raw_comp, float* raw_reg, float* losses,
                            float* d_course_ft, float* d_stpp_ft, float* d_act_w, float* d_act_b, float* d_comp_w,
                            float* d_comp_b, float* d_reg_w, float* d_reg_b, void* workspace, void* stream);

/* ---- BinaryClassifier (TAG actionness) head + loss: classifier_fc (binary_model.py:231) + torch.nn.CrossEntropyLoss()
 *      (mean over rows, binary_train.py:135,162) + loss.backward() down to the segment-mean features ------------------------
 * x [n, in_dim] (the course features), w [K, in_dim], b [K], target int64 [n] -> logits [n,K], loss[1] = mean_i
 * (logsumexp(logits_i) - logits_i[target_i]), dx [n, in_dim], dw [K, in_dim], db [K] (overwritten).  Every gradient is
 * multiplied by loss_scale (1/world_size for data parallel; a power of two scales them exactly); the loss is not.
 * Two launches, no host synchronisation and no allocation (graph-capturable); deterministic: fixed-order reductions, no
 * floating-point atomics, so repeated calls are bitwise equal.  workspace: ssnb_classifier_ce_workspace_bytes(n, K) bytes.
 * 1 <= K <= 4096.  A target outside [0, K) is never used as an index: that row's loss is NaN, so the returned mean loss is
 * NaN, and the row contributes no gradient (torch raises instead; its ignore_index = -100 is not honoured here). */
size_t ssnb_classifier_ce_workspace_bytes(int n, int num_class);
int ssnb_classifier_ce_fwd_bwd(const float* x, const float* w, const float* b, const int64_t* target, int n, int in_dim,
                               int num_class, float loss_scale, float* logits, float* loss, float* dx, float* dw, float* db,
                               void* workspace, void* stream);

/* ---- detection post-processing of one video (eval_detection_results.py:91-183, ops/utils.py:38-40,56-82) --------------
 * rel_props [N,2] (start, end in [0,1]), act_scores [N,K+1], comp_scores [N,K], reg_scores [N,K,2] (already de-normalised,
 * ssn_test.py:89-92) ->  per class c: combined score softmax(act)[:,c+1] * exp(comp[:,c]), greedy temporal NMS at
 * nms_thresh in descending score order, then (regress != 0) the location regression of the survivors.
 * detections [K, N, 5] rows (t0, t1, score, loc, dur) in kept order, counts [K] int32; combined_ws: N*K floats of scratch.
 * N <= 8192.  act_scores == NULL: combined_ws already holds the [N,K] scores to rank by
 * (plain class-wise temporal_nms, ops/utils.py:56-82). */
int ssnb_detect_postprocess(const float* rel_props, const float* act_scores, const float* comp_scores, const float* reg_scores,
                            int n_props, int num_class, double nms_thresh, int regress, float* detections, int* counts,
                            float* combined_ws, void* stream);

/* ---- detection post-processing of many videos (eval_detection_results.py:91-145 gen_detection_results, all three branches;
 *      :153-183 class-wise temporal_nms (ops/utils.py:56-82) and perform_regression (:162-174)) -------------------------------
 * Video v owns proposal rows offsets[v] .. offsets[v+1]-1 of rel_props [sum N, 2], act [sum N, K+1], comp [sum N, K] and
 * reg [sum N, K, 2] (NULL: zeros, the script's reg_scores = None; the boxes are still regressed when `regress`).  Per mode:
 *   SSNB_DET_ALL   (:103-113)  softmax(act)[:, 1:] * exp(comp), every (proposal, class) pair;
 *   SSNB_DET_TOPK  (:114-129)  softmax(act[:, 1:]) * exp(comp), the top_k pairs of the video (all when N*K < top_k);
 *   SSNB_DET_CLS   (:130-145)  softmax(act)[:, 1:] * exp(comp) (softmax_before_filter) or act[:, 1:] * exp(comp), every
 *                              proposal of the n_sel classes cls_sel[v, :] (device int32 [V, n_sel], distinct, in [0, K);
 *                              others are ignored).
 * then per non-empty (video, class): temporal NMS at nms_thresh and (regress) the location regression.  Ranking: NaN first,
 * then descending score, equal scores by larger proposal index first (a stable ascending argsort reversed).
 * Slots: video v has S_v = N_v*K (all), min(top_k, N_v*K) (top_k) or N_v*n_sel (cls) of them, starting at slot0[v] =
 * S_0 + ... + S_{v-1}.  dets [sum S, 5] (t0, t1, score, loc, dur): video v's survivors from slot0[v] on, class by class in
 * ascending class order, each class in kept (descending score) order; counts [V, K] int32.  Slots past the survivors are
 * not written.  Optional traces (NULL: not written): combined [sum N, K] fp32 (the ranked scores) and sel [sum S] int32, the
 * selected pairs row * K + class (global row) of video v at slots slot0[v] .. slot0[v] + S_v - 1 in ranking order.
 * offsets (int64 [V+1], offsets[0] = 0, non-decreasing) are HOST memory; offsets_dev holds the same values on the device.
 * Kernels only: no host synchronisation, no allocation, no copy from host memory (graph-capturable).  sum N * K and the
 * slot total must fit in int32. */
enum { SSNB_DET_ALL = 0, SSNB_DET_TOPK = 1, SSNB_DET_CLS = 2 };
typedef struct {
  int32_t mode;                   /* SSNB_DET_ALL | SSNB_DET_TOPK | SSNB_DET_CLS */
  int32_t top_k;                  /* SSNB_DET_TOPK: >= 1 */
  int32_t n_sel;                  /* SSNB_DET_CLS: classes per video, 1..K */
  int32_t softmax_before_filter;  /* SSNB_DET_CLS: 1 = softmax(act)[:, 1:], 0 = act[:, 1:] */
  int32_t regress;                /* 0: --no_regression */
  int32_t reserved;
  double nms_thresh;              /* not NaN */
} ssnb_detect_batch_cfg;
/* 0 for arguments ssnb_detect_batch would reject */
size_t ssnb_detect_batch_workspace_bytes(const ssnb_detect_batch_cfg* cfg, int num_class, const int64_t* offsets, int n_videos);
int ssnb_detect_batch(const ssnb_detect_batch_cfg* cfg, const float* rel_props, const float* act, const float* comp, const float* reg,
                      int num_class, const int64_t* offsets, const int64_t* offsets_dev, int n_videos, const int32_t* cls_sel,
                      float* dets, int32_t* counts, float* combined, int32_t* sel, void* workspace, size_t workspace_bytes,
                      void* stream);

/* ---- detection AP (anet_toolkit/Evaluation/eval_detection.py:160-235 compute_average_precision_detection, utils.py:14-51
 *      interpolated_prec_rec / segment_iou), every class and tIoU threshold of eval_detection_results.py:216-237 in one call --
 * Detections: ssnb_detect_batch's output for V videos (dets, counts [V, K], det_slot0 = device int64 [V+1], slot0[V] =
 * n_slots).  Ground truth: n_gt rows of gt_cls int32 and gt_seg double [n_gt, 2] (t0, t1), packed per video: video v's rows
 * are gt_offsets[v] .. gt_offsets[v+1]-1 (device int64 [V+1]); rows gt_offsets[V] .. n_gt-1 are ground truth of videos
 * without detections, counted in npos only.  Classes outside [0, K) are ignored.  Per class: predictions sorted by
 * descending score over all videos (NaN first; equal scores: the later (video, kept position) first); each is matched to
 * the unlocked ground truth of its own video and class with the highest double tIoU not below the threshold (a NaN tIoU,
 * from two zero-length segments, ranks first and matches; equal tIoU: larger ground-truth index first); precision and
 * recall from the cumulative counts, ap = the interpolated sum.  No ground truth and >= 1 prediction: NaN; no prediction: 0.
 * thresholds: host double [n_thr], 1..64.  ap: device double [K, n_thr].  Optional traces: rank [n_slots] int32 (a
 * survivor's position in its class-wide order), tp [n_thr, n_slots] uint8 (1 = true positive, 0 = false positive), both
 * written at survivor slots only.  Kernels only (graph-capturable), no host synchronisation, allocation or host copy. */
size_t ssnb_detection_ap_workspace_bytes(int n_videos, int num_class, int64_t n_slots, int64_t n_gt, int n_thresholds);
int ssnb_detection_ap(const float* dets, const int32_t* counts, const int64_t* det_slot0, int n_videos, int num_class, int64_t n_slots,
                      const int64_t* gt_offsets, const int32_t* gt_cls, const double* gt_seg, int64_t n_gt, const double* thresholds,
                      int n_thresholds, double* ap, int32_t* rank, uint8_t* tp, void* workspace, size_t workspace_bytes, void* stream);

/* ---- TAG bottom-up proposals of many videos (gen_bottom_up_proposals.py:116-142, ops/sequence_funcs.py:11-34,71-136) ----
 * Per video v with T_v = offsets[v+1] - offsets[v] ticks of the merged crop-mean score f_score [T_v, num_cols] (rows
 * offsets[v] .. offsets[v+1]-1 of one packed fp32 [offsets[V], num_cols] array): softmax (ops/metrics.py:8-11), column
 * cls + 1, scipy.ndimage.gaussian_filter(col, sigma) (truncate 4, 'reflect', double, rounded to fp32), labels col > fp32(thr)
 * per threshold, build_box_by_search per (threshold, tolerance) with box scores summed left to right in fp32 over the raw
 * column f_score[:, cls+1], temporal_nms_fallback(boxes, nms_thresh) with tied scores kept in search order, then seconds
 * (start / T * duration, end / T * duration, double) and the filter t1 - t0 > minimum_len.
 * Box slots: a video has at most n_thresholds * n_tolerances * (T_v + 1) boxes; its outputs start at slot
 * n_thresholds * n_tolerances * (offsets[v] + v), so every per-slot array below holds
 * n_thresholds * n_tolerances * (offsets[V] + V) entries (<= INT_MAX; split larger batches).
 *   frames [slots, 2] int32 (start, end frame), scores [slots] fp32, seconds [slots, 2] double: the kept boxes of video v in
 *   NMS order, counts[v] of them.  Optional (NULL: not written): smoothed [offsets[V]] fp32 (the softmax column when sigma is
 *   0), labels [offsets[V]] uint32 (bit k: threshold k), raw_frames [slots, 2] / raw_scores [slots] the boxes before NMS in the
 *   reference's order, raw_counts [V].
 * offsets (int64 [V+1], offsets[0] = 0, strictly increasing) and the config's threshold / tolerance arrays are HOST memory:
 * they are validated and size the call.  offsets_dev (the same V+1 values) and durations_dev (double [V], seconds) are device
 * memory, as is everything else.  The call enqueues kernels only: no host synchronisation, no allocation, no copy from host
 * memory, so it can be captured in a CUDA graph. */
typedef struct {
  int32_t cls;               /* foreground column cls + 1 (gen_prop: 0) */
  int32_t n_thresholds;      /* 1..32 */
  int32_t n_tolerances;      /* 1..32 */
  int32_t reserved;
  double sigma;              /* Gaussian bandwidth (gen_prop: 3); 0 = no smoothing (bw=None); radius int(4 sigma + 0.5) <= 63 */
  double nms_thresh;         /* [0, 1) (gen_prop: 0.9) */
  double minimum_len;        /* seconds (--minimum_len, default 0) */
  const double* thresholds;  /* host [n_thresholds] */
  const double* tolerances;  /* host [n_tolerances] */
} ssnb_tag_proposals_cfg;
/* 0 for arguments ssnb_tag_proposals would reject */
size_t ssnb_tag_proposals_workspace_bytes(int n_videos, int64_t total_ticks, int n_thresholds, int n_tolerances);
int ssnb_tag_proposals(const ssnb_tag_proposals_cfg* cfg, const float* f_score, int num_cols, const int64_t* offsets,
                       const int64_t* offsets_dev, int n_videos, const double* durations_dev, int32_t* frames, float* scores, double* seconds, int32_t* counts, float* smoothed,
                       uint32_t* labels, int32_t* raw_frames, float* raw_scores, int32_t* raw_counts, void* workspace,
                       size_t workspace_bytes, void* stream);

/* ---- proposal lists: labelling proposals against ground truth, recall, sliding windows, frame windows, the SSN data set's
 *      training targets and test-time proposal inputs, many ragged videos per call (csrc/proposal_lists.cu) ------------------
 * Packed layout shared by the calls below.  Proposals: boxes double [rows, 2] (start, end) with device first int64 [V] and
 * count int32 [V]: video v owns rows first[v] .. first[v] + count[v] - 1.  That is the seconds / slot0 / counts of
 * ssnb_tag_proposals read in place; a compact [sum N, 2] array is the case first = exclusive cumsum of count.  Per-row
 * outputs are written at the row's own index; rows outside every video are not touched.  Ground truth: gt double [sum G, 2],
 * gt_label int32 [sum G], video v's rows gt_offsets[v] .. gt_offsets[v+1]-1 (int64 [V+1], gt_offsets[0] = 0, ascending;
 * HOST memory, validated; gt_offsets_dev is the device copy the kernels read).  max_count: a bound of count[v] known to the
 * host that sizes the grid only -- any value >= 0 gives the same result.  No cap on N_v or G_v; V = 0, N_v = 0 and G_v = 0
 * are valid.  Every call enqueues kernels and memsets only: no host synchronisation, allocation or host copy, so it can be
 * captured in a CUDA graph.
 *
 * ssnb_name_proposals: name_proposal (ops/detection_metrics.py:54-76) of every proposal: label = gt_label + 1, max_overlap =
 * temporal_iou (:7-20), overlap_self = overlap_over_b (:23-28) of the ground truth selected by `ov > thresh and ov >
 * max_overlap` in ground-truth order (the first of equal overlaps; NaN never); 0 / 0 / 0 when none.  Bitwise the reference's
 * doubles (Python min / max, one IEEE division).  gt_best double [sum G]: per ground truth the maximum tIoU over its video's
 * proposals (0 without an overlapping one; NaN overlaps ignored), which answers temporal_recall (:31-51) at every threshold. */
int ssnb_name_proposals(const double* boxes, const int64_t* first, const int32_t* count, int n_videos, int64_t max_count, const double* gt,
                        const int32_t* gt_label, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, double thresh, int32_t* label,
                        double* max_overlap, double* overlap_self, double* gt_best, void* stream);
/* get_temporal_proposal_recall (ops/detection_metrics.py:79-83) for n_thresholds (1..32, HOST) thresholds at once: hits int32
 * [V, n_thresholds] = ground truth of video v with gt_best > threshold; totals int64 [2 * n_thresholds + 1] = per threshold
 * the videos with hits == G_v (G_v = 0 counts, as 0 == 0 does), then per threshold the sum of hits, then sum G. */
int ssnb_proposal_recall(const double* gt_best, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, int n_videos, const double* thresholds,
                         int n_thresholds, int32_t* hits, int64_t* totals, void* stream);
/* gen_exponential_sw_proposal (ops/sequence_funcs.py:37-54) for V durations (device double [V]).  Level l (1..32 levels; HOST
 * arrays): boxes (k * steps[l], k * steps[l] + t_spans[l]) for k * steps[l] < duration, kept when min(duration, end) - start
 * >= 1; level-major, start ascending.  steps[l] = int(ceil(t_spans[l] * time_step * (1 - overlap))) is the caller's (an integer
 * >= 1); the end uses t_span, not the span in seconds, as the reference does.  A duration that is not positive and finite has
 * no windows.  Writes count [V], first [V] (exclusive cumsum), level_count int32 [V, n_levels], total int64 [1], and the boxes
 * double [capacity, 2] (rows at or past capacity are dropped: compare total; capacity 0 only counts). */
int ssnb_sliding_windows(const double* durations, int n_videos, const double* t_spans, const double* steps, int n_levels, int64_t max_count,
                         int64_t capacity, double* boxes, int64_t* first, int32_t* count, int32_t* level_count, int64_t* total, void* stream);
/* Frame windows.  SECONDS: dump_window_list (ops/io.py:109-127), int(x * real_fps) with real_fps = float(frame_cnt) /
 * float(duration); NORMALISED: process_proposal_list (ops/io.py:44-47), int(float(x) * frame_cnt); AS_GIVEN: x holds frame
 * integers already (a parsed list).  int() truncates toward zero; a product outside int64 saturates and NaN gives 0 (the
 * reference raises).  frames int64 [rows, 2]: what the list file holds.  Optional (NULL: not written), SSNVideoRecord's rules
 * (ssn_dataset.py:13-21,81-93): keep uint8 = end > start and start < frame_cnt; valid int64 [rows, 2] = (start, min(end,
 * frame_cnt)); coverage double = (end - start) / frame_cnt with the unclipped end.  Ground truth goes through the same call
 * with first = gt_offsets[:-1] and count = their differences. */
enum { SSNB_PROPFRAMES_SECONDS = 0, SSNB_PROPFRAMES_NORMALISED = 1, SSNB_PROPFRAMES_AS_GIVEN = 2 };
int ssnb_proposal_frames(const double* boxes, const int64_t* first, const int32_t* count, int n_videos, int64_t max_count, const double* durations,
                         const int32_t* frame_cnt, int mode, int64_t* frames, int64_t* valid, double* coverage, uint8_t* keep, void* stream);
/* What SSNDataSet._parse_prop_file derives (ssn_dataset.py:29-55,103-131,196-227,382-391) from kept rows only (valid frames,
 * coverage, and best_iou / overlap_self as the caller chooses to pass them: the list's 4-decimal values or fresh ones):
 *   tags uint8 [rows]: SSNB_TAG_FG best_iou > fg_thresh; SSNB_TAG_INCOMPLETE best_iou < incomplete_iou_thresh and overlap_self >
 *     incomplete_overlap_thresh; SSNB_TAG_BACKGROUND not incomplete and best_iou < bg_iou_thresh and coverage >
 *     bg_coverage_thresh (a row may be fg and incomplete, as the reference's two lists may both hold it);
 *   reg double [rows, 2]: (loc_reg, size_reg) of every fg row against the first ground truth of maximum frame tIoU
 *     (ops/utils.py:40-53, np.argmax), (0, 0) elsewhere.  The reference computes targets for the members of the fg list only,
 *     so a row with best_iou == fg_thresh has none.  loc_reg is bitwise; size_reg is CUDA's double log;
 *   pool_counts int32 [V, 4]: fg, incomplete, background proposals and ground truth of the video; totals int64 [5]: their sums
 *     and the number of videos used; exclude_empty drops videos without ground truth from everything (tags 0), as the data
 *     set does.  Without exclude_empty an fg row of a video without ground truth gets (0, 0) (np.argmax raises there);
 *   stats double [4]: np.mean and np.std (population) of the fg rows' targets (mean loc, mean size, std loc, std size), summed
 *     per video and then over the videos in a fixed order (repeatable to the bit; NaN when there is no fg row).
 * gt_frames int64 [sum G, 2]: the kept ground truth's valid frames. */
enum { SSNB_TAG_FG = 1, SSNB_TAG_INCOMPLETE = 2, SSNB_TAG_BACKGROUND = 4 };
typedef struct {
  double fg_thresh;                 /* fg_iou_thresh (0.7) */
  double incomplete_iou_thresh;     /* 0.3 */
  double bg_iou_thresh;             /* 0.01 */
  double bg_coverage_thresh;        /* 0.02 */
  double incomplete_overlap_thresh; /* 0.7 */
  int32_t exclude_empty;            /* 1 */
  int32_t reserved;
} ssnb_proposal_targets_cfg;
size_t ssnb_proposal_targets_workspace_bytes(int n_videos);
int ssnb_proposal_targets(const ssnb_proposal_targets_cfg* cfg, const int64_t* frames, const double* best_iou, const double* overlap_self,
                          const double* coverage, const int64_t* first, const int32_t* count, int n_videos, const int64_t* gt_frames,
                          const int64_t* gt_offsets, const int64_t* gt_offsets_dev, uint8_t* tags, double* reg, int32_t* pool_counts,
                          int64_t* totals, double* stats, void* workspace, size_t workspace_bytes, void* stream);
/* get_test_data's proposal half (ssn_dataset.py:393-428) from kept rows' valid frames.  num_ticks int32 [V] =
 * len(np.arange(0, frame_cnt - new_length, test_interval)).  Video v's output rows start at out_first[v] (device int64 [V];
 * a video without proposals owns one row, the reference's fallback proposal (0, frame_cnt - 1), so out_first is the exclusive
 * cumsum of max(count, 1)): rel_prop double [rows, 2], ticks int64 [rows, 4], scaling double [rows, 2], bitwise the
 * reference's, each operation rounded on its own.  Optional ticks32 int32 [rows, 4] / scaling32 float [rows, 2]: the same
 * values in the types ssnb_stpp_reorg_prefix takes.  A zero-length fallback (frame_cnt 1) divides by zero
 * where the reference raises. */
int ssnb_test_proposals(const int64_t* frames, const int64_t* first, const int32_t* count, const int64_t* out_first, int n_videos,
                        int64_t max_count, const int32_t* frame_cnt, int new_length, int test_interval, int32_t* num_ticks, double* rel_prop,
                        int64_t* ticks, double* scaling, int32_t* ticks32, float* scaling32, void* stream);

/* ---- ActivityNet proposal evaluation: average recall against the average number of proposals per video (AR-AN) of
 *      anet_toolkit/Evaluation/eval_proposal.py:158-273 (segment_iou, utils.py:25-75), every video and threshold in one call
 *      (csrc/proposal_ar.cu) ------------------------------------------------------------------------------------------------
 * Proposals in the packed layout above: boxes double [rows, 2] (t0, t1) and scores double [rows], video v's rows first[v] ..
 * first[v] + count[v] - 1 (device int64 / int32 [n_videos]).  Ground truth gt_seg double [sum G, 2], video v's instances
 * gt_offsets[v] .. gt_offsets[v+1]-1 (int64 [n_videos + 1], HOST memory, validated; gt_offsets_dev is the device copy).  The
 * evaluated videos are those with G_v > 0, in packed order (V of them); a video with G_v = 0 adds its count to P_all only,
 * which is how proposals of videos outside the ground truth are passed.  Per evaluated video: the proposals ranked by the
 * toolkit's score.argsort()[::-1] (NaN first, then descending score with -0 == +0, ties by descending row), the first
 * nr_v = min(int(P_v * ratio), P_v) kept, ratio = max_avg * V / P_all in double, max_avg <= 0 meaning P_all / V; a video
 * without proposals has one phantom column of tIoU 0.0.  tIoU is segment_iou with NaN-propagating max / min / clip (a 0 / 0
 * union is NaN and matches nothing); an instance is matched at (t, j) when one of the first min(int(P'_v * pcn_j), P'_v)
 * columns has tIoU >= thresholds[t], pcn_j = (j / 100.0) * (max_avg * V / total_nr), j = 1..100.
 * thresholds: HOST double [n_thresholds], 1..64, not NaN; max_avg finite.  Outputs (device): recall double [n_thr, 100],
 * avg_recall double [100] (recall summed over the thresholds in order, then / n_thr), proposals_per_video double [100]
 * (pcn_j * (total_nr / V)), total_nr int64 [1]; all bitwise the toolkit's.  total_nr == 0 (the toolkit divides by zero):
 * the three curves are NaN.  Optional traces (NULL: kept in the workspace): nr int32 [n_videos] (nr_v, 0 for videos without
 * ground truth or proposals) and first_hit int32 [sum G, n_thr] (the first column with tIoU >= threshold, INT_MAX: none).
 * rows <= INT_MAX and sum G <= INT_MAX / 64.  Kernels and memsets only: no host synchronisation, allocation or host copy, so
 * the call can be captured in a CUDA graph.  The workspace (about 24 bytes per row plus 4 (n_thr + 1) per instance) is 0 for
 * arguments ssnb_proposal_ar would reject. */
size_t ssnb_proposal_ar_workspace_bytes(int n_videos, int64_t rows, const int64_t* gt_offsets, int n_thresholds);
int ssnb_proposal_ar(const double* boxes, const double* scores, int64_t rows, const int64_t* first, const int32_t* count, int n_videos,
                     const double* gt_seg, const int64_t* gt_offsets, const int64_t* gt_offsets_dev, const double* thresholds,
                     int n_thresholds, double max_avg, double* recall, double* avg_recall, double* proposals_per_video,
                     int64_t* total_nr, int32_t* nr, int32_t* first_hit, void* workspace, size_t workspace_bytes, void* stream);

/* ---- ActivityNet untrimmed video classification: per-class average precision and video hit@k of
 *      anet_toolkit/Evaluation/eval_classification.py:124-249 (and eval_kinetics.py, the same code), every class and video in
 *      one call (csrc/classification_ap.cu) -----------------------------------------------------------------------------
 * Predictions: rows of video int32, label int32 and score double (device [rows]).  Ground truth: n_gt (video, label) pairs
 * gt_video / gt_label int32 (device [n_gt]); repeated pairs count once (drop_duplicates).  Videos are 0..n_videos-1, classes
 * 0..num_class-1; a row or pair outside them is ignored.  Ranking: the toolkit's score.argsort()[::-1] -- NaN first, then
 * descending score (-0 == +0), equal scores the later row first -- over a class's rows for AP and over a video's rows for
 * hit@k.  Per class c: a row is a true positive when (its video, c) is ground truth and no higher-ranked row of c has the
 * same video, else a false positive; npos = distinct ground-truth videos of c; ap[c] = interpolated_prec_rec of cumsum(tp) /
 * npos and tp / (tp + fp) (no row: 0; rows but npos = 0: NaN).  Per video v with ground truth: hits[v] = its distinct
 * ground-truth labels found among its top_k ranked rows (a duplicate row takes a place); hit_at_k = the fraction of these
 * videos with hits > 0 (exact), avg_hit_at_k = the mean of hits[v] / labels[v] (summed in a fixed order; NaN without a
 * ground-truth video).  num_class 1..1024, num_class * n_videos < INT_MAX, rows and n_gt < INT_MAX, top_k >= 1.
 * Outputs (device): ap double [num_class], hit_at_k double [1], avg_hit_at_k double [1].  Optional traces (NULL: not
 * written): hits int32 [n_videos], gt_labels int32 [n_videos] (distinct ground-truth labels per video), tp uint8 [rows] (1:
 * the row is a true positive).  Kernels, memsets and device copies only: no host synchronisation, allocation or host copy, so
 * the call can be captured in a CUDA graph.  The workspace (about 70 bytes per row, 8 per pair, 12 per video and class) is 0
 * for arguments ssnb_classification_ap would reject. */
size_t ssnb_classification_ap_workspace_bytes(int64_t rows, int64_t n_gt, int n_videos, int num_class);
int ssnb_classification_ap(const int32_t* video, const int32_t* label, const double* score, int64_t rows, const int32_t* gt_video,
                           const int32_t* gt_label, int64_t n_gt, int n_videos, int num_class, int top_k, double* ap, double* hit_at_k,
                           double* avg_hit_at_k, int32_t* hits, int32_t* gt_labels, uint8_t* tp, void* workspace, size_t workspace_bytes,
                           void* stream);

/* ---- video-level classification from snippet scores: the aggregation and fusion functions of the reference's
 *      ops/video_funcs.py and the metrics of ops/metrics.py, many ragged videos per call (csrc/video_agg.cu) --------------
 * Scores: packed fp32 [sum T, crops, D] (device), video v's ticks at tick_offsets[v] .. tick_offsets[v+1] (int64 [V+1], [0] = 0,
 * every video at least one tick).  tick_offsets is HOST memory: validated, it sizes the call; tick_offsets_dev holds the same
 * values on the device.  Modes and their output out [V, K] (device):
 *   SSNB_VAGG_DEFAULT  default_aggregation_func (:8-18): crop reduction, mean over ticks                  fp32, K = D
 *   SSNB_VAGG_TOP_K    top_k_aggregation_func (:21-26): crop reduction, mean of the top_k largest ticks   fp32, K = D
 *                      per class (all T when top_k > T)
 *   SSNB_VAGG_SLIDING  sliding_window_aggregation_func (:29-57): crop MEAN; per span s (spans[i] * fps ticks) the maxima of  fp32, K = D
 *                      the windows [i, i + s) clipped at T, i in range(0, T, ceil(s * (1 - overlap))); the mean of their
 *                      max(15, n_windows // 4) largest; the mean over spans
 *   SSNB_VAGG_TPP      tpp_aggregation_func (:60-70): crop mean; tick t adds its stage int(t * (stage / T)) of the       float64, K = num_class
 *                      D = stage * num_class columns, in float64 from 0; divided by T
 * crop_agg: SSNB_CROP_MEAN or SSNB_CROP_MAX (default and top-k only); normalize (not tpp): metrics.softmax of each output row.
 * The fp32 sums run in numpy's order (crops, then ticks, then the top k from the k-th largest up, then spans, each from its
 * first term; the softmax denominator by numpy's pairwise rule) and every fp32 operation is rounded on its own, so only the
 * softmax's expf differs from numpy (a few ulp).  NaN propagates as numpy's max and sort put it; top-k and sliding-window
 * take at most 32768 ticks per video.  Workspace (ssnb_video_aggregate_workspace_bytes; 0 for arguments the call rejects):
 * 4 sum T * D bytes for top-k and sliding window, 1 otherwise.  Bad arguments are refused before any launch; kernels only: no
 * host synchronisation, allocation or copy (graph-capturable). */
enum { SSNB_VAGG_DEFAULT = 0, SSNB_VAGG_TOP_K = 1, SSNB_VAGG_SLIDING = 2, SSNB_VAGG_TPP = 3 };
enum { SSNB_CROP_MEAN = 0, SSNB_CROP_MAX = 1 };
size_t ssnb_video_aggregate_workspace_bytes(const int64_t* tick_offsets, int n_videos, int crops, int D, int mode, int crop_agg, int top_k,
                                            const int32_t* spans, int n_spans, double overlap, int fps, int num_class);
int ssnb_video_aggregate(const float* scores, const int64_t* tick_offsets, const int64_t* tick_offsets_dev, int n_videos, int crops, int D,
                         int mode, int crop_agg, int normalize, int top_k, const int32_t* spans, int n_spans, double overlap, int fps,
                         int num_class, void* out, void* workspace, size_t workspace_bytes, void* stream);
/* default_fusion_func (:73-80) over rows x num_class fp32 streams (device): out = major, then out += others[i] * (float)weights[i]
 * in stream order (each product and sum rounded to fp32, numpy's rule for a Python float weight), then with normalize the
 * softmax exp((x - max) * temperature) / sum of each row (metrics.softmax; temperature 1 for the fusion).  others and weights
 * are HOST arrays of at most 8; out may be major.  Kernels only (graph-capturable). */
int ssnb_video_fuse(const float* major, const float* const* others, const double* weights, int n_others, int64_t rows, int num_class,
                    int normalize, double temperature, float* out, void* stream);
/* metrics.py over video scores [V, K] (device, fp32, or float64 with scores_f64) and the (label_video, label) pairs (device
 * int32 [n_labels]; repeated pairs count once, pairs outside 0..V-1 / 0..K-1 are ignored).  Each video's classes are ranked by
 * descending score with NaN first (rank_key.cuh) and equal scores the HIGHER class first (a stable ascending argsort's
 * [-k:]); top_k_idx (optional, int32 [V, min(top_k, K)]) is that ranking's head, best first.  hits[v] = labels of v among
 * them, label_count[v] = distinct labels of v (top_k_acc); top_k_accuracy = videos with a hit / V (top_k_accuracy).  ap [K]:
 * sklearn's average_precision_score per class (the step AP over distinct thresholds; 0 for a class without a positive);
 * mean_ap = their mean (video_mean_ap, average='macro').  class_label (optional, int32 [V]) gives mean_class_accuracy:
 * np.argmax per video (the first NaN, else the first maximum), confusion (optional, int32 [3, K]: label counts, prediction
 * counts, hits) and the mean of hits / label count over the classes labelled or predicted (NaN when one is never labelled, or
 * without class_label).  V >= 1, K in 1..1024, V * K < INT_MAX, top_k >= 1.  Kernels, memsets and device copies only
 * (graph-capturable); workspace about 25 bytes per (video, class). */
size_t ssnb_video_metrics_workspace_bytes(int n_videos, int num_class);
int ssnb_video_metrics(const void* scores, int scores_f64, int n_videos, int num_class, const int32_t* label_video, const int32_t* label,
                       int64_t n_labels, const int32_t* class_label, int top_k, int32_t* hits, int32_t* label_count, int32_t* top_k_idx,
                       double* top_k_accuracy, double* ap, double* mean_ap, int32_t* confusion, double* mean_class_accuracy,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- frame transforms: the PIL group transforms of the data pipeline (transforms.py:41-206) followed by Stack(roll=True),
 *      ToTorchFormatTensor(div=False) and GroupNormalize (transforms.py:67-80,256-288), bitwise equal to PIL 8-bit BILINEAR --
 * Modes (cfg->mode):
 *   SSNB_FRAMES_TRAIN       GroupMultiScaleCrop (:135-206) + GroupRandomHorizontalFlip (:49-64) with the crop window and flip
 *                           drawn on the host: each group's images are cropped to (crop_x, crop_y, crop_w, crop_h) and resized
 *                           to out_size x out_size (get_augmentation, ssn_models.py; ssn_train.py:106-117)
 *   SSNB_FRAMES_OVERSAMPLE  GroupOverSample(out_size, scale_size) (:99-132): GroupScale then the five fill_fix_offset(False)
 *                           windows, each window's images plain then flipped (ssn_test.py / binary_test.py --test_crops 10)
 *   SSNB_FRAMES_CENTER      GroupScale(scale_size) + GroupCenterCrop(out_size) (:41-46,83-96; ssn_test.py:107-110, val_loader)
 * GroupScale is torchvision Resize of the shorter edge to scale_size (long = int(scale_size * long / short)); it is skipped when
 * the shorter edge already equals scale_size.  A window that reaches outside the image reads zeros, as PIL's crop fills.
 * Group g's images are src[src_offset ..] as uint8 [images, height, width, channels] (RGB or L).  Output: fp32 planes
 * [out_size, out_size] from dst + dst_offset, plane ((crop * images + image) * channels + c) with c in BGR order for RGB,
 * crop 0..9 (OVERSAMPLE: window crop / 2, flipped when odd) or 0; value (v - mean[p % n_mean]) / std[p % n_mean] in fp32,
 * p the plane index within the group.  A flipped image at an even position of its group becomes 255 - v when invert_even
 * is set (Flow, transforms.py:59-61,125-126).
 * ssnb_frame_transform_workspace_bytes validates cfg and the HOST table, fills in each group's first_image, dst_offset and
 * scratch_offset, and returns the workspace size and the floats dst must hold.  ssnb_frame_transform takes that host table
 * (validated again, it sizes the launch) and groups_dev, a device copy of it that the kernels read: kernels only, no host
 * synchronisation, allocation or host copy, so the call can be captured in a CUDA graph and replayed after new frames and
 * new crop windows / flips are written to src and groups_dev (height, width, images and the layout fields must stay). */
enum { SSNB_FRAMES_TRAIN = 0, SSNB_FRAMES_OVERSAMPLE = 1, SSNB_FRAMES_CENTER = 2 };
typedef struct {
  int32_t mode;         /* SSNB_FRAMES_TRAIN | SSNB_FRAMES_OVERSAMPLE | SSNB_FRAMES_CENTER */
  int32_t channels;     /* 3 (RGB, written BGR) or 1 (L: Flow x / y planes) */
  int32_t out_size;     /* crop size, 1..1024 (224) */
  int32_t scale_size;   /* OVERSAMPLE / CENTER: GroupScale's shorter edge, out_size..4096 (256) */
  int32_t invert_even;  /* 1: Flow */
  int32_t n_mean;       /* 1..8 entries of mean / std, cycled over the stacked planes; images * channels % n_mean == 0 */
  float mean[8];
  float std[8];
} ssnb_frame_cfg;
typedef struct {
  int64_t src_offset;      /* bytes */
  int64_t dst_offset;      /* floats; filled in by ssnb_frame_transform_workspace_bytes */
  int64_t scratch_offset;  /* workspace bytes of the GroupScale output; filled in likewise */
  int32_t first_image;     /* images of the groups before this one; filled in likewise */
  int32_t height, width;   /* 1..16384 */
  int32_t images;          /* >= 1 */
  int32_t crop_x, crop_y;  /* TRAIN: window offset (may be negative), |.| <= 16384 */
  int32_t crop_w, crop_h;  /* TRAIN: window size, 1..16 * out_size */
  int32_t flip;            /* TRAIN: 1 = GroupRandomHorizontalFlip flipped this group */
  int32_t reserved;
} ssnb_frame_group;
int ssnb_frame_transform_workspace_bytes(const ssnb_frame_cfg* cfg, ssnb_frame_group* groups, int n_groups, size_t* workspace_bytes,
                                         int64_t* dst_floats);
int ssnb_frame_transform(const ssnb_frame_cfg* cfg, const ssnb_frame_group* groups, const ssnb_frame_group* groups_dev, int n_groups,
                         const uint8_t* src, size_t src_bytes, float* dst, int64_t dst_floats, void* workspace, size_t workspace_bytes,
                         void* stream);

/* ---- JPEG decode: the frame loading of the data sets, Image.open(path).convert('RGB') for RGB frames and .convert('L') for
 * the x / y planes of Flow (SSNDataSet._load_image, ssn_dataset.py:187-194; BinaryDataSet._load_image,
 * load_binary_score.py:198-205), bitwise equal to Pillow over libjpeg-turbo.  Huffman-coded sequential 8-bit JPEG (SOF0 /
 * SOF1), grayscale or YCbCr with luma sampling 1x1, 2x1 or 2x2 over 1x1 chroma, any size, restart intervals; the islow IDCT,
 * fancy upsampling, libjpeg's YCbCr -> RGB tables and PIL's RGB -> L.
 *
 * ssnb_jpeg_plan_create parses every image of a call from HOST bytes into one table: geometry, dequantisation and expanded
 * Huffman tables (identical tables are stored once), restart intervals with their byte ranges, the output offsets.  A stream
 * the decoder does not support (progressive, lossless, hierarchical, arithmetic-coded, 12-bit, CMYK / YCCK, Adobe RGB, other
 * sampling factors, multi-scan) is refused with SSNB_ENOSUPPORT, a malformed or truncated header or a scan that references an
 * undefined table with SSNB_EINVAL; *bad_image gets the image's index and ssnb_last_error(NULL) "jpeg: image i: reason".
 * Nothing is launched.
 * ssnb_jpeg_plan_write_table writes the plan's device table (table_bytes) to host memory; the caller copies it to the device
 * together with the bytes.  ssnb_jpeg_decode then only enqueues: a memset of status, the entropy decode (one thread per restart
 * interval), the IDCT of every block and the upsampling / colour conversion into out: image i is uint8 [height, width,
 * channels] at info.out_offset, images back to back in call order.  src_dev holds the call's bytes at the offsets the plan was
 * made with.  status int32 [n]: 0, or the largest SSNB_JPEG_* code of a corrupt entropy-coded segment of that image; the bit
 * reader never reads outside an image's segment and every other image of the call decodes as if alone. */
typedef struct {
  int64_t offset;          /* the image's first byte in src */
  int64_t bytes;
  int32_t channels;        /* 3: convert('RGB'), 1: convert('L') */
  int32_t reserved;
} ssnb_jpeg_input;
typedef struct {
  int32_t width, height;
  int32_t components;      /* 1 grayscale, 3 YCbCr */
  int32_t h_samp, v_samp;  /* luma sampling over 1x1 chroma (1, 1 for grayscale) */
  int32_t channels;
  int32_t restart_interval, intervals;  /* MCUs per interval (0: none), intervals of the scan */
  int64_t scan_offset, scan_bytes;      /* the entropy-coded segment in src */
  int64_t out_offset;                   /* first output byte */
} ssnb_jpeg_image_info;
enum { SSNB_JPEG_OK = 0, SSNB_JPEG_TRUNCATED = 1, SSNB_JPEG_BAD_CODE = 2, SSNB_JPEG_BAD_RUN = 3, SSNB_JPEG_BAD_RESTART = 4 };
typedef struct ssnb_jpeg_plan_s* ssnb_jpeg_plan;
int ssnb_jpeg_plan_create(const uint8_t* src, size_t src_bytes, const ssnb_jpeg_input* images, int n, ssnb_jpeg_plan* plan,
                          int* bad_image);
int ssnb_jpeg_plan_destroy(ssnb_jpeg_plan plan);
int ssnb_jpeg_plan_sizes(ssnb_jpeg_plan plan, size_t* table_bytes, size_t* workspace_bytes, int64_t* out_bytes);
int ssnb_jpeg_plan_image(ssnb_jpeg_plan plan, int i, ssnb_jpeg_image_info* info);
int ssnb_jpeg_plan_write_table(ssnb_jpeg_plan plan, void* dst, size_t dst_bytes);
int ssnb_jpeg_decode(ssnb_jpeg_plan plan, const void* table_dev, const uint8_t* src_dev, size_t src_bytes, uint8_t* out, int64_t out_bytes,
                     int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---- InceptionV3 backbone at test time: replaces model_zoo.InceptionV3 (pytorch_load.py:64-67, inceptionv3.yaml) as used by
 *      SSN.test_forward and BinaryClassifier scoring with --arch InceptionV3 (ssn_models.py:133-139, binary_model.py:175-178) ----
 * Forward only, frozen BatchNorm folded into each convolution, in every precision: EXACT_FP32 (fp32 SIMT convolutions),
 * FAST_FP16 and EXACT_TC (every convolution on the wgmma kernel; EXACT_TC with split operands, an fp32 epilogue and the
 * output's operand planes).  Planned and run by the same host-side graph core as the BNInception engine, under a handle of
 * its own: the BNInception functions above do not take it, and errors are read with ssnb_last_error(NULL).  Creation only plans (no device call), so the plan can be inspected without a
 * GPU.  Activations are NHWC fp32; the branch ends of every inception block are channel slices of the block's concat buffer
 * ("<block>_join"), so no concat runs; each value has a buffer of its own (no reuse across the pass). */
typedef struct ssnb_iv3* ssnb_iv3_handle;
typedef struct {
  int32_t in_channels; /* 3 (RGB) or 10 (Flow 2x5) */
  int32_t frames;      /* F images per call, >= 1 */
  int32_t precision;   /* SSNB_EXACT_FP32 | SSNB_FAST_FP16 | SSNB_EXACT_TC */
  int32_t reserved;
} ssnb_iv3_config;
/* the 94 convolutions in graph order; name is the yaml's blob (conv id "<name>_Conv2D", BatchNorm id "<name>_batchnorm") */
int ssnb_iv3_num_convs(void);
int ssnb_iv3_conv_info(int idx, int in_channels, char* name, int name_cap, int* cin, int* cout, int* kh, int* kw, int* stride, int* pad_h,
                       int* pad_w);
int ssnb_iv3_create(const ssnb_iv3_config* cfg, ssnb_iv3_handle* out);
int ssnb_iv3_destroy(ssnb_iv3_handle h);
size_t ssnb_iv3_workspace_bytes(ssnb_iv3_handle h);
/* dev_ptr 1024-byte aligned, at least ssnb_iv3_workspace_bytes; packed weights must be set again afterwards */
int ssnb_iv3_set_workspace(ssnb_iv3_handle h, void* dev_ptr, size_t bytes);
/* arrays of 94 device pointers in graph order, reference shapes: w [cout, cin, kh, kw], b / gamma / beta / mean / var [cout]
 * (BatchNorm eps 1e-5).  Call again whenever a parameter changes. */
int ssnb_iv3_pack_weights(ssnb_iv3_handle h, const float* const* w, const float* const* b, const float* const* gamma,
                          const float* const* beta, const float* const* mean, const float* const* var, void* stream);
/* input [F, C, 299, 299] fp32 NCHW -> feat [F, 2048] fp32 (top_cls_pool, the 8x8 average pool; top_cls_fc is replaced by
 * Identity / Dropout) */
int ssnb_iv3_forward(ssnb_iv3_handle h, const float* input_nchw, float* feat, void* stream);
/* the same forward over the first `frames` frames, 1 <= frames <= F (SSNB_EINVAL otherwise, before any launch): input
 * [frames, C, 299, 299] -> feat [frames, 2048], rows bitwise those of an engine planned for `frames`, with that many frames'
 * launches on this engine's workspace; graph-capturable.  frames == F is ssnb_iv3_forward. */
int ssnb_iv3_forward_frames(ssnb_iv3_handle h, const float* input_nchw, int frames, float* feat, void* stream);
/* introspection for the plan and the launch-by-launch tests: op kinds "conv" | "maxpool" | "avgpool" | "gpool", the names of the
 * values an op reads and writes (the yaml's blob names; the last op writes "top_cls_global_pool", the feat output), its
 * convolution index (-1 for pools) and a pool's window, stride and pad (0 / 1 / 0 for convolutions).  A value's shape, its buffer and its channel offset in that buffer. */
int ssnb_iv3_num_ops(ssnb_iv3_handle h);
int ssnb_iv3_op_info(ssnb_iv3_handle h, int op, char* kind, int kind_cap, char* in_name, int in_cap, char* out_name, int out_cap, int* conv,
                     int* k, int* stride, int* pad);
int ssnb_iv3_value_info(ssnb_iv3_handle h, const char* name, int* c, int* hh, int* ww, char* buffer, int buffer_cap, int* coff);
/* NCHW fp32 [F, C, H, W] copies in and out of a value (FAST: of its fp16 storage; EXACT_TC: a write also refreshes its operand
 * planes); planes = 1 (EXACT_TC only) reads hi + lo of the value's operand planes instead.  ssnb_iv3_run_op runs one op on
 * what the workspace holds (feat: the last op's output, else unused) */
int ssnb_iv3_value_write(ssnb_iv3_handle h, const char* name, const float* src_nchw, void* stream);
int ssnb_iv3_value_read(ssnb_iv3_handle h, const char* name, int planes, float* dst_nchw, void* stream);
int ssnb_iv3_run_op(ssnb_iv3_handle h, int op, float* feat, void* stream);

/* fused SGD-momentum step over flat fp32 buffers (ssn_train.py:141-144 torch.optim.SGD semantics), the whole model in ONE
 * launch: the flat buffers are cut into n_seg <= 512 segments (one per parameter tensor; seg_end = cumulative element ends,
 * device int64) with their parameter group's learning rate and weight decay (device fp32 arrays): the per-group lr_mult /
 * decay_mult of SSN.get_optim_policies (ssn_models.py:203-251) as applied by adjust_learning_rate (ssn_train.py:391-398).
 * Per element: g = grad*grad_mult + wd*p; buf = mom*buf + g; p -= lr*buf */
int ssnb_sgd_step_groups(float* param, const float* grad, float* momentum_buf, size_t n, const int64_t* seg_end,
                         const float* seg_lr, const float* seg_wd, int n_seg, float momentum, float grad_mult, void* stream);

/* ---- the rest of the training step between loss.backward() and optimizer.step(), and the loop's meters ----
 * All four calls are graph-capturable: they neither synchronise the host nor allocate, and every argument is checked
 * before any launch (SSNB_EINVAL).
 *
 * Extra gradients: tensors model.parameters() holds but no optimiser group does, so the flat buffers do not either (the
 * first BatchNorm2d's weight and bias under bn_mode='partial': get_optim_policies leaves them out, ssn_models.py:203-251,
 * while clip_grad_norm(model.parameters()) counts and scales them).  The struct is read on the host during the call. */
enum { SSNB_GRAD_NORM_CTAS = 512, SSNB_MAX_EXTRA_GRADS = 8 };
typedef struct {
  int32_t count;                        /* 0 .. SSNB_MAX_EXTRA_GRADS */
  int32_t reserved;
  float* grad[SSNB_MAX_EXTRA_GRADS];    /* device fp32, may be NULL where numel is 0 */
  int64_t numel[SSNB_MAX_EXTRA_GRADS];
} ssnb_extra_grads;
/* the total L2 norm of clip_grad_norm(model.parameters(), clip) (ssn_train.py:245-250, binary_train.py:192-197) after the
 * iter_size division (ssn_train.py:238-243, binary_train.py:185-190): norm = sqrt(sum (grad[i]*grad_mult)^2 + sum extra^2)
 * into the device fp32 scalar *norm.  The extras are not divided (the reference divides the optimiser groups only).  Two
 * deterministic stages: fp64 partials of a fixed grid of SSNB_GRAD_NORM_CTAS CTAs (independent of the SM count) into
 * `partials` (SSNB_GRAD_NORM_CTAS doubles of device scratch), then one CTA adds them in a fixed order.  Bitwise repeatable,
 * and identical on every rank given identical gradients; a NaN or inf gradient gives a NaN or inf norm.  extra may be NULL. */
int ssnb_grad_norm(const float* grad, size_t n, float grad_mult, const ssnb_extra_grads* extra, double* partials, float* norm,
                   void* stream);
/* the scaling half of clip_grad_norm (torch 0.3): c = max_norm / (*norm + 1e-6) in fp64; where c < 1 every gradient of the
 * flat buffer (n elements, may be 0) and of the extras is multiplied by (float)c in place, else nothing changes (a NaN
 * norm gives a NaN c, which is not < 1: no clipping, as in the reference).  *norm is read on the device. */
int ssnb_grad_clip(const float* norm, float max_norm, float* grad, size_t n, const ssnb_extra_grads* extra, void* stream);
/* ssnb_sgd_step_groups with the clip folded in: the gradient is multiplied by grad_mult * (float)c where c < 1 (c as in
 * ssnb_grad_clip), else by grad_mult, so where no clipping happens the parameters and momentum are bitwise those of
 * ssnb_sgd_step_groups.  write_back != 0 also stores that scaled gradient into grad and scales the extras by c (what the
 * reference's .grad holds after the division and clip_grad_norm); write_back == 0 leaves grad and the extras untouched. */
int ssnb_sgd_step_groups_clipped(float* param, float* grad, float* momentum_buf, size_t n, const int64_t* seg_end,
                                 const float* seg_lr, const float* seg_wd, int n_seg, float momentum, float grad_mult,
                                 const float* norm, float max_norm, int write_back, const ssnb_extra_grads* extra,
                                 void* stream);
/* the loop's AverageMeter updates of one step (ssn_train.py:213-233 with accuracy() :401-415 and AverageMeter :373-386;
 * binary_train.py:170-180 with :288-321), from outputs already on the device.  scores [rows, cols] fp32 with targets
 * [rows] int64: SSN's raw_act [n, K+1] of heads_loss_fused with prop_type [n] (the activity rows are those of type 0 or 2,
 * in order: activity_out), BinaryClassifier's [n, 2] scores with prop_type NULL (every row).  meters: device fp64 (sum,
 * count) pairs, n_losses + 3 of them: loss i gets sum += losses[i] * loss_n, count += loss_n (loss_n: out_frames.size(0));
 * then top-1 accuracy in percent over all activity rows (n = their count m), over the even ones (fg, view(-1, 2, .)[:, 0],
 * n = m / 2) and over the odd ones (bg, [:, 1], n = m / 2), each as the reference computes it:
 * val = float(correct) * float(100.0 / n), sum += val * n, count += n; a meter with n = 0 is left alone.  top-1 takes the
 * highest score, NaN above every number, and among equal scores the LOWEST class index (torch.topk leaves the order of
 * ties unspecified).  A target outside [0, cols) is never correct.  One CTA; rows <= 65536. */
int ssnb_train_meters(const float* scores, int rows, int cols, const int64_t* target, const int64_t* prop_type,
                      const float* losses, int n_losses, double loss_n, double* meters, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SSNB_H */
