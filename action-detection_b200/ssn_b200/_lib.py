"""ctypes binding of libssn_b200.so (C ABI declared in include/ssnb.h).

The library is the product: there is no CPU or PyTorch fallback.  If the shared object is missing
the import fails loudly; build it with `python -c "import __graft_entry__ as g; g.build()"` or
action-detection_b200/csrc/build.sh.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libssn_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError("libssn_b200.so not found at %s — build the CUDA extension first "
                      "(action-detection_b200/csrc/build.sh); there is no fallback path." % LIB_PATH)

lib = C.CDLL(LIB_PATH)

EXACT_FP32, FAST_FP16, EXACT_TC = 0, 1, 2


class Config(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("frames", C.c_int32), ("precision", C.c_int32),
                ("training", C.c_int32), ("grad_scale", C.c_float), ("bn1_train", C.c_int32), ("reserved", C.c_int32 * 2)]


class IV3Config(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("frames", C.c_int32), ("precision", C.c_int32), ("reserved", C.c_int32)]


class HeadsCfg(C.Structure):
    _fields_ = [("n", C.c_int32), ("props_per_video", C.c_int32), ("num_class", C.c_int32),
                ("feat_dim", C.c_int32), ("feat_mult", C.c_int32), ("fg_per_video", C.c_int32),
                ("comp_group", C.c_int32), ("global_videos", C.c_int32), ("keep_neg", C.c_int32),
                ("comp_denom", C.c_float), ("comp_w", C.c_float), ("reg_w", C.c_float),
                ("loss_scale", C.c_float)]


class TagProposalsCfg(C.Structure):
    _fields_ = [("cls", C.c_int32), ("n_thresholds", C.c_int32), ("n_tolerances", C.c_int32), ("reserved", C.c_int32),
                ("sigma", C.c_double), ("nms_thresh", C.c_double), ("minimum_len", C.c_double),
                ("thresholds", C.POINTER(C.c_double)), ("tolerances", C.POINTER(C.c_double))]


class DetectBatchCfg(C.Structure):
    _fields_ = [("mode", C.c_int32), ("top_k", C.c_int32), ("n_sel", C.c_int32), ("softmax_before_filter", C.c_int32),
                ("regress", C.c_int32), ("reserved", C.c_int32), ("nms_thresh", C.c_double)]


DET_ALL, DET_TOPK, DET_CLS = 0, 1, 2


class FrameCfg(C.Structure):
    _fields_ = [("mode", C.c_int32), ("channels", C.c_int32), ("out_size", C.c_int32), ("scale_size", C.c_int32),
                ("invert_even", C.c_int32), ("n_mean", C.c_int32), ("mean", C.c_float * 8), ("std", C.c_float * 8)]


class FrameGroup(C.Structure):
    _fields_ = [("src_offset", C.c_int64), ("dst_offset", C.c_int64), ("scratch_offset", C.c_int64), ("first_image", C.c_int32),
                ("height", C.c_int32), ("width", C.c_int32), ("images", C.c_int32), ("crop_x", C.c_int32), ("crop_y", C.c_int32),
                ("crop_w", C.c_int32), ("crop_h", C.c_int32), ("flip", C.c_int32), ("reserved", C.c_int32)]


FRAMES_TRAIN, FRAMES_OVERSAMPLE, FRAMES_CENTER = 0, 1, 2


class JpegInput(C.Structure):
    _fields_ = [("offset", C.c_int64), ("bytes", C.c_int64), ("channels", C.c_int32), ("reserved", C.c_int32)]


class JpegImageInfo(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("components", C.c_int32), ("h_samp", C.c_int32),
                ("v_samp", C.c_int32), ("channels", C.c_int32), ("restart_interval", C.c_int32), ("intervals", C.c_int32),
                ("scan_offset", C.c_int64), ("scan_bytes", C.c_int64), ("out_offset", C.c_int64)]


JPEG_OK, JPEG_TRUNCATED, JPEG_BAD_CODE, JPEG_BAD_RUN, JPEG_BAD_RESTART = 0, 1, 2, 3, 4


class ProposalTargetsCfg(C.Structure):
    _fields_ = [("fg_thresh", C.c_double), ("incomplete_iou_thresh", C.c_double), ("bg_iou_thresh", C.c_double),
                ("bg_coverage_thresh", C.c_double), ("incomplete_overlap_thresh", C.c_double), ("exclude_empty", C.c_int32),
                ("reserved", C.c_int32)]


GRAD_NORM_CTAS, MAX_EXTRA_GRADS = 512, 8


class ExtraGrads(C.Structure):
    _fields_ = [("count", C.c_int32), ("reserved", C.c_int32), ("grad", C.c_void_p * MAX_EXTRA_GRADS),
                ("numel", C.c_int64 * MAX_EXTRA_GRADS)]


PROPFRAMES_SECONDS, PROPFRAMES_NORMALISED, PROPFRAMES_AS_GIVEN = 0, 1, 2
TAG_FG, TAG_INCOMPLETE, TAG_BACKGROUND = 1, 2, 4

_vp, _i, _f, _sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
_ip = C.POINTER(C.c_int)
_pp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); every symbol include/ssnb.h declares
SIGNATURES = {
    "ssnb_create": (_i, [C.POINTER(Config), C.POINTER(_vp)]),
    "ssnb_destroy": (_i, [_vp]),
    "ssnb_last_error": (C.c_char_p, [_vp]),
    "ssnb_version": (C.c_char_p, []),
    "ssnb_num_convs": (_i, []),
    "ssnb_conv_info": (_i, [_i, _i, C.c_char_p, _i, _ip, _ip, _ip, _ip, _ip]),
    "ssnb_workspace_bytes": (_sz, [_vp]),
    "ssnb_set_workspace": (_i, [_vp, _vp, _sz]),
    "ssnb_pack_weights": (_i, [_vp, _pp, _pp, _pp, _pp, _pp, _pp, _vp]),
    "ssnb_set_bn1": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f]),
    "ssnb_backbone_fwd": (_i, [_vp, _vp, _vp, _vp]),
    "ssnb_backbone_fwd_frames": (_i, [_vp, _vp, _i, _vp, _vp]),
    "ssnb_backbone_bwd": (_i, [_vp, _vp, _pp, _pp, _vp]),
    "ssnb_backbone_bwd_range": (_i, [_vp, _vp, _pp, _pp, _i, _i, _vp]),
    "ssnb_bind_grads": (_i, [_vp, _pp, _pp]),
    "ssnb_set_grad_accumulate": (_i, [_vp, _i]),
    "ssnb_num_ops": (_i, [_vp]),
    "ssnb_op_info": (_i, [_vp, _i, C.c_char_p, _i, C.c_char_p, _i, C.c_char_p, _i]),
    "ssnb_value_shape": (_i, [_vp, C.c_char_p, _ip, _ip, _ip]),
    "ssnb_value_write": (_i, [_vp, C.c_char_p, _i, _vp, _vp]),
    "ssnb_value_read": (_i, [_vp, C.c_char_p, _i, _vp, _vp]),
    "ssnb_run_op": (_i, [_vp, _i, _i, _vp]),
    "ssnb_launch_count": (C.c_int64, [_vp]),
    "ssnb_global_launch_count": (C.c_int64, []),
    "ssnb_stpp_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _ip, _ip, _ip, _ip, _i, _i, _vp, _vp, _vp]),
    "ssnb_stpp_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _ip, _ip, _ip, _ip, _i, _i, _vp, _vp]),
    "ssnb_gpool_stpp_fwd": (_i, [_vp, _vp, _vp, _i, _i, _ip, _ip, _ip, _ip, _i, _i, _vp, _vp, _vp, _vp]),
    "ssnb_stpp_reorg_workspace_bytes": (_sz, [_i, _i]),
    "ssnb_stpp_reorg_prefix": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _i, _i, _ip, _ip, _vp, _vp, _vp, _vp, _vp]),
    "ssnb_stpp_reorg_batch_workspace_bytes": (_sz, [C.POINTER(C.c_int64), _i, _i]),
    "ssnb_stpp_reorg_batch": (_i, [_vp, _i, C.POINTER(C.c_int64), _vp, _vp, _vp, C.POINTER(C.c_int64), _vp, _i, _i, _i, _i, _ip, _ip,
                                   C.POINTER(C.c_double), _vp, _vp, _vp, _vp, _sz, _vp]),
    "ssnb_linear_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "ssnb_test_fc_cropmean": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "ssnb_linear_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "ssnb_ohem_hinge_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "ssnb_ohem_hinge_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "ssnb_classwise_reg_fwd": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    "ssnb_classwise_reg_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "ssnb_heads_loss_workspace_bytes": (_sz, [C.POINTER(HeadsCfg)]),
    "ssnb_heads_loss_fwd_bwd": (_i, [C.POINTER(HeadsCfg)] + [_vp] * 25),
    "ssnb_classifier_ce_workspace_bytes": (_sz, [_i, _i]),
    "ssnb_classifier_ce_fwd_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ssnb_grad_overflow": (_i, [_vp, _i]),
    "ssnb_timing_begin": (_i, [_vp]),
    "ssnb_timing_report": (C.c_char_p, []),
    "ssnb_timing_launches": (C.c_char_p, []),
    "ssnb_detect_postprocess": (_i, [_vp, _vp, _vp, _vp, _i, _i, C.c_double, _i, _vp, _vp, _vp, _vp]),
    "ssnb_detect_batch_workspace_bytes": (_sz, [C.POINTER(DetectBatchCfg), _i, C.POINTER(C.c_int64), _i]),
    "ssnb_detect_batch": (_i, [C.POINTER(DetectBatchCfg), _vp, _vp, _vp, _vp, _i, C.POINTER(C.c_int64), _vp, _i, _vp, _vp, _vp, _vp, _vp,
                               _vp, _sz, _vp]),
    "ssnb_detection_ap_workspace_bytes": (_sz, [_i, _i, C.c_int64, C.c_int64, _i]),
    "ssnb_detection_ap": (_i, [_vp, _vp, _vp, _i, _i, C.c_int64, _vp, _vp, _vp, C.c_int64, C.POINTER(C.c_double), _i, _vp, _vp, _vp,
                               _vp, _sz, _vp]),
    "ssnb_tag_proposals_workspace_bytes": (_sz, [_i, C.c_int64, _i, _i]),
    "ssnb_tag_proposals": (_i, [C.POINTER(TagProposalsCfg), _vp, _i, C.POINTER(C.c_int64), _vp, _i, _vp] + [_vp] * 10
                           + [_sz, _vp]),
    "ssnb_name_proposals": (_i, [_vp, _vp, _vp, _i, C.c_int64, _vp, _vp, C.POINTER(C.c_int64), _vp, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "ssnb_proposal_recall": (_i, [_vp, C.POINTER(C.c_int64), _vp, _i, C.POINTER(C.c_double), _i, _vp, _vp, _vp]),
    "ssnb_sliding_windows": (_i, [_vp, _i, C.POINTER(C.c_double), C.POINTER(C.c_double), _i, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp,
                                  _vp, _vp]),
    "ssnb_proposal_frames": (_i, [_vp, _vp, _vp, _i, C.c_int64, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "ssnb_proposal_targets_workspace_bytes": (_sz, [_i]),
    "ssnb_proposal_targets": (_i, [C.POINTER(ProposalTargetsCfg)] + [_vp] * 6 + [_i, _vp, C.POINTER(C.c_int64)] + [_vp] * 7 + [_sz, _vp]),
    "ssnb_test_proposals": (_i, [_vp, _vp, _vp, _vp, _i, C.c_int64, _vp, _i, _i] + [_vp] * 7),
    "ssnb_proposal_ar_workspace_bytes": (_sz, [_i, C.c_int64, C.POINTER(C.c_int64), _i]),
    "ssnb_proposal_ar": (_i, [_vp, _vp, C.c_int64, _vp, _vp, _i, _vp, C.POINTER(C.c_int64), _vp, C.POINTER(C.c_double), _i, C.c_double]
                         + [_vp] * 7 + [_sz, _vp]),
    "ssnb_classification_ap_workspace_bytes": (_sz, [C.c_int64, C.c_int64, _i, _i]),
    "ssnb_classification_ap": (_i, [_vp, _vp, _vp, C.c_int64, _vp, _vp, C.c_int64, _i, _i, _i] + [_vp] * 7 + [_sz, _vp]),
    "ssnb_video_aggregate_workspace_bytes": (_sz, [C.POINTER(C.c_int64), _i, _i, _i, _i, _i, _i, _ip, _i, C.c_double, _i, _i]),
    "ssnb_video_aggregate": (_i, [_vp, C.POINTER(C.c_int64), _vp, _i, _i, _i, _i, _i, _i, _i, _ip, _i, C.c_double, _i, _i, _vp, _vp,
                                  _sz, _vp]),
    "ssnb_video_fuse": (_i, [_vp, _pp, C.POINTER(C.c_double), _i, C.c_int64, _i, _i, C.c_double, _vp, _vp]),
    "ssnb_video_metrics_workspace_bytes": (_sz, [_i, _i]),
    "ssnb_video_metrics": (_i, [_vp, _i, _i, _i, _vp, _vp, C.c_int64, _vp, _i] + [_vp] * 8 + [_vp, _sz, _vp]),
    "ssnb_frame_transform_workspace_bytes": (_i, [C.POINTER(FrameCfg), C.POINTER(FrameGroup), _i, C.POINTER(_sz), C.POINTER(C.c_int64)]),
    "ssnb_frame_transform": (_i, [C.POINTER(FrameCfg), C.POINTER(FrameGroup), _vp, _i, _vp, _sz, _vp, C.c_int64, _vp, _sz, _vp]),
    "ssnb_jpeg_plan_create": (_i, [_vp, _sz, C.POINTER(JpegInput), _i, C.POINTER(_vp), _ip]),
    "ssnb_jpeg_plan_destroy": (_i, [_vp]),
    "ssnb_jpeg_plan_sizes": (_i, [_vp, C.POINTER(_sz), C.POINTER(_sz), C.POINTER(C.c_int64)]),
    "ssnb_jpeg_plan_image": (_i, [_vp, _i, C.POINTER(JpegImageInfo)]),
    "ssnb_jpeg_plan_write_table": (_i, [_vp, _vp, _sz]),
    "ssnb_jpeg_decode": (_i, [_vp, _vp, _vp, _sz, _vp, C.c_int64, _vp, _vp, _sz, _vp]),
    "ssnb_iv3_num_convs": (_i, []),
    "ssnb_iv3_conv_info": (_i, [_i, _i, C.c_char_p, _i] + [_ip] * 7),
    "ssnb_iv3_create": (_i, [C.POINTER(IV3Config), C.POINTER(_vp)]),
    "ssnb_iv3_destroy": (_i, [_vp]),
    "ssnb_iv3_workspace_bytes": (_sz, [_vp]),
    "ssnb_iv3_set_workspace": (_i, [_vp, _vp, _sz]),
    "ssnb_iv3_pack_weights": (_i, [_vp, _pp, _pp, _pp, _pp, _pp, _pp, _vp]),
    "ssnb_iv3_forward": (_i, [_vp, _vp, _vp, _vp]),
    "ssnb_iv3_forward_frames": (_i, [_vp, _vp, _i, _vp, _vp]),
    "ssnb_iv3_num_ops": (_i, [_vp]),
    "ssnb_iv3_op_info": (_i, [_vp, _i, C.c_char_p, _i, C.c_char_p, _i, C.c_char_p, _i, _ip, _ip, _ip, _ip]),
    "ssnb_iv3_value_info": (_i, [_vp, C.c_char_p, _ip, _ip, _ip, C.c_char_p, _i, _ip]),
    "ssnb_iv3_value_write": (_i, [_vp, C.c_char_p, _vp, _vp]),
    "ssnb_iv3_value_read": (_i, [_vp, C.c_char_p, _i, _vp, _vp]),
    "ssnb_iv3_run_op": (_i, [_vp, _i, _vp, _vp]),
    "ssnb_sgd_step_groups": (_i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i, _f, _f, _vp]),
    "ssnb_grad_norm": (_i, [_vp, _sz, _f, C.POINTER(ExtraGrads), _vp, _vp, _vp]),
    "ssnb_grad_clip": (_i, [_vp, _f, _vp, _sz, C.POINTER(ExtraGrads), _vp]),
    "ssnb_sgd_step_groups_clipped": (_i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i, _f, _f, _vp, _f, _i, C.POINTER(ExtraGrads), _vp]),
    "ssnb_train_meters": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, C.c_double, _vp, _vp]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)          # AttributeError here == symbol missing from the .so
    _fn.restype = _res
    _fn.argtypes = _args


def check(rc, handle=None, what=""):
    if rc != 0:
        msg = lib.ssnb_last_error(handle)
        raise RuntimeError("libssn_b200 %s failed (code %d): %s" % (what, rc, (msg or b"").decode()))


def int_array(seq):
    return (C.c_int * len(seq))(*[int(v) for v in seq])


def ptr_array(tensors):
    return (C.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])
