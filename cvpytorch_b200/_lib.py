"""ctypes binding of libcvb200.so (the C ABI declared in include/cvb200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, an exception is
raised.  The reference has no FFI (it is pure PyTorch); this file is the "binding a maintainer would add"
shown in INTEGRATION.md.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# CVB_DIAG_LIB=1 (developer tools only) loads the diagnostics build of the same sources (csrc/build.sh diag: cycle counters + CVB_DBG switches)
LIB_PATH = os.path.join(_HERE, 'libcvb200_diag.so' if os.environ.get('CVB_DIAG_LIB') == '1' else 'libcvb200.so')

CVB_ACT_NONE, CVB_ACT_SILU, CVB_ACT_RELU = 0, 1, 2
CVB_OUT_SPLIT16, CVB_OUT_F32, CVB_OUT_YOLO = 0, 1, 2


class CvbView(ctypes.Structure):
    _fields_ = [('base', c_void_p), ('B', c_int32), ('H', c_int32), ('W', c_int32), ('C', c_int32),
                ('c_pitch', c_int32), ('plane_stride', c_int64)]


class CvbYoloDecode(ctypes.Structure):
    _fields_ = [('na', c_int32), ('no', c_int32), ('anchors_px', c_float * 8), ('stride', c_float), ('z', c_void_p), ('z_rows', c_int64),
                ('z_off', c_int64), ('nms_workspace', c_void_p), ('conf_thres', c_float), ('multi_label', c_int32)]


class CvbConvDesc(ctypes.Structure):
    _fields_ = [('inp', CvbView), ('out', CvbView), ('weights', c_void_p), ('cout_pad', c_int32),
                ('bias', c_void_p), ('kh', c_int32), ('kw', c_int32), ('stride', c_int32), ('pad', c_int32),
                ('dilation', c_int32), ('act', c_int32), ('out_kind', c_int32), ('residual', CvbView),
                ('up_partial', CvbView), ('block_n', c_int32), ('sm_limit', c_int32), ('no_resident', c_int32), ('residual_before_act', c_int32), ('w_window', c_int32), ('halo', c_int32), ('yolo', POINTER(CvbYoloDecode)), ('residual_scale', c_float), ('schedule', c_int32)]


class CvbNmsParams(ctypes.Structure):
    _fields_ = [('B', c_int32), ('A', c_int32), ('nc', c_int32), ('conf_thres', c_float),
                ('iou_thres', c_double), ('multi_label', c_int32), ('max_nms', c_int32), ('max_det', c_int32),
                ('max_wh', c_float), ('hist_ready', c_int32)]


class CvbEmaEntry(ctypes.Structure):
    _fields_ = [('ema', c_void_p), ('src', c_void_p), ('numel', c_int64)]


CVB_EMA_TABLE_ENTRY_BYTES = 32


class CvbSgdGroup(ctypes.Structure):
    _fields_ = [('lr', c_float), ('weight_decay', c_float), ('momentum', c_float), ('flags', c_int32)]


class CvbSgdEntry(ctypes.Structure):
    _fields_ = [('param', c_void_p), ('grad', c_void_p), ('momentum_buffer', c_void_p), ('valid', c_void_p), ('numel', c_int64),
                ('group', c_int32)]


CVB_SGD_TABLE_ENTRY_BYTES = 64
CVB_SGD_CHUNK = 4096
CVB_SGD_MAX_GROUPS = 1024
CVB_SGD_NESTEROV, CVB_SGD_WEIGHT_DECAY, CVB_SGD_MOMENTUM = 1, 2, 4

CVB_COCO_IOU_THRS, CVB_COCO_REC_THRS = 10, 101
CVB_COCO_MAX_IMAGES, CVB_COCO_MAX_CATS, CVB_COCO_MAX_GT, CVB_COCO_MAX_DETS = 1 << 20, 4000, 1 << 26, 1 << 28


class CvbCocoEvalParams(ctypes.Structure):
    _fields_ = [('n_images', c_int32), ('n_cats', c_int32), ('n_gt', c_int32), ('n_det', c_int32), ('iou_thrs', c_double * CVB_COCO_IOU_THRS),
                ('rec_thrs', c_double * CVB_COCO_REC_THRS)]


CVB_SEG_U8, CVB_SEG_I32, CVB_SEG_I64 = 0, 1, 2
CVB_SEG_ERR_NEGATIVE, CVB_SEG_ERR_OVERFLOW = 1, 2
CVB_SEG_MAX_N = (1 << 31) - 1  # pixels per cvb_seg_confusion_update call

# name -> (restype, argtypes); must list every symbol include/cvb200.h declares
SYMBOLS = {
    'cvb_conv_plan_create': (c_int32, [POINTER(CvbConvDesc), POINTER(c_void_p)]),
    'cvb_conv_plan_run': (c_int32, [c_void_p, c_void_p]),
    'cvb_conv_plan_destroy': (None, [c_void_p]),
    'cvb_conv_plan_run_many': (c_int32, [POINTER(c_void_p), c_int32, c_void_p]),
    'cvb_letterbox_u8': (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, POINTER(c_int32), c_void_p, c_void_p]),
    'cvb_coco_pack': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_pack_weights': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_conv': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_conv_dgrad_s2': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_conv_wgrad': (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    'cvb_train_bn_stats': (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_silu_fwd': (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_silu_bwd': (c_int32, [c_void_p, c_int32, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_partial': (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_merge': (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_silu_bwd_reduce': (c_int32, [c_void_p, c_int32, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_bn_silu_bwd_apply': (c_int32, [c_void_p, c_int32, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_focus_s2d': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    'cvb_train_spp_pool_fwd': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_spp_pool_bwd': (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    'cvb_train_sppf_chain_fwd': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_sppf_chain_bwd': (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_upsample_cat_fwd': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_void_p]),
    'cvb_train_upsample_cat_bwd': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_conv_pad': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_train_conv_wgrad_pad': (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p]),
    'cvb_train_pred_conv': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p]),
    'cvb_train_pred_grad': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_train_yolox_loss_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'cvb_train_yolox_loss_fwd': (c_int32, [POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), c_int32, c_int32, c_void_p, c_int32, c_int32,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'cvb_train_yolox_loss_bwd': (c_int32, [POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), c_int32, c_int32, c_void_p, c_int32, c_int32,
                                           c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_void_p), c_void_p]),
    'cvb_train_yolov5_loss_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32]),
    'cvb_train_yolov5_loss_fwd': (c_int32, [POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), POINTER(c_float), c_int32, c_int32, c_int32, c_void_p,
                                            c_int32, POINTER(c_float), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'cvb_train_yolov5_loss_bwd': (c_int32, [POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), POINTER(c_float), c_int32, c_int32, c_int32, c_void_p,
                                            c_int32, POINTER(c_float), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_void_p),
                                            c_void_p]),
    'cvb_train_fcos_loss_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32]),
    'cvb_train_fcos_loss_fwd': (c_int32, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), POINTER(c_float),
                                          c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                          c_void_p]),
    'cvb_train_fcos_loss_bwd': (c_int32, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_int32), POINTER(c_float), POINTER(c_float),
                                          c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, POINTER(c_void_p),
                                          POINTER(c_void_p), POINTER(c_void_p), c_void_p]),
    'cvb_ema_table_upload':(c_int32, [c_void_p, c_int32, c_void_p, c_void_p]),
    'cvb_ema_update': (c_int32, [c_void_p, c_int32, c_float, c_float, c_void_p]),
    'cvb_sgd_table_upload': (c_int32, [POINTER(CvbSgdEntry), c_int32, c_int32, c_void_p, c_void_p]),
    'cvb_sgd_step': (c_int32, [c_void_p, c_int32, POINTER(CvbSgdGroup), c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_coco_eval_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32]),
    'cvb_coco_eval_bbox': (c_int32, [POINTER(CvbCocoEvalParams), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'cvb_seg_confusion_nc_max': (c_int32, []),
    'cvb_seg_confusion_update': (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_int64, c_int32, c_void_p, c_void_p, c_void_p]),
    'cvb_conv_plan_set_profile': (c_int32, [c_void_p, c_void_p, POINTER(c_int32)]),
    'cvb_nchw_to_split': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_int32, POINTER(CvbView), c_void_p]),
    'cvb_split_to_nchw': (c_int32, [POINTER(CvbView), c_void_p, c_void_p]),
    'cvb_f32nhwc_to_nchw': (c_int32, [POINTER(CvbView), c_void_p, c_void_p]),
    'cvb_stem_s2d': (c_int32, [c_void_p, c_int32, c_int32, c_int32, POINTER(CvbView), c_int32, c_void_p]),
    'cvb_stem_s2d_u8': (c_int32, [c_void_p, c_int32, c_int32, c_int32, POINTER(c_float), POINTER(c_float), c_int32, POINTER(CvbView), c_int32, c_void_p]),
    'cvb_maxpool3x3s2': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_void_p]),
    'cvb_split_to_f32nhwc': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_void_p]),
    'cvb_groupnorm_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'cvb_groupnorm_relu': (c_int32, [POINTER(CvbView), c_int32, c_void_p, c_void_p, c_float, c_int32, POINTER(CvbView), c_void_p,
                                     c_size_t, c_void_p]),
    'cvb_sppf_pool': (c_int32, [POINTER(CvbView), POINTER(CvbView), POINTER(CvbView), POINTER(CvbView), c_void_p]),
    'cvb_yolo_decode': (c_int32, [POINTER(CvbView), c_int32, c_int32, c_void_p, c_float, c_void_p, c_int64,
                                  c_int64, c_void_p, c_void_p, c_float, c_int32, c_void_p]),
    'cvb_nms_workspace_reset': (c_int32, [c_void_p, c_size_t, c_int32, c_void_p]),
    'cvb_nms_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32]),
    'cvb_yolo_nms': (c_int32, [c_void_p, POINTER(CvbNmsParams), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                               c_void_p, c_void_p]),
    'cvb_dwconv3x3': (c_int32, [POINTER(CvbView), c_void_p, c_void_p, c_int32, c_int32, POINTER(CvbView), c_void_p]),
    'cvb_global_avgpool': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_void_p]),
    'cvb_bilinear_resize': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_void_p]),
    'cvb_upsample_argmax': (c_int32, [POINTER(CvbView), c_int32, c_void_p, c_int32, c_int32, c_void_p]),
    'cvb_fcos_decode': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_int32, c_float, c_float, c_void_p, c_void_p, c_void_p, c_int64,
                                  c_int64, c_void_p]),
    'cvb_fcos_nms': (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_float, c_float, c_int32, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_yolox_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'cvb_yolox_decode': (c_int32, [POINTER(CvbView), POINTER(CvbView), c_int32, c_float, c_void_p, c_int64, c_int64, c_void_p]),
    'cvb_yolox_nms': (c_int32, [c_void_p, c_int32, c_int32, c_float, c_double, c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'cvb_rescale_clip_boxes': (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'cvb_confusion_matrix': (c_int32, [c_void_p, c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    'cvb_last_error_string': (c_char_p, []),
    'cvb_version': (c_int32, []),
    'cvb_launch_count': (c_int64, []),
}

_lib = None


class CvbError(RuntimeError):
    pass


def lib():
    """Loads libcvb200.so once; raises if it has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            how = ('`bash cvpytorch_b200/csrc/build.sh diag` (the diagnostics build used by tools/*profile*.py)' if LIB_PATH.endswith('_diag.so')
                   else '`python -c "import __graft_entry__ as g; g.build()"` (cvpytorch_b200/csrc/build.sh)')
            raise CvbError(f'{LIB_PATH} not found: build it with {how}. The H100 path has no CPU fallback.')
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc, what=''):
    if rc != 0:
        msg = lib().cvb_last_error_string()
        raise CvbError(f'{what}: cvb error {rc}: {msg.decode() if msg else "?"}')


def launch_count():
    return int(lib().cvb_launch_count())
