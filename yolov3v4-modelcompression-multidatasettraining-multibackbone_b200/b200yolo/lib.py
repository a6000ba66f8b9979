"""ctypes binding of libb200yolo.so (C ABI in include/b200yolo.h).

PyTorch is only the owner of device memory and streams here: every call passes raw device pointers,
explicit shapes and the current CUDA stream to the native library.  There is no CPU fallback: if the
shared library is missing the import of this module raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_PKG, "libb200yolo.so")

ACT = {"linear": 0, "leaky": 1, "mish": 2, "relu": 3, "relu6": 4, "h_swish": 5, "swish": 6}
OUT_F16, OUT_F32, OUT_I8 = 0, 1, 2
DT_F16, DT_BF16 = 0, 1


class ConvDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int), ("in_h", C.c_int), ("in_w", C.c_int), ("in_c", C.c_int),
        ("in_pitch", C.c_longlong),
        ("out_c", C.c_int), ("ksize", C.c_int), ("stride", C.c_int), ("pad", C.c_int),
        ("out_h", C.c_int), ("out_w", C.c_int),
        ("out_pitch", C.c_longlong),
        ("act", C.c_int), ("slope", C.c_float),
        ("out_dtype", C.c_int),
        ("res_pitch", C.c_longlong),
        ("w_layout", C.c_int),
    ]


WLAYOUT_DENSE, WLAYOUT_S2_PAIRS = 0, 1

OPT_MAX_GROUPS, OPT_TILE, OPT_TILE_L1 = 4, 4096, 4


class OptGroup(C.Structure):
    _fields_ = [("lr", C.c_float), ("momentum", C.c_float), ("weight_decay", C.c_float),
                ("one_minus_beta1", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float), ("eps", C.c_float),
                ("step_size", C.c_float), ("bc2_sqrt", C.c_float)]


class OptStep(C.Structure):
    _fields_ = [("group", OptGroup * OPT_MAX_GROUPS), ("grad_scale", C.c_float), ("l1_coeff", C.c_float),
                ("ema_decay", C.c_float), ("first_step", C.c_int)]


class PackItem(C.Structure):
    _fields_ = [("w", C.c_void_p), ("w_fwd", C.c_void_p), ("w_dgrad", C.c_void_p),
                ("O", C.c_int), ("Opad", C.c_int), ("I", C.c_int), ("k", C.c_int), ("stride", C.c_int),
                ("pad", C.c_int), ("tile_begin", C.c_int), ("Ipad", C.c_int), ("col_map", C.c_void_p)]


class UnpackItem(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p),
                ("O", C.c_int), ("I", C.c_int), ("k", C.c_int), ("accumulate", C.c_int),
                ("tile_begin", C.c_int), ("Ipad", C.c_int)]


class LoadItem(C.Structure):
    _fields_ = [("src", C.c_void_p), ("src_pitch", C.c_longlong), ("src_h", C.c_int), ("src_w", C.c_int),
                ("rs_h", C.c_int), ("rs_w", C.c_int), ("area_kx", C.c_int), ("area_ky", C.c_int),
                ("scale_x", C.c_double), ("scale_y", C.c_double), ("top", C.c_int), ("left", C.c_int),
                ("slot", C.c_int), ("reserved", C.c_int)]


class MosaicTile(C.Structure):
    _fields_ = [("src", C.c_void_p), ("src_pitch", C.c_longlong), ("src_h", C.c_int), ("src_w", C.c_int),
                ("rs_h", C.c_int), ("rs_w", C.c_int), ("scale_x", C.c_double), ("scale_y", C.c_double),
                ("x1a", C.c_int), ("y1a", C.c_int), ("x2a", C.c_int), ("y2a", C.c_int), ("dx", C.c_int), ("dy", C.c_int)]


class MosaicItem(C.Structure):
    _fields_ = [("tiles", MosaicTile * 4), ("slot", C.c_int), ("reserved", C.c_int)]


class AffineItem(C.Structure):
    _fields_ = [("im", C.c_double * 6), ("lut", C.c_ubyte * 768), ("hsv", C.c_int), ("flip", C.c_int),
                ("slot", C.c_int), ("reserved", C.c_int)]


class QConvDesc(C.Structure):
    _fields_ = [
        ("conv", ConvDesc),
        ("acc_scale", C.c_float), ("out_scale", C.c_float),
        ("q_lo", C.c_float), ("q_hi", C.c_float),
        ("out_kind", C.c_int), ("requant", C.c_int), ("clamp_addends", C.c_int),
    ]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libb200yolo.so not built: run `python %s` (nvcc, sm_90a). There is no fallback path."
            % os.path.join(_PKG, "build.py"))
    return C.CDLL(LIB_PATH)


_lib = _load()

vp, ll, i32, f32, sz = C.c_void_p, C.c_longlong, C.c_int, C.c_float, C.c_size_t
_PROTOS = {
    "b2y_abi_version": (i32, []),
    "b2y_strerror": (C.c_char_p, [i32]),
    "b2y_last_cuda_error": (i32, []),
    "b2y_device_sm_count": (i32, []),
    "b2y_conv2d_fwd": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp]),
    "b2y_conv2d_fwd_stats": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp]),
    "b2y_stem_conv_fwd": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp]),
    "b2y_stem_workspace_bytes": (sz, [C.POINTER(ConvDesc)]),
    "b2y_pack_stem_weights": (i32, [vp, i32, i32, i32, vp, vp]),
    "b2y_stem_conv_fwd_fused": (i32, [C.POINTER(ConvDesc), vp, i32, f32, vp, vp, vp, vp]),
    "b2y_stem_conv_fwd_fused_q": (i32, [C.POINTER(ConvDesc), vp, i32, f32, vp, vp, vp, f32, f32, f32, vp]),
    "b2y_stem_conv_fwd_tc": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp, vp]),
    "b2y_pack_conv_weights": (i32, [vp, vp, vp, vp, vp, vp, f32, i32, i32, i32, vp, vp, vp, vp]),
    "b2y_upsample_nearest": (i32, [vp, ll, vp, ll, i32, i32, i32, i32, i32, vp]),
    "b2y_maxpool": (i32, [vp, ll, vp, ll, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b2y_copy_channels": (i32, [vp, ll, vp, ll, ll, i32, vp]),
    "b2y_add": (i32, [vp, ll, vp, ll, vp, ll, ll, i32, i32, vp]),
    "b2y_act_fwd_f32": (i32, [vp, vp, ll, i32, f32, vp]),
    "b2y_act_bwd_f32": (i32, [vp, vp, vp, ll, i32, f32, vp]),
    "b2y_nchw_f32_to_nhwc_f16": (i32, [vp, vp, ll, i32, i32, i32, i32, vp]),
    "b2y_nhwc_f16_to_nchw_f32": (i32, [vp, ll, vp, i32, i32, i32, i32, vp]),
    "b2y_yolo_decode": (i32, [vp, ll, vp, vp, ll, ll, i32, i32, i32, i32, i32, vp, f32, vp]),
    "b2y_yolo_loss_workspace_bytes": (sz, [i32, i32, i32, i32, i32]),
    "b2y_yolo_loss": (i32, [vp, vp, i32, vp, i32, i32, i32, i32, i32, f32, f32, f32, f32, f32, f32, f32, f32, vp,
                            vp, vp, vp]),
    "b2y_build_targets": (i32, [vp, i32, vp, i32, i32, i32, i32, f32, vp, vp, vp, vp, vp]),
    "b2y_qconv2d_fwd": (i32, [C.POINTER(QConvDesc), vp, vp, vp, vp, vp]),
    "b2y_qconv2d_shortcut_fwd": (i32, [C.POINTER(QConvDesc), vp, vp, vp, vp, ll, f32, f32, f32, f32, f32, f32, vp, vp]),
    "b2y_fakequant_f32": (i32, [vp, vp, ll, f32, f32, f32, vp]),
    "b2y_quantize_f16_to_i8": (i32, [vp, ll, vp, ll, ll, i32, f32, f32, f32, vp]),
    "b2y_cos_scale_search": (i32, [vp, ll, i32, i32, vp, vp, sz, vp]),
    "b2y_cos_scale_search_ex": (i32, [vp, ll, i32, i32, i32, vp, vp, sz, vp]),
    "b2y_minmax_f32": (i32, [vp, ll, ll, i32, vp, vp]),
    "b2y_pack_qconv_weights": (i32, [vp, i32, i32, i32, f32, f32, f32, vp, vp]),
    "b2y_qshortcut_i8": (i32, [vp, ll, vp, ll, vp, ll, ll, i32, f32, f32, f32, f32, f32, f32, f32, vp]),
    "b2y_requant_i8": (i32, [vp, ll, vp, ll, ll, i32, f32, f32, f32, f32, vp]),
    "b2y_upsample_nearest_i8": (i32, [vp, ll, vp, ll, i32, i32, i32, i32, i32, vp]),
    "b2y_maxpool_i8": (i32, [vp, ll, vp, ll, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b2y_stem_conv_fwd_q": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, f32, f32, f32, vp]),
    "b2y_bn_act_bwd_reduce": (i32, [vp, ll, vp, ll, vp, vp, vp, vp, vp, vp, vp, ll, i32, i32, f32, i32, vp]),
    "b2y_conv2d_bwd_data": (i32, [C.POINTER(ConvDesc), vp, vp, vp, i32, i32, i32, vp, vp]),
    "b2y_pack_dgrad_weights": (i32, [C.POINTER(ConvDesc), vp, vp, i32, vp]),
    "b2y_conv2d_bwd_weight": (i32, [C.POINTER(ConvDesc), vp, vp, vp, f32, i32, vp, vp]),
    "b2y_unpack_wgrad": (i32, [vp, vp, i32, i32, i32, f32, i32, vp]),
    "b2y_axpby_f32": (i32, [vp, vp, ll, f32, f32, vp]),
    "b2y_yolo_grad_to_raw": (i32, [vp, vp, ll, i32, i32, i32, i32, i32, f32, vp, i32, vp]),
    "b2y_upsample_nearest_bwd": (i32, [vp, ll, vp, ll, i32, i32, i32, i32, i32, i32, vp]),
    "b2y_maxpool_bwd": (i32, [vp, ll, vp, ll, vp, ll, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
    "b2y_stem_conv_bwd_weight": (i32, [C.POINTER(ConvDesc), vp, vp, vp, f32, i32, vp]),
    "b2y_bn_train_fwd": (i32, [vp, ll, vp, vp, ll, vp, vp, f32, f32, vp, vp, vp, vp, ll, vp, ll, ll, i32, i32, f32, vp]),
    "b2y_bn_train_fwd_lw": (i32, [vp, ll, vp, vp, ll, vp, vp, f32, f32, vp, vp, vp, vp, ll, vp, ll, ll, i32, i32, i32,
                                  f32, vp]),
    "b2y_bn_train_bwd_reduce": (i32, [vp, ll, vp, ll, vp, vp, vp, ll, i32, i32, f32, i32, vp]),
    "b2y_bn_train_bwd_apply": (i32, [vp, ll, vp, ll, vp, vp, vp, vp, ll, ll, i32, i32, f32, i32, vp, vp, vp, vp, f32,
                                     vp]),
    "b2y_dwconv_fwd": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp, vp]),
    "b2y_dwconv_bwd_data": (i32, [C.POINTER(ConvDesc), vp, vp, vp, i32, i32, vp, vp]),
    "b2y_dwconv_bwd_weight": (i32, [C.POINTER(ConvDesc), vp, vp, vp, f32, vp, vp]),
    "b2y_se_fwd": (i32, [vp, ll, vp, vp, vp, ll, i32, i32, i32, i32, vp, vp]),
    "b2y_se_bwd": (i32, [vp, ll, vp, ll, vp, vp, vp, vp, vp, ll, i32, vp, vp, f32, i32, i32, i32, i32, i32, vp]),
    "b2y_dwconv_fwd_f32": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp]),
    "b2y_dwconv_bwd_f32": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp]),
    "b2y_dwconv_stats_f32": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp]),
    "b2y_dwconv_stats_bwd_f32": (i32, [C.POINTER(ConvDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b2y_se_fwd_f32": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp]),
    "b2y_se_bwd_f32": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "b2y_bn_f32_fwd": (i32, [vp, ll, i32, vp, vp, f32, f32, vp, vp, i32, vp, vp, i32, f32, vp]),
    "b2y_bn_f32_bwd": (i32, [vp, vp, ll, i32, vp, vp, i32, vp, vp, vp, vp, i32, f32, vp]),
    "b2y_fakequant_bwd_f32": (i32, [vp, vp, vp, ll, f32, f32, f32, f32, vp]),
    "b2y_tpsq_fwd_f32": (i32, [vp, vp, ll, f32, i32, vp]),
    "b2y_tpsq_bwd_f32": (i32, [vp, vp, vp, vp, ll, f32, i32, vp]),
    "b2y_layout_tile_i": (i32, [i32]),
    "b2y_pack_conv_weights_multi": (i32, [vp, i32, i32, vp]),
    "b2y_unpack_wgrad_multi": (i32, [vp, i32, i32, vp]),
    "b2y_sgd_grouped": (i32, [vp, vp, vp, vp, vp, i32, C.POINTER(OptStep), vp]),
    "b2y_adam_grouped": (i32, [vp, vp, vp, vp, vp, vp, i32, C.POINTER(OptStep), vp]),
    "b2y_kd_soft_rows": (i32, [vp, vp, ll, i32, i32, i32, f32, f32, vp, vp, vp]),
    "b2y_kd_box": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, f32, vp, vp, vp, vp]),
    "b2y_letterbox_u8": (i32, [vp, i32, i32, i32, ll, i32, i32, i32, i32, vp, i32, i32, i32, i32, vp]),
    "b2y_load_batch_u8": (i32, [vp, vp, i32, vp, i32, i32, i32, i32, i32, i32, vp]),
    "b2y_mosaic_u8": (i32, [vp, vp, i32, vp, i32, i32, i32, vp]),
    "b2y_affine_hsv_u8": (i32, [vp, vp, i32, vp, vp, i32, i32, i32, vp]),
    "b2y_nms_count_workspace_bytes": (sz, [i32, i32]),
    "b2y_nms_count": (i32, [vp, i32, i32, i32, f32, i32, vp, vp, vp, vp, sz, vp]),
    "b2y_nms_run_workspace_bytes": (sz, [ll]),
    "b2y_nms_run": (i32, [vp, i32, i32, i32, f32, C.c_double, i32, i32, vp, vp, vp, ll, vp, sz, vp, vp, vp]),
    "b2y_tp_match_workspace_bytes": (sz, [ll, ll]),
    "b2y_tp_match": (i32, [vp, vp, vp, ll, vp, vp, vp, ll, vp, i32, i32, f32, f32, vp, sz, vp, vp]),
}

EXPORTS = sorted(_PROTOS)
MISSING = []
for _name, (_res, _args) in _PROTOS.items():
    try:
        _fn = getattr(_lib, _name)
    except AttributeError:
        MISSING.append(_name)
        continue
    _fn.restype = _res
    _fn.argtypes = _args


class B2YError(RuntimeError):
    pass


def check(status, what=""):
    if status != 0:
        msg = _lib.b2y_strerror(status).decode()
        extra = ""
        if status == -2:
            extra = " (cudaError %d)" % _lib.b2y_last_cuda_error()
        raise B2YError("%s failed: %s%s" % (what or "b200yolo call", msg, extra))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    if RECORD is not None:
        KEEPALIVE.append(t)
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def raw():
    return _lib


# Launch recorder (measurement only, bench.py / tools): while RECORD is a list every C-ABI call is appended as
# (name, args) so that a family of launches (e.g. all wgmma convolutions of one step) can be replayed back to back.
RECORD = None
KEEPALIVE = []      # tensors whose pointers were handed out while recording (temporaries must outlive the replay)


def call(name, *args):
    if RECORD is not None:
        RECORD.append((name, args))
    check(getattr(_lib, name)(*args), name)
