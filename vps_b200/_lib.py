"""ctypes binding of libvps_b200.so -- the only native entry into the product path.

There is NO fallback: if the library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvps_b200.so")

VPS_F32, VPS_BF16 = 0, 1
ACT_NONE, ACT_RELU, ACT_LRELU, ACT_SIGMOID = 0, 1, 2, 3


class VpsTensor(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
                ("c", C.c_int32), ("cs", C.c_int32), ("dtype", C.c_int32)]


class VpsConvArgs(C.Structure):
    _fields_ = [("x", VpsTensor), ("y", VpsTensor), ("res", VpsTensor),
                ("w", C.c_void_p), ("bias", C.c_void_p),
                ("kh", C.c_int32), ("kw", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
                ("ph", C.c_int32), ("pw", C.c_int32),
                ("oh", C.c_int32), ("ow", C.c_int32),
                ("oy_mul", C.c_int32), ("oy_off", C.c_int32), ("ox_mul", C.c_int32), ("ox_off", C.c_int32),
                ("cin", C.c_int32), ("cout", C.c_int32),
                ("act", C.c_int32), ("slope", C.c_float), ("res_after_act", C.c_int32),
                ("out_scale", C.c_float), ("cin_gran", C.c_int32)]


class VpsError(RuntimeError):
    pass


_lib = None


def lib():
    """Load (once) and return the ctypes handle. Raises if the .so has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VpsError(
                "libvps_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'`; "
                "there is no CPU/PyTorch fallback for the product path" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        _lib.vps_last_error.restype = C.c_char_p
        _lib.vps_launch_count.restype = C.c_int64
        _lib.vps_packed_tc_bytes.restype = C.c_int64
        _lib.vps_packed_tc32_bytes.restype = C.c_int64
        _lib.vps_correlation_tc32_ws_bytes.restype = C.c_int64
        _lib.vps_unify_pan_ws_bytes.restype = C.c_int64
        _lib.vps_unify_pan_error_offset.restype = C.c_int64
        _lib.vps_tube_confusion_ws_bytes.restype = C.c_int64
        _lib.vps_tube_confusion_ws_bytes.argtypes = [C.c_int64]
        _lib.vps_add_launch_count.restype = None
        _lib.vps_add_launch_count.argtypes = [C.c_int64]
    return _lib


def check(status, what=""):
    if status != 0:
        raise VpsError("%s failed (%d): %s" % (what, status, lib().vps_last_error().decode()))


# every symbol include/vps_b200.h declares (tests assert the .so exports all of them)
EXPORTS = [
    "vps_last_error", "vps_version", "vps_launch_count", "vps_add_launch_count",
    "vps_conv2d_tc", "vps_conv2d_tc_multi", "vps_conv2d_tc_plan", "vps_conv2d_simt", "vps_pack_weights_tc", "vps_pack_weights_simt",
    "vps_packed_tc_bytes", "vps_im2col",
    "vps_conv2d_tc32", "vps_conv2d_tc32_multi", "vps_conv2d_tc32_plan", "vps_pack_weights_tc32", "vps_packed_tc32_bytes", "vps_tc32_overflow", "vps_deform_conv_tc32", "vps_deform_conv_tc32_plan",
    "vps_correlation", "vps_correlation_tc", "vps_correlation_simt", "vps_correlation_tc32", "vps_correlation_tc32_ws_bytes", "vps_resample2d", "vps_channelnorm", "vps_flownet_input", "vps_flownet_stage", "vps_flownet_cat3", "vps_flow_deconv",
    "vps_nchw_to_nhwc", "vps_nhwc_to_nchw", "vps_copy_scale", "vps_axpby",
    "vps_space_to_depth2", "vps_tap_gather3x3", "vps_preprocess_u8", "vps_preprocess_resize_u8", "vps_resize_bilinear", "vps_resize_nearest", "vps_pool2d", "vps_groupnorm",
    "vps_bfp_gather", "vps_bfp_scatter", "vps_flow_warp", "vps_tcea_temporal", "vps_tcea_combine",
    "vps_deform_im2col", "vps_deform_conv_tc",
    "vps_roi_align", "vps_sort_desc", "vps_rpn_decode", "vps_nms", "vps_nms_batch", "vps_sigmoid_flat", "vps_gather_rows",
    "vps_maskroi_candidates", "vps_track_assign",
    "vps_rpn_finalize", "vps_maskroi_finalize", "vps_select_class", "vps_track_update", "vps_det_split",
    "vps_mask_removal", "vps_panoptic_fuse", "vps_unify_pan", "vps_unify_pan_image", "vps_unify_pan_ws_bytes", "vps_unify_pan_error", "vps_unify_pan_error_offset", "vps_tube_confusion", "vps_tube_confusion_ws_bytes", "vps_rgb_to_id", "vps_pan2ch_ids",
    "vps_pan2ch_image_ids", "vps_seg_confusion", "vps_seg_confusion_nearest",
]
