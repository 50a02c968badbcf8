"""ctypes binding of include/mcb200.h.  No fallback: a missing library or a failing call raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmcb200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "libmcb200.so not built: run `python __graft_entry__.py` (nvcc, sm_90a). There is no CPU fallback.")

lib = C.CDLL(LIB_PATH)
lib.mcb_last_error.restype = C.c_char_p
lib.mcb_version.restype = C.c_int

vp, ci, fp = C.c_void_p, C.c_int, C.POINTER(C.c_float)


class ConvFwdArgs(C.Structure):
    _fields_ = [("x", vp * 2), ("cin", ci * 2), ("n", ci), ("h", ci), ("w", ci), ("weight", vp), ("cout", ci),
                ("ksize", ci), ("stride", ci), ("bias", vp), ("relu", ci), ("stats", vp), ("y", vp), ("scale", vp),
                ("residual", vp)]


class ConvDgradArgs(C.Structure):
    _fields_ = [("dy", vp), ("n", ci), ("h", ci), ("w", ci), ("weight", vp), ("cout", ci), ("cin_total", ci),
                ("ci_off", ci), ("cin", ci), ("ksize", ci), ("stride", ci), ("dx", vp), ("relu_mask", vp),
                ("accumulate", ci), ("bn_z", vp), ("bn_mean", vp), ("bn_invstd", vp), ("bn_dbeta", vp),
                ("bn_dgamma", vp), ("bn_gamma", vp), ("bn_beta", vp), ("dx_channel_sum", vp)]


class ConvWgradArgs(C.Structure):
    _fields_ = [("dy", vp), ("x", vp), ("n", ci), ("h", ci), ("w", ci), ("cout", ci), ("cin_total", ci),
                ("ci_off", ci), ("cin", ci), ("ksize", ci), ("stride", ci), ("dw", vp)]


class ConvtFwdArgs(C.Structure):
    _fields_ = [("x", vp), ("n", ci), ("h", ci), ("w", ci), ("cin", ci), ("weight", vp), ("cout", ci), ("bias", vp),
                ("relu", ci), ("y", vp), ("ksize", ci)]


class ConvtDgradArgs(C.Structure):
    _fields_ = [("dy", vp), ("n", ci), ("h", ci), ("w", ci), ("cin", ci), ("weight", vp), ("cout", ci), ("dx", vp),
                ("relu_mask", vp), ("accumulate", ci), ("dx_channel_sum", vp), ("ksize", ci)]


class ConvtWgradArgs(C.Structure):
    _fields_ = [("dy", vp), ("x", vp), ("n", ci), ("h", ci), ("w", ci), ("cin", ci), ("cout", ci), ("dw", vp),
                ("ksize", ci)]


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("libmcb200 %s failed (%d): %s" % (what, rc, lib.mcb_last_error().decode()))


def ptr(t):
    """device pointer of a torch tensor (or None)"""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name, args=None, *extra):
    fn = getattr(lib, name)
    if args is None:
        rc = fn(*extra, stream_ptr())
    else:
        rc = fn(C.byref(args), *extra, stream_ptr())
    check(rc, name)


class LossArgs(C.Structure):
    _fields_ = [("logits", vp), ("target", vp), ("n", ci), ("h", ci), ("w", ci), ("mode", ci), ("w0", C.c_float),
                ("sigma", C.c_float), ("size_c", C.c_float), ("dice_weight", C.c_float), ("ce_weight", C.c_float),
                ("dice_smooth", C.c_float), ("dice_activation", ci)]


cl, cf = C.c_long, C.c_float
_SIGS = {
    "mcb_nchw_f32_to_nhwc_bf16": [vp, vp, ci, ci, ci, ci, vp],
    "mcb_nhwc_bf16_to_nchw_f32": [vp, vp, ci, ci, ci, ci, vp],
    "mcb_stem_im2col": [vp, vp, ci, ci, ci, vp],
    "mcb_stem_pack_weight": [vp, vp, vp],
    "mcb_stem_unpack_wgrad": [vp, vp, vp],
    "mcb_vgg_input_im2col": [vp, vp, ci, ci, ci, vp],
    "mcb_vgg_input_pack_weight": [vp, vp, vp],
    "mcb_vgg_input_unpack_wgrad": [vp, vp, vp],
    "mcb_maxpool2_bwd_skip_relu": [vp, vp, vp, vp, ci, ci, ci, ci, vp],
    "mcb_bn_finalize": [vp, cl, vp, vp, vp, vp, cf, cf, vp, vp, vp, vp, ci, vp],
    "mcb_bn_eval_params": [vp, vp, vp, vp, cf, vp, vp, ci, vp],
    "mcb_bn_apply": [vp, vp, vp, vp, vp, vp, ci, vp, cl, ci, vp],
    "mcb_bn_bwd_reduce": [vp, vp, vp, vp, vp, vp, vp, cl, ci, vp],
    "mcb_bn_bwd_apply": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, cl, ci, vp],
    "mcb_bn_bwd_apply_global": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, cl, cl, ci, vp],
    "mcb_channel_sum": [vp, vp, cl, ci, vp],
    "mcb_det_sum_f32": [vp, ci, cl, cl, cl, vp, cl, vp],
    "mcb_maxpool2_fwd": [vp, vp, ci, ci, ci, ci, vp],
    "mcb_maxpool2_bwd": [vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "mcb_final_conv_fwd": [vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "mcb_final_conv_bwd": [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "mcb_adam_step": [vp, vp, vp, vp, vp, cl, cf, C.c_double, C.c_double, cf, cf, ci, cf, vp],
    "mcb_adam_step_dyn": [vp, vp, vp, vp, vp, cl, vp, cf, cf, cf, cf, cf, vp],
    "mcb_cast_f32_bf16": [vp, vp, cl, vp],
    "mcb_loss_partials": [C.POINTER(LossArgs), vp, vp],
    "mcb_loss_grad": [C.POINTER(LossArgs), vp, cl, cf, vp, vp, vp],
    "mcb_softmax2": [vp, vp, ci, ci, ci, vp],
}
for _n, _a in _SIGS.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci
for _n in ("mcb_conv_fwd", "mcb_conv_dgrad", "mcb_conv_wgrad", "mcb_convt_fwd", "mcb_convt_dgrad", "mcb_convt_wgrad"):
    getattr(lib, _n).restype = ci


def dp(t):
    """raw device pointer (int) of a tensor, or None"""
    return None if t is None else t.data_ptr()


def fcall(name, *args):
    """call a flat-signature entry point, appending the current stream"""
    import torch
    rc = getattr(lib, name)(*args, torch.cuda.current_stream().cuda_stream)
    check(rc, name)

_SIGS2 = {
    "mcb_resize_bilinear_f64": [vp, vp, vp, ci, ci, ci, ci, ci, ci, vp],
    "mcb_threshold_layers": [vp, ci, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "mcb_ccl_label": [vp, ci, vp, vp, vp, ci, ci, ci, vp],
    "mcb_morph_rect": [vp, vp, ci, ci, ci, ci, ci, ci, vp],
    "mcb_add_dropped_objects": [vp, vp, vp, vp, ci, ci, ci, vp],
    "mcb_instance_scores": [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, vp],
}
for _n, _a in _SIGS2.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

_SIGS3 = {
    "mcb_crf_rgb_from_normalized": [vp, vp, ci, ci, ci, vp],
    "mcb_dense_crf": [vp, vp, vp, vp, ci, ci, ci, cf, cf, cf, cf, cf, ci, vp],
}
for _n, _a in _SIGS3.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

lib.mcb_watershed.argtypes = [vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, vp]
lib.mcb_watershed.restype = ci


class BNTrain(C.Structure):
    _fields_ = [("stats", vp), ("gamma", vp), ("beta", vp), ("running_mean", vp), ("running_var", vp), ("mean", vp),
                ("invstd", vp)]


lib.mcb_bn_train_apply.argtypes = [vp, C.POINTER(BNTrain), vp, C.POINTER(BNTrain), ci, vp, cl, ci, cf, cf, vp]
lib.mcb_bn_train_apply.restype = ci
lib.mcb_bn_train_apply_global.argtypes = [vp, C.POINTER(BNTrain), vp, C.POINTER(BNTrain), ci, vp, cl, cl, ci, cf, cf, vp]
lib.mcb_bn_train_apply_global.restype = ci

lib.mcb_bn_eval_params_batched.argtypes = [vp, ci, ci, cf, vp]
lib.mcb_bn_eval_params_batched.restype = ci

lib.mcb_instance_scores_strided.argtypes = [vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, vp]
lib.mcb_instance_scores_strided.restype = ci

_SIGS4 = {
    "mcb_argmax_channels": [vp, ci, vp, ci, ci, ci, ci, vp],
    "mcb_tta_transform": [vp, vp, vp, vp, ci, ci, ci, ci, vp],
    "mcb_tta_variants_u8": [vp, vp, vp, vp, ci, ci, ci, vp],
    "mcb_tta_aggregate": [vp, ci, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp],
    "mcb_instance_geometry": [vp, vp, ci, vp, vp, vp, vp, vp, ci, ci, ci, vp],
    "mcb_rle_walk": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp],
    "mcb_rle_counts": [vp, vp, vp, vp, vp, cl, ci, vp],
    "mcb_pair_intersections": [vp, vp, vp, ci, ci, ci, ci, vp],
    "mcb_contour_length": [vp, vp, vp, vp, ci, ci, ci, vp],
}
for _n, _a in _SIGS4.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

lib.mcb_zero_bytes.argtypes = [vp, C.c_size_t, vp]
lib.mcb_zero_bytes.restype = ci


def zero(t):
    """t.zero_() without a torch kernel: cudaMemsetAsync on the current stream"""
    fcall("mcb_zero_bytes", t.data_ptr(), t.numel() * t.element_size())

_SIGS5 = {
    "mcb_image_pad_normalize": [vp, vp, ci, ci, ci, ci, ci, ci, fp, fp, vp],
    "mcb_edt_two_nearest": [vp, ci, ci, ci, vp, vp, vp, vp],
    "mcb_pil_resize_bilinear_u8": [vp, vp, vp, vp, vp, ci, vp, vp, ci, ci, ci, ci, ci, ci, ci, vp],
    "mcb_size_matrix": [vp, vp, vp, ci, ci, vp],
    "mcb_target_channels": [vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, vp],
    "mcb_target_channels_u8": [vp, vp, ci, ci, ci, ci, ci, ci, ci, vp],
    "mcb_augment_warp": [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp, vp],
}
for _n, _a in _SIGS5.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

_SIGS6 = {
    "mcb_rle_pair_iou": [vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, vp],
    "mcb_iou_row_max": [vp, vp, ci, vp, vp],
    "mcb_coco_match": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ci, ci, ci, C.c_longlong, C.c_longlong, vp,
                       vp, vp, vp, vp],
}
for _n, _a in _SIGS6.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

_SIGS7 = {
    "mcb_rasterize_polygons": [vp, vp, vp, ci, C.c_longlong, vp, vp, ci, ci, ci, vp],
    "mcb_plane_stats": [vp, ci, ci, ci, ci, vp, vp],
    "mcb_plane_union": [vp, vp, vp, ci, ci, ci, vp, vp],
    "mcb_category_overlay": [vp, vp, ci, ci, ci, ci, vp, vp],
    "mcb_border_class": [vp, vp, ci, ci, ci, C.c_double, vp],
    "mcb_edt_two_nearest_batched": [vp, vp, vp, vp, ci, ci, ci, ci, vp, vp, vp, vp],
    "mcb_size_matrix_batched": [vp, vp, vp, ci, ci, ci, vp],
    "mcb_binary_morph_rect": [vp, vp, ci, ci, ci, ci, ci, vp],
}
for _n, _a in _SIGS7.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

_SIGS8 = {
    "mcb_jpeg_entropy_decode": [vp, vp, ci, vp, vp, ci, vp, vp, vp],
    "mcb_jpeg_entropy_decode_parallel": [vp, vp, ci, vp, vp, ci, vp, ci, vp, vp, vp, vp],
    "mcb_jpeg_subsequence_bits": [],
    "mcb_jpeg_idct": [vp, vp, vp, ci, ci, vp, vp],
    "mcb_jpeg_upsample_rgb": [vp, vp, vp, ci, ci, ci, vp, vp],
}
for _n, _a in _SIGS8.items():
    getattr(lib, _n).argtypes = _a
    getattr(lib, _n).restype = ci

lib.mcb_forest_predict.argtypes = [vp, ci, ci, vp, ci, vp, vp, vp, vp, vp, vp, ci, ci, vp, ci, vp, vp]
lib.mcb_forest_predict.restype = ci

lib.mcb_sync_step_bump.argtypes = [vp, vp]
lib.mcb_sync_step_bump.restype = ci
lib.mcb_sync_exchange.argtypes = [vp, vp, ci, ci, cl, cl, ci, vp, vp, vp, vp, ci, cf, vp]
lib.mcb_sync_exchange.restype = ci

