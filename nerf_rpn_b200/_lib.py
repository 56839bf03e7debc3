"""ctypes binding of libnerf_rpn_b200.so (the C ABI declared in include/nerf_rpn_b200.h).

The library is the product: if it is missing or fails to load, importing the compute path fails loudly --
there is no PyTorch / CPU fallback anywhere in this package.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libnerf_rpn_b200.so")

MAX_LEVELS = 4
MAX_TAPS = 64

c_f32p = ctypes.c_void_p
c_stream = ctypes.c_void_p


class ConvLevel(ctypes.Structure):
    _fields_ = [("x", ctypes.c_void_p), ("y", ctypes.c_void_p), ("res", ctypes.c_void_p), ("n", ctypes.c_int32),
                ("xi", ctypes.c_int32), ("yi", ctypes.c_int32), ("zi", ctypes.c_int32),
                ("xo", ctypes.c_int32), ("yo", ctypes.c_int32), ("zo", ctypes.c_int32),
                ("xr", ctypes.c_int32), ("yr", ctypes.c_int32), ("zr", ctypes.c_int32),
                ("ldy", ctypes.c_int32), ("ldr", ctypes.c_int32)]


class ConvDesc(ctypes.Structure):
    _fields_ = [("cin", ctypes.c_int32), ("cout", ctypes.c_int32), ("n_taps", ctypes.c_int32),
                ("tap_off", (ctypes.c_int8 * 3) * MAX_TAPS), ("stride", ctypes.c_int32), ("relu", ctypes.c_int32),
                ("out_fp32", ctypes.c_int32), ("w", ctypes.c_void_p), ("shift", ctypes.c_void_p),
                ("n_levels", ctypes.c_int32), ("level", ConvLevel * MAX_LEVELS), ("act_fp16", ctypes.c_int32),
                ("wsplit", ctypes.c_int32)]


class RpnLevel(ctypes.Structure):
    _fields_ = [("pred", ctypes.c_void_p), ("ld", ctypes.c_int32), ("gx", ctypes.c_int32), ("gy", ctypes.c_int32),
                ("gz", ctypes.c_int32), ("sx", ctypes.c_int32), ("sy", ctypes.c_int32), ("sz", ctypes.c_int32)]


class RpnDesc(ctypes.Structure):
    _fields_ = [("n_levels", ctypes.c_int32), ("level", RpnLevel * MAX_LEVELS), ("num_anchors", ctypes.c_int32),
                ("cell_anchors", ((ctypes.c_float * 6) * 16) * MAX_LEVELS), ("rotated", ctypes.c_int32),
                ("pre_nms_top_n", ctypes.c_int32), ("post_nms_top_n", ctypes.c_int32), ("nms_thresh", ctypes.c_float),
                ("score_thresh", ctypes.c_float), ("min_size", ctypes.c_float), ("mesh", ctypes.c_int32 * 3),
                ("valid", ctypes.c_int32 * 3)]


class WgradLevel(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int32), ("x", ctypes.c_int32), ("y", ctypes.c_int32), ("z", ctypes.c_int32),
                ("dy_cl", ctypes.c_void_p), ("x_cl", ctypes.c_void_p), ("ld_dy", ctypes.c_int32), ("ld_x", ctypes.c_int32),
                ("xx", ctypes.c_int32), ("xy", ctypes.c_int32), ("xz", ctypes.c_int32)]


class WgradDesc(ctypes.Structure):
    _fields_ = [("cin", ctypes.c_int32), ("cout", ctypes.c_int32), ("n_taps", ctypes.c_int32),
                ("tap_off", (ctypes.c_int8 * 3) * MAX_TAPS), ("n_levels", ctypes.c_int32), ("level", WgradLevel * MAX_LEVELS),
                ("dw", ctypes.c_void_p), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_size_t),
                ("act_fp16", ctypes.c_int32), ("dw_layout", ctypes.c_int32)]


class StemSrc(ctypes.Structure):
    """nrpn_stem_src: one scene for nrpn_pack_stem_input, with its layout (STEM_F32_NCDHW, STEM_F32_XYZC or STEM_U8_XYZC)."""
    _fields_ = [("grid", ctypes.c_void_p), ("x", ctypes.c_int32), ("y", ctypes.c_int32), ("z", ctypes.c_int32), ("layout", ctypes.c_int32)]


STEM_MAX_SCENES = 32
STEM_F32_NCDHW, STEM_F32_XYZC, STEM_U8_XYZC = 0, 1, 2


class GnLevel(ctypes.Structure):
    _fields_ = [("x", ctypes.c_void_p), ("voxels", ctypes.c_int32)]


class FcosLevel(ctypes.Structure):
    _fields_ = [("cls", ctypes.c_void_p), ("reg", ctypes.c_void_p), ("ld_cls", ctypes.c_int32), ("ld_reg", ctypes.c_int32),
                ("gx", ctypes.c_int32), ("gy", ctypes.c_int32), ("gz", ctypes.c_int32), ("stride", ctypes.c_int32),
                ("scale", ctypes.c_float)]


class FcosDesc(ctypes.Structure):
    _fields_ = [("n_levels", ctypes.c_int32), ("level", FcosLevel * MAX_LEVELS), ("use_obb", ctypes.c_int32),
                ("pre_nms_top_n", ctypes.c_int32), ("post_nms_top_n", ctypes.c_int32), ("pre_nms_thresh", ctypes.c_float),
                ("nms_thresh", ctypes.c_float), ("min_size", ctypes.c_float), ("grid_size", ctypes.c_int32 * 3),
                ("padded", ctypes.c_int32)]


class FcosTargetDesc(ctypes.Structure):
    _fields_ = [("n_levels", ctypes.c_int32), ("n_points", ctypes.c_int32 * MAX_LEVELS), ("stride", ctypes.c_int32 * MAX_LEVELS),
                ("size_lo", ctypes.c_float * MAX_LEVELS), ("size_hi", ctypes.c_float * MAX_LEVELS),
                ("center_sampling_radius", ctypes.c_float), ("norm_reg_targets", ctypes.c_int32)]


class FcosLossLevel(ctypes.Structure):
    _fields_ = [("cls", ctypes.c_void_p), ("reg", ctypes.c_void_p), ("ctr", ctypes.c_void_p), ("dcls", ctypes.c_void_p),
                ("dreg", ctypes.c_void_p), ("dctr", ctypes.c_void_p), ("n_points", ctypes.c_int32)]


class FcosLossDesc(ctypes.Structure):
    _fields_ = [("n_levels", ctypes.c_int32), ("level", FcosLossLevel * MAX_LEVELS), ("n_images", ctypes.c_int32),
                ("use_obb", ctypes.c_int32), ("loss_type", ctypes.c_int32), ("additional_l1", ctypes.c_int32)]


_SIGNATURES = {
    "nrpn_version": (ctypes.c_int, []),
    "nrpn_status_string": (ctypes.c_char_p, [ctypes.c_int]),
    "nrpn_last_cuda_error": (ctypes.c_int, []),
    "nrpn_launch_count": (ctypes.c_ulonglong, []),
    "nrpn_iou3d_pairs": (ctypes.c_int, [c_f32p, c_f32p, ctypes.c_int, ctypes.c_int, c_f32p, c_stream]),
    "nrpn_iou3d_pairs_verbose": (ctypes.c_int, [c_f32p, c_f32p, ctypes.c_int, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_stream]),
    "nrpn_iou3d_pairs_backward": (ctypes.c_int, [c_f32p, c_f32p, ctypes.c_int, c_f32p, c_f32p, c_f32p, c_f32p, c_stream]),
    "nrpn_iou3d_matrix": (ctypes.c_int, [c_f32p, ctypes.c_int, c_f32p, ctypes.c_int, ctypes.c_int, c_f32p, c_stream]),
    "nrpn_sort_vertices": (ctypes.c_int, [c_f32p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_void_p, c_stream]),
    "nrpn_set_iou_mode": (ctypes.c_int, [ctypes.c_int]),
    "nrpn_get_iou_mode": (ctypes.c_int, []),
    "nrpn_nms_max_boxes": (ctypes.c_int, []),
    "nrpn_nms_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int]),
    "nrpn_nms": (ctypes.c_int, [c_f32p, ctypes.c_int, c_f32p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float,
                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_conv3d_block_n": (ctypes.c_int, [ctypes.c_int]),
    "nrpn_conv3d_variant": (ctypes.c_char_p, [ctypes.POINTER(ConvDesc)]),
    "nrpn_conv3d_fprop": (ctypes.c_int, [ctypes.POINTER(ConvDesc), c_stream]),
    "nrpn_conv3d_wgrad_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(WgradDesc)]),
    "nrpn_conv3d_wgrad_variant": (ctypes.c_char_p, [ctypes.POINTER(WgradDesc)]),
    "nrpn_conv3d_wgrad": (ctypes.c_int, [ctypes.POINTER(WgradDesc), c_stream]),
    "nrpn_bias_grad_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int]),
    "nrpn_bias_grad": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_f32p, ctypes.c_void_p,
                                      ctypes.c_size_t, c_stream]),
    "nrpn_relu_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, c_stream]),
    "nrpn_pack_stem_input": (ctypes.c_int, [ctypes.POINTER(StemSrc), ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, c_stream]),
    "nrpn_maxpool3d_k3s2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_maxpool3d_k2s2_ceil": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_pack_stem_input_s1": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_groupnorm_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    "nrpn_groupnorm_relu": (ctypes.c_int, [ctypes.POINTER(GnLevel), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           c_f32p, c_f32p, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_patch_embed_pack": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_layernorm": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_int,
                                      c_f32p, c_f32p, ctypes.c_float, ctypes.c_int, c_stream]),
    "nrpn_patch_merge_ln": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_void_p, c_f32p, c_f32p, ctypes.c_float, ctypes.c_int, c_stream]),
    "nrpn_window_attention": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_f32p, c_f32p, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_stream]),
    "nrpn_fcos_max_proposals": (ctypes.c_int, [ctypes.POINTER(FcosDesc)]),
    "nrpn_fcos_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(FcosDesc)]),
    "nrpn_fcos_proposals": (ctypes.c_int, [ctypes.POINTER(FcosDesc), c_f32p, c_f32p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_size_t, c_stream]),
    "nrpn_assign_targets_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    "nrpn_assign_targets": (ctypes.c_int, [c_f32p, ctypes.c_int, c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_float,
                                           ctypes.c_float, ctypes.c_int, c_f32p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_anchor_padding_mask": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                ctypes.c_int, ctypes.c_int, ctypes.c_void_p, c_stream]),
    "nrpn_rowmax_f32": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, c_f32p, ctypes.c_void_p, c_stream]),
    "nrpn_recall_match": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, c_f32p, c_stream]),
    # ---- training step (csrc/train.cu)
    "nrpn_chan_reduce_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int]),
    "nrpn_bn_stats": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_float, c_f32p, c_f32p, c_f32p,
                                     ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_bn_apply": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long, ctypes.c_int, c_f32p, c_f32p, c_f32p,
                                     ctypes.c_int, ctypes.c_int, c_stream]),
    "nrpn_bn_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long,
                                        ctypes.c_int, c_f32p, c_f32p, c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_maxpool3d_k3s2_argmax": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_maxpool3d_k3s2_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_maxpool3d_k2s2_ceil_argmax": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_maxpool3d_k2s2_ceil_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                         ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_upsample_nearest_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                      ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, c_stream]),
    "nrpn_stride2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, c_stream]),
    "nrpn_add_inplace": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, c_stream]),
    "nrpn_rpn_loss": (ctypes.c_int, [ctypes.POINTER(RpnDesc), ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_int, c_f32p, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, c_f32p, c_f32p,
                                     ctypes.c_int, c_stream]),
    "nrpn_pack_weights": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_stream]),
    "nrpn_gather_pack": (ctypes.c_int, [c_f32p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, c_f32p, ctypes.c_int, c_stream]),
    "nrpn_grad_norm_workspace_bytes": (ctypes.c_size_t, []),
    "nrpn_grad_norm": (ctypes.c_int, [c_f32p, ctypes.c_size_t, ctypes.c_float, c_f32p, ctypes.c_void_p, ctypes.c_size_t, c_stream]),
    "nrpn_adamw_step": (ctypes.c_int, [c_f32p, c_f32p, c_f32p, c_f32p, ctypes.c_size_t, c_f32p, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                       ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int, c_stream]),
    "nrpn_fcos_targets": (ctypes.c_int, [ctypes.POINTER(FcosTargetDesc), c_f32p, c_f32p, ctypes.c_int, ctypes.c_int, c_f32p, c_f32p, c_stream]),
    "nrpn_fcos_loss_workspace_bytes": (ctypes.c_size_t, []),
    "nrpn_fcos_loss": (ctypes.c_int, [ctypes.POINTER(FcosLossDesc), c_f32p, c_f32p, ctypes.c_void_p, c_f32p, ctypes.c_void_p, ctypes.c_void_p,
                                      ctypes.c_size_t, c_stream]),
    "nrpn_set_nms_cull_mode": (None, [ctypes.c_int]),
    "nrpn_get_nms_cull_mode": (ctypes.c_int, []),
    "nrpn_nms_cells_stats": (ctypes.c_int, [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]),
    "nrpn_augment_scene": (ctypes.c_int, [c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_float, ctypes.c_float, c_stream]),
    "nrpn_rpn_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(RpnDesc)]),
    "nrpn_rpn_proposals": (ctypes.c_int, [ctypes.POINTER(RpnDesc), c_f32p, c_f32p, c_f32p, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_size_t, c_stream]),
}

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib():
    """Load the native library (once). Raises NativeLibraryError if it is missing: build it with `make`."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} not found: the CUDA extension is required (run `make` or __graft_entry__.build()); "
                "nerf_rpn_b200 has no CPU / PyTorch fallback")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)       # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def check(status, what=""):
    if status != 0:
        L = lib()
        msg = L.nrpn_status_string(status).decode()
        raise RuntimeError(f"nerf_rpn_b200: {what} failed: {msg} (status {status}, cuda error {L.nrpn_last_cuda_error()})")
