"""ctypes binding of libosvos_b200.so (the C ABI declared in include/osvos_b200.h).

This is the stub a maintainer of the reference would add to call the native hot
path from Python (INTEGRATION.md).  There is deliberately NO fallback: if the
library cannot be loaded, or a call fails, an exception is raised.
"""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_size_t, c_uint8, c_uint32,
                    c_uint64, c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libosvos_b200.so")

FLAG_RELU = 1
FLAG_FAST = 2
FLAG_RELU_MASK = 4
FLAG_ACCUMULATE = 8
FLAG_DEFER_FINISH = 16
FLAG_DETERMINISTIC = 32
FLAG_VOID_LABELS = 64
WGRAD_FINISH_MAX = 24


class NativeLibraryError(RuntimeError):
    pass


class Conv3x3Args(Structure):
    _fields_ = [("x_hi", c_void_p), ("x_lo", c_void_p), ("w_packed", c_void_p), ("bias", c_void_p),
                ("y_hi", c_void_p), ("y_lo", c_void_p), ("y_f32", c_void_p), ("mask_hi", c_void_p),
                ("proj_w", c_void_p), ("proj_b", c_void_p), ("pq", c_void_p),
                ("pool_hi", c_void_p), ("pool_lo", c_void_p), ("colsum", c_void_p),
                ("n", c_int), ("h", c_int), ("w", c_int), ("cin", c_int), ("cout", c_int), ("flags", c_int)]


class Stage1Args(Structure):
    _fields_ = [("x", c_void_p), ("w1", c_void_p), ("b1", c_void_p), ("w2_packed", c_void_p), ("b2", c_void_p),
                ("y_hi", c_void_p), ("y_lo", c_void_p), ("pool_hi", c_void_p), ("pool_lo", c_void_p),
                ("n", c_int), ("h", c_int), ("w", c_int)]


class TailFwdArgs(Structure):
    _fields_ = [("pq", c_void_p * 4), ("fuse_bias", c_void_p), ("out", c_void_p * 5), ("label", c_void_p),
                ("sums", c_void_p), ("losses", c_void_p), ("loss_weights", c_float * 5), ("divisor", c_float),
                ("n", c_int), ("h", c_int), ("w", c_int), ("flags", c_int)]


TAIL_SUMS = 15


class TailLossBwdArgs(Structure):
    _fields_ = [("logits", c_void_p * 5), ("label", c_void_p), ("sums", c_void_p), ("upstream", c_void_p),
                ("loss_weights", c_float * 5), ("divisor", c_float), ("dpq", c_void_p * 4), ("fuse_bias_grad", c_void_p),
                ("n", c_int), ("h", c_int), ("w", c_int), ("flags", c_int)]


class WgradArgs(Structure):
    _fields_ = [("x_hi", c_void_p), ("x_lo", c_void_p), ("dz_hi", c_void_p), ("dz_lo", c_void_p), ("dw", c_void_p),
                ("workspace", c_void_p), ("n", c_int), ("h", c_int), ("w", c_int), ("cin", c_int), ("cout", c_int),
                ("dz_channels", c_int), ("flags", c_int)]


class WgradFinishItem(Structure):
    _fields_ = [("workspace", c_void_p), ("dw", c_void_p), ("cout", c_int), ("cin", c_int), ("dz_channels", c_int),
                ("accumulate", c_int), ("scale", c_float)]


class FoldItem(Structure):
    """osvos_fold_item (include/osvos_b200.h)."""
    _fields_ = [("side_w", c_void_p), ("side_b", c_void_p), ("proj_w", c_void_p), ("proj_b", c_void_p),
                ("packed", c_void_p), ("bias2", c_void_p), ("folded_f32", c_void_p), ("cin", c_int)]


class SideWgradItem(Structure):
    """osvos_side_wgrad_item (include/osvos_b200.h)."""
    _fields_ = [("x_hi", c_void_p), ("x_lo", c_void_p), ("dpq", c_void_p), ("g", c_void_p), ("n", c_int), ("h", c_int),
                ("w", c_int), ("c", c_int)]


class SideGradsItem(Structure):
    """osvos_side_grads_item (include/osvos_b200.h)."""
    _fields_ = [("g", c_void_p), ("side_w", c_void_p), ("side_b", c_void_p), ("proj_w", c_void_p),
                ("d_side_w", c_void_p), ("d_side_b", c_void_p), ("d_score_w", c_void_p), ("d_score_b", c_void_p),
                ("d_fuse_w", c_void_p), ("c", c_int), ("accumulate", c_int)]


class TailBwdArgs(Structure):
    _fields_ = [("grad_out", c_void_p * 5), ("dpq", c_void_p * 4), ("n", c_int), ("h", c_int), ("w", c_int),
                ("flags", c_int)]


class SgdSegment(Structure):
    """osvos_sgd_segment (include/osvos_b200.h); 80 bytes, uploaded as a device table."""
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("momentum", c_void_p), ("numel", c_uint64),
                ("lr", c_float), ("weight_decay", c_float), ("momentum_coef", c_float),
                ("cout", c_int32), ("cin", c_int32), ("colp_fwd", c_int32), ("colp_flip", c_int32),
                ("work_items", c_uint32), ("packed_fwd", c_void_p), ("packed_flip", c_void_p)]


class JpegArgs(Structure):
    """osvos_jpeg_args (include/osvos_b200.h)."""
    _fields_ = [("blob", c_void_p), ("blob_bytes", c_size_t), ("out", c_void_p), ("status", c_void_p),
                ("workspace", c_void_p), ("n", c_int), ("h", c_int), ("w", c_int), ("nseg", c_int),
                ("chunk_bits", c_int), ("reserved", c_int)]


class PngDecodeArgs(Structure):
    """osvos_png_decode_args (include/osvos_b200.h)."""
    _fields_ = [("blob", c_void_p), ("blob_bytes", c_size_t), ("out", c_void_p), ("status", c_void_p),
                ("workspace", c_void_p), ("path", c_void_p), ("n", c_int), ("h", c_int), ("w", c_int), ("nseg", c_int)]


class UpsamplingFoldArgs(Structure):
    """osvos_upsampling_fold_args (include/osvos_b200.h)."""
    _fields_ = [("upscale_w", c_void_p * 4), ("upscale1_w", c_void_p * 4), ("fuse_w", c_void_p), ("vtab", c_void_p),
                ("atab", c_void_p)]


class TailGeneralFwdArgs(Structure):
    """osvos_tail_general_fwd_args (include/osvos_b200.h)."""
    _fields_ = [("feat", c_void_p * 4), ("pq", c_void_p * 4), ("vtab", c_void_p), ("atab", c_void_p),
                ("fuse_bias", c_void_p), ("out", c_void_p * 5), ("label", c_void_p), ("sums", c_void_p),
                ("losses", c_void_p), ("loss_weights", c_float * 5), ("divisor", c_float), ("n", c_int), ("h", c_int),
                ("w", c_int), ("flags", c_int)]


class TailGeneralBwdArgs(Structure):
    """osvos_tail_general_bwd_args (include/osvos_b200.h)."""
    _fields_ = [("feat", c_void_p * 4), ("pq", c_void_p * 4), ("score_w", c_void_p * 4), ("vtab", c_void_p),
                ("atab", c_void_p), ("src", c_void_p * 5), ("label", c_void_p), ("sums", c_void_p),
                ("upstream", c_void_p), ("loss_weights", c_float * 5), ("divisor", c_float), ("df_hi", c_void_p * 4),
                ("df_lo", c_void_p * 4), ("red", c_void_p * 4), ("fuse_bias_grad", c_void_p), ("workspace", c_void_p),
                ("n", c_int), ("h", c_int), ("w", c_int), ("flags", c_int)]


class UpsamplingGradsArgs(Structure):
    """osvos_upsampling_grads_args (include/osvos_b200.h)."""
    _fields_ = [("red", c_void_p * 4), ("upscale_w", c_void_p * 4), ("fuse_w", c_void_p), ("d_upscale_w", c_void_p * 4),
                ("d_upscale1_w", c_void_p * 4), ("d_fuse_w", c_void_p), ("d_score_w", c_void_p * 4),
                ("d_score_b", c_void_p * 4), ("d_side_b", c_void_p * 4), ("accumulate", c_int)]


OVERLAY_MAX_COLORS = 256


class OverlayColors(Structure):
    """osvos_overlay_colors (include/osvos_b200.h): BGR triples, entry k the colour of object id k."""
    _fields_ = [("bgr", c_uint8 * (3 * OVERLAY_MAX_COLORS))]


UPSAMPLING_TAPS = 1360
U8_PROB, U8_BYTESCALE, U8_MASK = 0, 1, 2
RESIZE_BILINEAR, RESIZE_NEAREST = 0, 1
SGD_MAX_SEGMENTS = 64

# name -> (restype, argtypes); mirrors include/osvos_b200.h one to one (tests/test_abi.py checks it)
SIGNATURES = {
    "osvos_version": (c_int, []),
    "osvos_last_error": (c_char_p, []),
    "osvos_packed_weight_bytes": (c_size_t, [c_int, c_int]),
    "osvos_pack_conv3x3_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_nchw_to_act": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_act_to_nchw": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_conv_first_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                     c_void_p]),
    "osvos_conv3x3": (c_int, [POINTER(Conv3x3Args), c_void_p]),
    "osvos_stage1_fused": (c_int, [POINTER(Stage1Args), c_void_p]),
    "osvos_set_pdl": (c_int, [c_int]),
    "osvos_side_folded_multi": (c_int, [POINTER(Conv3x3Args), c_int, c_void_p]),
    "osvos_fold_side_weights_multi": (c_int, [POINTER(FoldItem), c_int, c_void_p]),
    "osvos_conv3x3_simt": (c_int, [POINTER(Conv3x3Args), c_void_p]),
    "osvos_maxpool2x2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_tail_fwd": (c_int, [POINTER(TailFwdArgs), c_void_p]),
    "osvos_cbce_fwd_sums": (c_size_t, [c_size_t, c_int]),
    "osvos_cbce_fwd": (c_int, [c_void_p, c_void_p, c_size_t, c_double, c_void_p, c_void_p, c_int, c_void_p]),
    "osvos_cbce_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_size_t, c_void_p, c_void_p]),
    "osvos_cbce_bwd_void": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_size_t, c_void_p, c_void_p]),
    "osvos_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "osvos_conv3x3_wgrad": (c_int, [POINTER(WgradArgs), c_void_p]),
    "osvos_wgrad_finish": (c_int, [POINTER(WgradFinishItem), POINTER(c_int), c_int, c_int, c_void_p]),
    "osvos_tail_bwd": (c_int, [POINTER(TailBwdArgs), c_void_p]),
    "osvos_tail_loss_bwd": (c_int, [POINTER(TailLossBwdArgs), c_void_p]),
    "osvos_sum_f32_scratch_bytes": (c_size_t, [c_int]),
    "osvos_sum_f32": (c_int, [c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_void_p]),
    "osvos_unpool_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_side_folded_wgrad_floats": (c_size_t, [c_int]),
    "osvos_side_folded_wgrad_workspace_bytes": (c_size_t, [POINTER(SideWgradItem), c_int, c_int]),
    "osvos_side_folded_wgrad_multi": (c_int, [POINTER(SideWgradItem), c_int, c_void_p, c_int, c_void_p]),
    "osvos_side_grads_finish": (c_int, [POINTER(SideGradsItem), c_int, c_void_p]),
    "osvos_conv_first_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "osvos_conv_first_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                     c_int, c_void_p]),
    "osvos_side_project": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osvos_logits_to_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_size_t, c_int, c_void_p]),
    "osvos_sgd_work_items": (c_uint32, [c_uint64, c_int, c_int]),
    "osvos_sgd_step": (c_int, [c_void_p, c_int, c_uint32, c_int, c_void_p]),
    "osvos_affine_warp": (c_int, [c_void_p, c_void_p, POINTER(c_double), POINTER(c_int), c_int, c_int, c_int, c_int,
                                  c_int, c_void_p]),
    "osvos_image_from_bgr8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float, c_float, c_void_p]),
    "osvos_label_stats_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osvos_label_from_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osvos_affine_warp_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_double), POINTER(c_int),
                                     c_int, c_int, c_int, c_float, c_float, c_float, c_void_p]),
    "osvos_affine_warp_u8_indexed": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int),
                                             POINTER(c_double), POINTER(c_int), c_int, c_int, c_int, c_int, c_float,
                                             c_float, c_float, c_void_p]),
    "osvos_labels_from_ids": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_affine_warp_ids": (c_int, [c_void_p, c_void_p, POINTER(c_int), POINTER(c_double), POINTER(c_int), c_int,
                                      c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_resize_u8_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "osvos_resize_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_resize_f32_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "osvos_resize_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_davis_measures_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "osvos_davis_measures": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "osvos_reduce_rows_scratch_floats": (c_size_t, [c_int, c_int]),
    "osvos_reduce_rows": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "osvos_conv3x3_colsum_rows": (c_size_t, [c_int, c_int, c_int]),
    "osvos_wgrad_deterministic_splits": (c_int, [c_int, c_int, c_int, c_int, c_int]),
    "osvos_unpool_colsum_rows": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "osvos_tail_fwd_deterministic_sums": (c_size_t, [c_int, c_int, c_int]),
    "osvos_tail_fwd_sums": (c_size_t, [c_int, c_int, c_int, c_int]),
    "osvos_jpeg_decode_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_size_t, c_int]),
    "osvos_jpeg_decode": (c_int, [POINTER(JpegArgs), c_void_p]),
    "osvos_upsampling_fold": (c_int, [POINTER(UpsamplingFoldArgs), c_void_p]),
    "osvos_tail_general_fwd_sums": (c_size_t, [c_int, c_int, c_int]),
    "osvos_tail_general_fwd": (c_int, [POINTER(TailGeneralFwdArgs), c_void_p]),
    "osvos_tail_general_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "osvos_tail_general_bwd": (c_int, [POINTER(TailGeneralBwdArgs), c_void_p]),
    "osvos_upsampling_grads_finish": (c_int, [POINTER(UpsamplingGradsArgs), c_void_p]),
    # train_online.py:187 (sm.imsave of each result) on the device
    "osvos_png_max_bytes": (c_size_t, [c_int, c_int]),
    "osvos_png_encode_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "osvos_png_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "osvos_png_decode_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_size_t]),
    "osvos_png_decode": (c_int, [POINTER(PngDecodeArgs), c_void_p]),
    # DAVIS-2017: palette label files, the merge of per-object maps and per-object measures (DESIGN.md §24)
    "osvos_png_max_bytes_palette": (c_size_t, [c_int, c_int, c_int]),
    "osvos_png_encode_palette": (c_int, [c_void_p, c_char_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_void_p]),
    "osvos_merge_objects": (c_int, [POINTER(c_void_p), c_int, c_void_p, c_size_t, c_void_p]),
    "osvos_upsample_merge_objects_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "osvos_upsample_merge_objects": (c_int, [POINTER(c_void_p), c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                             c_int, c_void_p]),
    "osvos_davis_measures_objects_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "osvos_davis_measures_objects": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                             c_void_p]),
    # helpers.py:15-40 overlay_mask and the vis_res display of train_online.py:160-205, written as JPEG files
    "osvos_overlay_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    # the same picture for a label map of K objects, each in its palette colour (DESIGN.md §25)
    "osvos_overlay_labels": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(OverlayColors), c_int,
                                     c_void_p]),
    "osvos_jpeg_max_bytes": (c_size_t, [c_int, c_int]),
    "osvos_jpeg_encode_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "osvos_jpeg_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
}

DAVIS_MAX_RADIUS = 31
DAVIS_MAX_OBJECTS = 254

_lib = None


def load():
    """Load the shared library once; raise NativeLibraryError if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} not found: build it with `python -m osvos_pytorch_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU / PyTorch fallback for the OSVOS hot path.")
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise NativeLibraryError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().osvos_last_error()
        raise NativeLibraryError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()
