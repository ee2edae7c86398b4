"""ctypes binding of libhipie_b200.so (the C-ABI declared in include/hipie_b200.h).

Fails loudly: no library -> RuntimeError, no silent fallback of any kind.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhipie_b200.so")

_lib = None

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_int64 = ctypes.c_int64
c_float = ctypes.c_float
c_double = ctypes.c_double


class GemmArgs(ctypes.Structure):
    _fields_ = [
        ("a_hi", c_void_p), ("a_lo", c_void_p), ("lda", c_int64), ("a_bstride", c_int64),
        ("w_hi", c_void_p), ("w_lo", c_void_p), ("ldw", c_int64), ("w_bstride", c_int64),
        ("bias", c_void_p), ("colscale", c_void_p), ("residual", c_void_p),
        ("ldr", c_int64), ("r_bstride", c_int64),
        ("c_f32", c_void_p), ("c_hi", c_void_p), ("c_lo", c_void_p), ("ldc", c_int64), ("c_bstride", c_int64),
        ("c_bits", c_void_p), ("bits_threshold", c_float),
        ("M", c_int), ("N", c_int), ("K", c_int), ("batch", c_int),
        ("act", c_int), ("prec", c_int), ("alpha", c_float), ("transposed", c_int), ("c_row_map", c_void_p),
        ("t_row_group", c_int), ("t_row_pad", c_int), ("relu_after_residual", c_int), ("c_fp16", c_int),
        ("a8", c_void_p), ("lda8", c_int64), ("w8", c_void_p), ("ldw8", c_int64), ("c8", c_void_p), ("ldc8", c_int64),
    ]


class AttnArgs(ctypes.Structure):
    _fields_ = [
        ("q_hi", c_void_p), ("q_lo", c_void_p), ("k_hi", c_void_p), ("k_lo", c_void_p),
        ("v_hi", c_void_p), ("v_lo", c_void_p),
        ("q_bs", c_int64), ("q_ts", c_int64), ("q_hs", c_int64),
        ("k_bs", c_int64), ("k_ts", c_int64), ("k_hs", c_int64),
        ("v_bs", c_int64), ("v_ts", c_int64), ("v_hs", c_int64),
        ("rel_h", c_void_p), ("rel_w", c_void_p), ("kh", c_int), ("kw", c_int),
        ("key_bias", c_void_p),
        ("out_f32", c_void_p), ("out_hi", c_void_p), ("out_lo", c_void_p), ("o_bs", c_int64), ("o_ts", c_int64),
        ("B", c_int), ("H", c_int), ("Tq", c_int), ("Tk", c_int), ("hd", c_int),
        ("scale", c_float), ("prec", c_int), ("key_mask", c_void_p),
    ]


# name -> (restype, argtypes); every symbol include/hipie_b200.h declares
SYMBOLS = {
    "hipie_last_error": (ctypes.c_char_p, []),
    "hipie_abi_version": (c_int, []),
    "hipie_launch_count": (c_int64, []),
    "hipie_set_option": (c_int, [ctypes.c_char_p, c_int]),
    "hipie_msda_forward": (c_int, [c_void_p] * 6 + [c_int] * 9 + [c_void_p]),
    "hipie_msda_fused_forward": (c_int, [c_void_p] * 5 + [c_int, c_void_p] + [c_int] * 9 + [c_void_p, c_void_p]),
    "hipie_msda_encoder_forward": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p, c_int, c_void_p]),
    "hipie_gemm": (c_int, [ctypes.POINTER(GemmArgs), c_void_p]),
    "hipie_split_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "hipie_layernorm": (c_int, [c_void_p] * 4 + [c_float] + [c_void_p] * 4 + [c_int64, c_int, c_void_p, c_void_p]),
    "hipie_layernorm_f16": (c_int, [c_void_p] * 4 + [c_float] + [c_void_p] * 4 + [c_int64, c_int, c_void_p, c_void_p]),
    "hipie_split_f16_e4m3": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "hipie_groupnorm_nhwc": (c_int, [c_void_p] * 3 + [c_float] + [c_void_p] * 5 + [c_int] * 5 + [c_int64] * 3 + [c_void_p]),
    "hipie_add_split": (c_int, [c_void_p] * 5 + [c_int64, c_void_p]),
    "hipie_patchify": (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_void_p] * 3),
    "hipie_im2col_nhwc": (c_int, [c_void_p] * 3 + [c_int] * 7 + [c_void_p]),
    "hipie_pixel_shuffle2": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_void_p]),
    "hipie_maxpool2_nhwc": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_void_p]),
    "hipie_maxpool3x3s2_nhwc": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_void_p]),
    "hipie_row_softmax": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "hipie_attention": (c_int, [ctypes.POINTER(AttnArgs), c_void_p]),
    "hipie_attention_tc": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int,
                                   c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                   c_int64, c_int64, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "hipie_attention_tc_planes": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int,
                                   c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                   c_int64, c_int64, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "hipie_relpos_bias": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int, c_int, c_int,
                                  c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hipie_relpos_bias_tc": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int, c_int, c_int,
                                     c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hipie_relpos_bias_tc_f16": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hipie_condinst_masks": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_void_p]),
    "hipie_seg_postprocess": (c_int, [c_void_p] * 7 + [c_int] * 8 + [c_void_p]),
    "hipie_sine_embed": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "hipie_upsample_threshold": (c_int, [c_void_p] * 2 + [c_int] * 6 + [c_float, c_void_p]),
    "hipie_class_scores": (c_int, [c_void_p] * 9 + [c_int] * 5 + [c_void_p]),
    "hipie_batched_nms": (c_int, [c_void_p] * 5 + [c_int, c_int, c_float, c_void_p]),
    "hipie_nms_sorted": (c_int, [c_void_p, c_int, c_float, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "hipie_topk": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "hipie_maskclip_patch_mask": (c_int, [c_void_p] + [c_int] * 8 + [c_void_p, c_int, c_int, c_void_p]),
    "hipie_clip_patches": (c_int, [c_void_p] + [c_int] * 4 + [c_void_p] * 4 + [c_int, c_void_p]),
    "hipie_clip_fuse": (c_int, [c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p, c_float, c_void_p, c_float, c_float, c_int,
                                c_void_p, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "hipie_sam_attention": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_int64, c_int64] + [c_int] * 5 + [c_float, c_void_p]),
    "hipie_sam_masks": (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
    "hipie_sam_mask_embed": (c_int, [c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "hipie_sam_postprocess": (c_int, [c_void_p] + [c_int] * 4 + [c_void_p] * 3 + [c_int64, c_void_p, c_void_p]),
    "hipie_sam_upscale": (c_int, [c_void_p] + [c_int] * 8 + [c_float] + [c_void_p] * 3),
    "hipie_sam_mask_stats": (c_int, [c_void_p] + [c_int] * 8 + [c_double, c_double, c_void_p, c_void_p]),
    "hipie_sam_mask_emit": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_float, c_void_p, c_void_p]),
    "hipie_part_assign": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 5),
    "hipie_part_masks": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "hipie_label_cover": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p] * 3),
    "hipie_sam_vote": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p] + [c_int] * 4 + [c_void_p] * 5),
    "hipie_semseg_confusion": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p, c_int] + [c_void_p] * 3),
    "hipie_panoptic_pairs": (c_int, [c_void_p] * 2 + [c_int] * 2 + [c_void_p] + [c_int] * 2 + [c_void_p] * 3),
    "hipie_mask_words": (c_int64, [c_int, c_int]),
    "hipie_mask_pack": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p] * 3),
    "hipie_rle_expand": (c_int, [c_void_p] * 2 + [c_int] * 3 + [c_void_p] * 3),
    "hipie_mask_overlaps": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 3 + [c_void_p] * 2),
}


def load():
    """Load the shared library (once).  Raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"hipie_b200: {LIB_PATH} is missing — run `python -m hipie_b200.build` (or __graft_entry__.build()). "
            "There is no CPU / PyTorch fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().hipie_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hipie_b200 {what} failed (code {rc}): {msg}")


def set_option(name: str, value: int):
    check(load().hipie_set_option(name.encode(), int(value)), f"set_option({name})")


def launch_count():
    return int(load().hipie_launch_count())
