"""ctypes binding of liblseg_b200.so (the C ABI declared in include/lseg_b200.h).

This is the reference-side FFI stub: plain pointers and sizes, no torch types cross the boundary
(torch only provides device memory and the current stream). There is no CPU fallback: if the
shared library is missing it is built with nvcc; if that fails, importing fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblseg_b200.so")

VIT_DEPTH = 24
TEXT_DEPTH = 12
ABI_VERSION = 4  # == LSEG_B200_ABI_VERSION of include/lseg_b200.h; the struct mirrors below follow that layout

ACT_NONE, ACT_GELU, ACT_QUICKGELU, ACT_RELU = 0, 1, 2, 3
HEAD_ACT = {"none": 0, "relu": 1, "lrelu": 2, "tanh": 3}
STORE_ROWMAJOR, STORE_D2S, STORE_NCHW_T = 0, 1, 2


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("lda", C.c_longlong), ("a_rows", C.c_int),
        ("w", C.c_void_p), ("w_rows", C.c_int),
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("conv", C.c_int), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("ksize", C.c_int), ("pad", C.c_int),
        ("bias", C.c_void_p), ("bias_group_rows", C.c_int), ("scale", C.c_void_p), ("act", C.c_int),
        ("res_f32", C.c_void_p), ("res2_f32", C.c_void_p), ("res_f16", C.c_void_p),
        ("out_f32", C.c_void_p), ("out_f16", C.c_void_p), ("out_f16_relu", C.c_void_p),
        ("ldc", C.c_longlong), ("store", C.c_int),
        ("d2s_s", C.c_int), ("d2s_cout", C.c_int), ("d2s_h", C.c_int), ("d2s_w", C.c_int),
        ("nchw_p", C.c_int), ("nchw_k", C.c_int), ("nchw_group", C.c_int),
        ("row_sumsq", C.c_void_p), ("row_sumsq_parts", C.c_int), ("row_scale", C.c_float),
        ("out_row_sumsq", C.c_void_p), ("relu_after_res", C.c_int),
    ]


class LinearW(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("out", C.c_int), ("in_", C.c_int), ("rows", C.c_int)]


class VitBlockW(C.Structure):
    _fields_ = [("ln1_g", C.c_void_p), ("ln1_b", C.c_void_p), ("ln2_g", C.c_void_p), ("ln2_b", C.c_void_p),
                ("qkv", LinearW), ("proj", LinearW), ("fc1", LinearW), ("fc2", LinearW)]


class RcuW(C.Structure):
    _fields_ = [("conv1", LinearW), ("conv2", LinearW),
                ("bn1_scale", C.c_void_p), ("bn1_shift", C.c_void_p),
                ("bn2_scale", C.c_void_p), ("bn2_shift", C.c_void_p)]


class TextBlockW(C.Structure):
    _fields_ = [("ln1_g", C.c_void_p), ("ln1_b", C.c_void_p), ("ln2_g", C.c_void_p), ("ln2_b", C.c_void_p),
                ("in_proj", LinearW), ("out_proj", LinearW), ("c_fc", LinearW), ("c_proj", LinearW)]


class BottleneckW(C.Structure):
    _fields_ = [("conv1", LinearW), ("conv2", LinearW), ("conv3", LinearW), ("down", LinearW),
                ("bn1_scale", C.c_void_p), ("bn1_shift", C.c_void_p), ("bn2_scale", C.c_void_p), ("bn2_shift", C.c_void_p),
                ("bn3_scale", C.c_void_p), ("bn3_shift", C.c_void_p), ("bnd_scale", C.c_void_p), ("bnd_shift", C.c_void_p),
                ("stride", C.c_int)]


RESNET_BLOCKS = 33


class Weights(C.Structure):
    _fields_ = [
        ("vit_dim", C.c_int), ("vit_depth", C.c_int), ("vit_heads", C.c_int), ("patch_size", C.c_int),
        ("patch", LinearW), ("cls_token", C.c_void_p), ("pos_embed", C.c_void_p), ("pos_grid", C.c_int),
        ("blocks", VitBlockW * VIT_DEPTH), ("hooks", C.c_int * 4),
        ("readout_tok", LinearW * 4), ("readout_cls", LinearW * 4), ("post_conv1x1", LinearW * 4),
        ("post_channels", C.c_int * 4), ("post_resample", C.c_int * 4), ("post_resample_w", LinearW * 4),
        ("layer_rn", LinearW * 4), ("rcu1", RcuW * 4), ("rcu2", RcuW * 4), ("out_conv", LinearW * 4),
        ("head1", LinearW), ("logit_scale", C.c_float),
        ("text_width", C.c_int), ("text_heads", C.c_int), ("out_c", C.c_int),
        ("tok_emb", C.c_void_p), ("text_pos", C.c_void_p), ("text_blocks", TextBlockW * TEXT_DEPTH),
        ("lnf_g", C.c_void_p), ("lnf_b", C.c_void_p), ("text_proj", LinearW),
        ("arch_option", C.c_int), ("block_depth", C.c_int), ("head_act", C.c_int),
        ("head_block_w", C.c_float * 9), ("head_block_b", C.c_float),
        ("trunk", C.c_int), ("rn_stem", LinearW), ("rn_stem_scale", C.c_void_p), ("rn_stem_shift", C.c_void_p),
        ("rn_layers", C.c_int * 4), ("rn_blocks", BottleneckW * RESNET_BLOCKS),
    ]


# every symbol include/lseg_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "lseg_last_error", "lseg_abi_version", "lseg_read_watchdog",
    "lseg_gemm", "lseg_debug_gemm_plan", "lseg_debug_gemm_cluster", "lseg_debug_set_gemm_cluster", "lseg_debug_set_trace_block", "lseg_mhsa", "lseg_mhsa_variant", "lseg_text_attn", "lseg_mhsa_trace", "lseg_debug_gemm_trace", "lseg_set_deterministic", "lseg_layernorm", "lseg_patchify", "lseg_pos_resize", "lseg_assemble_tokens",
    "lseg_readout_split", "lseg_im2col_3x3_s2", "lseg_stem_im2col", "lseg_maxpool3x3s2_nhwc", "lseg_subsample2_nhwc", "lseg_upsample2x_nhwc", "lseg_upsample2x_nhwc256", "lseg_l2norm_scale", "lseg_l2norm_f16",
    "lseg_upsample2x_nchw", "lseg_debug_upsample_layout", "lseg_upsample2x_nchw_bg", "lseg_upsample2x_nchw_f32", "lseg_head_block", "lseg_upsample2x_argmax", "lseg_forward_argmax", "lseg_text_embed", "lseg_text_eot_gather",
    "lseg_create", "lseg_destroy", "lseg_encode_text", "lseg_forward", "lseg_forward_lowres", "lseg_debug_buffer",
    "lseg_last_launch_count", "lseg_forward_profiled",
    "lseg_p2p_alloc", "lseg_p2p_open", "lseg_p2p_close", "lseg_p2p_free", "lseg_p2p_copy", "lseg_p2p_signal",
    "lseg_p2p_wait",
    "lseg_eval_make_crops", "lseg_eval_canvas", "lseg_eval_resize_add", "lseg_preprocess",
    "lseg_seg_stats_scores", "lseg_seg_stats_mask", "lseg_forward_segstats",
    "lseg_encode_image", "lseg_query", "lseg_embedding_features",
    "lseg_forward_ragged", "lseg_query_ragged", "lseg_gemm_ragged",
    "lseg_attn_probs", "lseg_encode_image_attention",
    "lseg_xent_scores", "lseg_forward_xent", "lseg_query_xent",
]

_lib = None


def load(build_if_missing=True):
    """dlopen the in-tree library, building it first if needed. Raises on failure (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _build
        stale = _build.needs_build()
        try:
            _build.build()
        except Exception as e:
            # a stale library may have another lseg_weights / lseg_gemm_args layout: never load it silently
            if stale and os.path.exists(LIB_PATH) and not os.environ.get("LSEG_ALLOW_STALE_LIB"):
                raise ImportError(f"liblseg_b200.so is older than its sources and rebuilding failed ({e}); refusing to "
                                  f"load a possibly ABI-incompatible library (LSEG_ALLOW_STALE_LIB=1 overrides)") from e
            if not os.path.exists(LIB_PATH):
                raise
    if not os.path.exists(LIB_PATH):
        raise ImportError("liblseg_b200.so is missing and could not be built; lseg_b200 has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    if lib.lseg_abi_version() != ABI_VERSION:
        raise ImportError(f"liblseg_b200.so has ABI version {lib.lseg_abi_version()}, this binding expects {ABI_VERSION}: "
                          f"rebuild with `python -m lang-seg_b200.build --force`")
    lib.lseg_last_error.restype = C.c_char_p
    lib.lseg_debug_buffer.restype = C.c_void_p
    lib.lseg_debug_buffer.argtypes = [C.c_void_p, C.c_char_p]
    lib.lseg_gemm.argtypes = [C.POINTER(GemmArgs), C.c_void_p]
    lib.lseg_debug_gemm_plan.argtypes = [C.POINTER(GemmArgs), C.POINTER(C.c_int * 5)]
    lib.lseg_debug_gemm_cluster.argtypes = [C.POINTER(GemmArgs), C.POINTER(C.c_int * 2)]
    lib.lseg_debug_set_gemm_cluster.argtypes = [C.c_int]
    lib.lseg_debug_set_trace_block.argtypes = [C.c_int]
    lib.lseg_mhsa.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_mhsa_variant.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_attn_probs.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_text_attn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_debug_gemm_trace.argtypes = [C.c_void_p]
    lib.lseg_set_deterministic.argtypes = [C.c_int]
    lib.lseg_mhsa_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.lseg_layernorm.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int,
                                   C.c_float, C.c_void_p]
    lib.lseg_patchify.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_pos_resize.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_assemble_tokens.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]
    lib.lseg_readout_split.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_im2col_3x3_s2.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_stem_im2col.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_maxpool3x3s2_nhwc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_subsample2_nhwc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_upsample2x_nhwc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_upsample2x_nhwc256.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p]
    lib.lseg_l2norm_scale.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_float, C.c_void_p]
    lib.lseg_l2norm_f16.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_upsample2x_nchw.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_debug_upsample_layout.argtypes = [C.c_int]
    lib.lseg_upsample2x_nchw_bg.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_upsample2x_nchw_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_head_block.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.POINTER(C.c_float), C.c_float, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_text_embed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                    C.c_void_p]
    lib.lseg_text_eot_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_read_watchdog.argtypes = [C.POINTER(C.c_int * 4), C.c_void_p]
    lib.lseg_create.argtypes = [C.POINTER(Weights), C.c_int, C.POINTER(C.c_void_p)]
    lib.lseg_destroy.argtypes = [C.c_void_p]
    lib.lseg_destroy.restype = None
    lib.lseg_encode_text.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.lseg_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                 C.c_longlong, C.c_void_p, C.c_void_p]
    lib.lseg_forward_lowres.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                        C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lseg_forward_argmax.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                        C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lseg_upsample2x_argmax.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_p2p_alloc.argtypes = [C.c_ulonglong, C.POINTER(C.c_void_p), C.c_char_p]
    lib.lseg_p2p_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
    lib.lseg_p2p_close.argtypes = [C.c_void_p]
    lib.lseg_p2p_free.argtypes = [C.c_void_p]
    lib.lseg_p2p_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p]
    lib.lseg_p2p_signal.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p]
    lib.lseg_p2p_wait.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_ulonglong, C.c_uint, C.c_void_p]
    lib.lseg_eval_make_crops.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.POINTER(C.c_float), C.c_void_p]
    lib.lseg_eval_canvas.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p]
    lib.lseg_eval_resize_add.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.lseg_preprocess.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]
    lib.lseg_seg_stats_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_void_p, C.c_void_p]
    lib.lseg_seg_stats_mask.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]
    lib.lseg_forward_segstats.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                          C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]
    _xent = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong]  # loss_target .. partials_len
    lib.lseg_xent_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]
    lib.lseg_forward_xent.argtypes = ([C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                       C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p] + _xent +
                                      [C.c_void_p, C.c_void_p, C.c_void_p])
    lib.lseg_query_xent.argtypes = ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                     C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                     C.c_void_p] + _xent + [C.c_void_p])
    lib.lseg_encode_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    lib.lseg_encode_image_attention.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]
    lib.lseg_query.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                               C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                               C.c_void_p, C.c_void_p]
    lib.lseg_embedding_features.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p]
    _ragged = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lseg_forward_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int] + _ragged
    lib.lseg_query_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int] + _ragged
    lib.lseg_gemm_ragged.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
    lib.lseg_last_launch_count.argtypes = [C.c_void_p]
    lib.lseg_forward_profiled.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                          C.c_longlong, C.c_void_p, C.c_void_p, C.POINTER(C.c_float),
                                          C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)]
    _lib = lib
    return lib


class LsegError(RuntimeError):
    pass


def check(status):
    if status != 0:
        raise LsegError(load().lseg_last_error().decode("utf-8", "replace"))
