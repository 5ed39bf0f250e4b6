"""ctypes binding of libvitron_b200.so (the C ABI declared in include/vitron_b200.h).

There is no CPU fallback: if the library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvitron_b200.so")

ACT_NONE, ACT_GELU, ACT_QUICK_GELU, ACT_RELU, ACT_SILU = 0, 1, 2, 3, 4
GLU_NONE, GLU_SWIGLU, GLU_GEGLU = 0, 1, 2

_ERR = {-1: "VB_ERR_ARG", -2: "VB_ERR_CUDA", -3: "VB_ERR_WORKSPACE", -4: "VB_ERR_UNSUPPORTED",
        -5: "VB_ERR_DRIVER"}


class Epilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p), ("rowbias", C.c_void_p), ("rowbias_rows", C.c_int64),
        ("residual", C.c_void_p), ("ldr", C.c_int64), ("alpha", C.c_float),
        ("act", C.c_int32), ("glu", C.c_int32), ("out_fp32", C.c_int32),
        ("rowscale", C.c_void_p), ("rms_eps", C.c_float),
    ]


_p, _i64, _i32, _f, _sz = C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_size_t

# name -> (restype, argtypes); mirrors include/vitron_b200.h one to one
SIGNATURES = {
    "vb200_version": (C.c_char_p, []),
    "vb200_last_error": (C.c_char_p, []),
    "vb200_device_ok": (_i32, []),
    "vb200_set_pdl": (_i32, [_i32]),
    "vb200_set_attention_impl": (_i32, [_i32]),
    "vb200_attention_watchdog": (_i32, [_p]),
    "vb200_attention_tc_occupancy": (_i32, [_i32]),
    "vb200_gemm_bf16_workspace_size": (_sz, [_i64, _i64, _i64]),
    "vb200_gemm_bf16": (_i32, [_p, _i64, _p, _i64, _p, _i64, _i64, _i64, _i64, C.POINTER(Epilogue), _p, _sz, _p]),
    "vb200_gemm_nf4": (_i32, [_p, _i64, _p, _p, _p, _p, _i64, _i64, _i64, _i64, C.POINTER(Epilogue), _p]),
    "vb200_nf4_dequant": (_i32, [_p, _p, _p, _p, _i64, _i64, _p]),
    "vb200_conv_nhwc_workspace_size": (_sz, [_i64, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32]),
    "vb200_conv_nhwc_bf16": (_i32, [_p, _p, _p, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32,
                                    C.POINTER(Epilogue), _p, _sz, _p]),
    "vb200_set_gemm_impl": (_i32, [_i32]),
    "vb200_set_gemm_debug": (_i32, [_i32, _i32]),
    "vb200_conv_nhwc_direct": (_i32, [_p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _p]),
    "vb200_rmsnorm": (_i32, [_p, _i64, _p, _p, _i64, _i64, _i64, _f, _p]),
    "vb200_row_rstd": (_i32, [_p, _i64, _p, _i64, _i64, _f, _p]),
    "vb200_layernorm": (_i32, [_p, _i64, _p, _p, _p, _i64, _i64, _i64, _f, _p]),
    "vb200_groupnorm_workspace_size": (_sz, [_i64, _i64, _i64]),
    "vb200_groupnorm_nhwc": (_i32, [_p, _p, _p, _p, _i64, _i64, _i64, _i64, _f, _i32, _p, _sz, _p]),
    "vb200_attention": (_i32, [_p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64] + [_i64] * 12 +
                        [_f, _i32, _p, _p, _i64, _i64, _i64, _p]),
    "vb200_attention_workspace_size": (_sz, [_i64, _i64, _i64, _i64, _i64, _i32]),
    "vb200_attention_ws": (_i32, [_p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64] + [_i64] * 12 +
                           [_f, _i32, _p, _p, _i64, _i64, _i64, _p, _sz, _p]),
    "vb200_attention_paged_workspace_size": (_sz, [_i64, _i64, _i64, _i64, _i64]),
    "vb200_attention_paged": (_i32, [_p, _i64, _i64, _i64, _p, _p, _i64, _p, _i64, _p, _p, _p, _i64, _i64, _i64,
                                     _i64, _i64, _i64, _i64, _i64, _i64, _f, _p, _sz, _p]),
    "vb200_attention_short": (_i32, [_p, _p, _p, _p, _i64, _i64, _i64, _i64] + [_i64] * 17 + [_f, _p]),
    "vb200_add_rowgroup": (_i32, [_p, _p, _p, _i64, _i64, _i64, _i64, _p]),
    "vb200_rope_kv_append": (_i32, [_p, _i64, _p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _i64, _i64, _f, _p]),
    "vb200_attn_decode_workspace_size": (_sz, [_i64, _i64, _i64, _i64]),
    "vb200_attn_decode_paged": (_i32, [_p, _i64, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, _i64, _i64,
                                       _f, _p, _sz, _p]),
    "vb200_rope_table": (_i32, [_p, _p, _i64, _i64, _f, _p]),
    "vb200_attn_decode_rope": (_i32, [_p, _i64, _p, _p, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64, _i64, _i64,
                                      _f, _p, _sz, _p]),
    "vb200_attn_decode_rope_beam": (_i32, [_p, _i64, _p, _p, _p, _p, _i64, _p, _p, _i64, _p, _p, _i64, _i64, _i64, _i64,
                                           _i64, _i64, _f, _p, _sz, _p]),
    "vb200_splice_multimodal": (_i32, [_p, _i64, _p, _i64, _p, _p, _i64, _i64, _p]),
    "vb200_argmax_rows": (_i32, [_p, _i32, _i64, _i64, _i64, _p, _p]),
    "vb200_argmax_advance": (_i32, [_p, _i64, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p]),
    "vb200_sample_advance": (_i32, [_p, _i64, _i64, _i64, _p, _p, _p, _p, _p, _p, _i64, _p, _p]),
    "vb200_beam_workspace_size": (_sz, [_i64]),
    "vb200_beam_advance": (_i32, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64, _p, _p,
                                  _p, _p, _i64, _p, _p, _sz, _p]),
    "vb200_beam_sample_advance": (_i32, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64,
                                         _p, _p, _p, _p, _i64, _p, _p, _sz, _p, _p]),
    "vb200_beam_advance_logprobs": (_i32, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _i64,
                                           _p, _p, _p, _p, _i64, _p, _p, _sz, _p]),
    "vb200_beam_sample_advance_logprobs": (_i32, [_p, _i64, _i64, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p,
                                                  _i64, _p, _p, _p, _p, _i64, _p, _p, _sz, _p, _p]),
    "vb200_logits_process": (_i32, [_p, _i64, _i64, _i64, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _i32, _p]),
    "vb200_patchify": (_i32, [_p, _i32, _p, _i64, _i64, _i64, _i64, _i64, _i64, _p]),
    "vb200_vit_embed_ln": (_i32, [_p, _p, _p, _p, _p, _p, _i64, _i64, _i64, _f, _p]),
    "vb200_upsample2x_nhwc": (_i32, [_p, _p, _i64, _i64, _i64, _i64, _p]),
    "vb200_add_bf16": (_i32, [_p, _p, _p, _i64, _i64, _p]),
    "vb200_cfg_combine": (_i32, [_p, _p, _p, _f, _i64, _p]),
    "vb200_region_mask_pool": (_i32, [_p, _p, _p, _i64, _i64, _i64, _i64, _p]),
    "vb200_seem_attn_mask": (_i32, [_p, _p, _i64, _i64, _i64, _i64, _i64, _p]),
    "vb200_resize_bilinear_nhwc": (_i32, [_p, _p, _i64, _i64, _i64, _i64, _i64, _i64, _p]),
    "vb200_softmax_rows": (_i32, [_p, _i64, _p, _i64, _i64, _i64, _p]),
    "vb200_preprocess_frames": (_i32, [_p, _p] + [_i64] * 11 + [_p, _p, _i32, _i32, _i32, _p]),
    "vb200_im2col_nchw": (_i32, [_p, _i32, _p] + [_i64] * 10 + [_p]),
    "vb200_set_dwconv_impl": (_i32, [_i32]),
    "vb200_dwconv_nhwc": (_i32, [_p, _i64, _p, _p, _i64, _i64, _i64, _i64, _i64, _i32, _p]),
    "vb200_colmean_workspace_size": (_sz, [_i64, _i64, _i64]),
    "vb200_colmean": (_i32, [_p, _p, _i64, _i64, _i64, _i32, _p, _sz, _p]),
    "vb200_focal_modulate": (_i32, [_p, _i64, _p, _i64, _p, _p, _i64, _i64, _i64, _f, _p]),
    "vb200_mul_rows": (_i32, [_p, _i64, _p, _i64, _p, _i64, _i64, _p]),
    "vb200_layernorm_add": (_i32, [_p, _i64, _p, _p, _p, _i64, _p, _i64, _i64, _i64, _f, _p]),
}

_lib = None


def load():
    """Load the shared library (once). Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m vitron_b200.build` "
            "(nvcc, sm_90a). vitron_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    mode = os.environ.get("VB200_GEMM_MODE")   # measurement aid: the `mode` argument of vb200_set_gemm_debug (A/B runs of bench.py)
    if mode:
        lib.vb200_set_gemm_debug(int(mode), -1)
    return lib


class VitronB200Error(RuntimeError):
    pass


def check(code, what):
    if code != 0:
        detail = load().vb200_last_error().decode() if code == -2 else ""
        raise VitronB200Error(f"{what} failed: {_ERR.get(code, code)} {detail}")
