"""ctypes binding of the C-ABI library (include/otter_b200.h).

The shared library is built in-tree by `__graft_entry__.build()` into otter_b200/lib/.  There is no
CPU / PyTorch fallback: if the library is missing the import of any op fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libotter_b200.so")


class OtbError(RuntimeError):
    pass


class GemmEpilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p), ("aux_in", C.c_void_p), ("aux_out", C.c_void_p), ("scale_ptr", C.c_void_p),
        ("residual", C.c_void_p), ("out", C.c_void_p),
        ("ld_out", C.c_int64), ("ld_aux_in", C.c_int64), ("ld_aux_out", C.c_int64), ("ld_res", C.c_int64),
        ("act", C.c_int32), ("scale_tanh", C.c_int32), ("out_fp32", C.c_int32), ("accumulate", C.c_int32),
        ("alpha", C.c_float), ("res_fp32", C.c_int32),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("kv1", C.c_void_p), ("kv2", C.c_void_p), ("out", C.c_void_p), ("lse", C.c_void_p),
        ("text_time", C.c_void_p),
        ("ldq", C.c_int64), ("ldkv1", C.c_int64), ("ldkv2", C.c_int64), ("ld_out", C.c_int64),
        ("q_cols", C.c_int32), ("kv1_cols", C.c_int32), ("kv2_cols", C.c_int32),
        ("q_col0", C.c_int32), ("k1_col0", C.c_int32), ("v1_col0", C.c_int32), ("k2_col0", C.c_int32),
        ("v2_col0", C.c_int32), ("out_col0", C.c_int32),
        ("n_per_media", C.c_int32), ("T_img", C.c_int32),
        ("P", C.c_int32), ("H", C.c_int32), ("Sq", C.c_int32), ("Sk1", C.c_int32), ("Sk2", C.c_int32),
        ("head_dim", C.c_int32),
        ("scale", C.c_float), ("mask_ge", C.c_int32), ("causal", C.c_int32),
    ]


class AttnGrads(C.Structure):
    _fields_ = [
        ("dout", C.c_void_p), ("dq", C.c_void_p), ("dkv1", C.c_void_p), ("dkv2", C.c_void_p), ("dq_ws", C.c_void_p),
        ("ld_dout", C.c_int64), ("ld_dq", C.c_int64), ("ld_dkv1", C.c_int64), ("ld_dkv2", C.c_int64),
        ("dout_cols", C.c_int32), ("dout_col0", C.c_int32), ("dq_col0", C.c_int32), ("dk1_col0", C.c_int32),
        ("dv1_col0", C.c_int32), ("dk2_col0", C.c_int32), ("dv2_col0", C.c_int32), ("_pad", C.c_int32),
    ]


class LmAttnDesc(C.Structure):
    _fields_ = [
        ("qkv", C.c_void_p), ("out", C.c_void_p), ("lse", C.c_void_p), ("alibi_slopes", C.c_void_p),
        ("ld_qkv", C.c_int64), ("ld_out", C.c_int64),
        ("qkv_cols", C.c_int32), ("q_col0", C.c_int32), ("k_col0", C.c_int32), ("v_col0", C.c_int32),
        ("out_col0", C.c_int32),
        ("B", C.c_int32), ("H", C.c_int32), ("S", C.c_int32), ("head_dim", C.c_int32), ("causal", C.c_int32),
        ("scale", C.c_float), ("kv_heads", C.c_int32),
    ]


class LmAttnGrads(C.Structure):
    _fields_ = [
        ("dout", C.c_void_p), ("dqkv", C.c_void_p), ("dq_ws", C.c_void_p),
        ("ld_dout", C.c_int64), ("ld_dqkv", C.c_int64),
        ("dout_cols", C.c_int32), ("dout_col0", C.c_int32), ("dq_col0", C.c_int32), ("dk_col0", C.c_int32),
        ("dv_col0", C.c_int32), ("_pad", C.c_int32),
    ]


class LmAttnDecodeDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p), ("ws", C.c_void_p),
        ("alibi_slopes", C.c_void_p),
        ("ld_q", C.c_int64), ("ld_out", C.c_int64), ("kv_batch_stride", C.c_int64), ("ld_kv", C.c_int64),
        ("B", C.c_int32), ("H", C.c_int32), ("T", C.c_int32), ("head_dim", C.c_int32),
        ("scale", C.c_float), ("_pad", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/otter_b200.h declares
_VP, _I, _I64, _F = C.c_void_p, C.c_int, C.c_int64, C.c_float
SIGNATURES = {
    "otb_last_error": (C.c_char_p, []),
    "otb_version": (_I, []),
    "otb_compiled_arch": (_I, []),
    "otb_launch_count": (C.c_longlong, []),
    "otb_tmap_cache_stat": (C.c_longlong, [_I]),
    "otb_abi_sizeof": (_I, [_I]),
    "otb_gemm_bf16": (_I, [_VP, _I, _I64, _VP, _I, _I64, _I, _I, _I, C.POINTER(GemmEpilogue), _VP]),
    "otb_attn_fwd": (_I, [C.POINTER(AttnDesc), _VP]),
    "otb_attn_bwd": (_I, [C.POINTER(AttnDesc), C.POINTER(AttnGrads), _VP]),
    "otb_xattn_out_fused": (_I, [C.POINTER(AttnDesc), _VP, _I64, _VP, _VP, _I64, _VP, _I64, _VP, _I64, _I, _VP]),
    "otb_lm_attn_fwd": (_I, [C.POINTER(LmAttnDesc), _VP]),
    "otb_lm_attn_bwd": (_I, [C.POINTER(LmAttnDesc), C.POINTER(LmAttnGrads), _VP]),
    "otb_lm_attn_decode_ws_floats": (C.c_longlong, [_I, _I, _I]),
    "otb_lm_attn_decode": (_I, [C.POINTER(LmAttnDecodeDesc), _VP]),
    "otb_linear_small_m": (_I, [_VP, _I64, _VP, _I64, _I, _I, _I, _F, _VP, _I, _VP, _I64, _VP, _I64, _VP]),
    "otb_text_time": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "otb_layernorm_fwd": (_I, [_VP, _I64, _VP, _VP, _VP, _I64, _VP, _VP, _I, _I, _F, _VP]),
    "otb_ln_chunks": (_I, [_I, _I]),
    "otb_layernorm_bwd": (_I, [_VP, _I64, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP, _I, _VP, _I, _I,
                               _VP]),
    "otb_cast_f32_bf16": (_I, [_VP, _VP, _I64, _VP]),
    "otb_cast_f32_bf16_multi": (_I, [_VP, _I, _I64, _VP]),
    "otb_cast_bf16_f32": (_I, [_VP, _VP, _I64, _VP]),
    "otb_cast_bf16_f32_scale": (_I, [_VP, _VP, _I64, _F, _VP]),
    "otb_bcast_rows": (_I, [_VP, _I, _I, _VP, _I, _I, _VP]),
    "otb_add_rowbias": (_I, [_VP, _VP, _I, _I, _VP, _I, _I, _VP]),
    "otb_grouped_colsum": (_I, [_VP, _I64, _I, _I, _I, _I, _VP, _I, _VP]),
    "otb_dot_blocks": (_I, []),
    "otb_gate_grad": (_I, [_VP, _VP, _I64, _VP, _VP, _I, _VP, _VP]),
    "otb_sqmean_loss": (_I, [_VP, _I64, _VP, _VP, _VP, _VP]),
    "otb_split3_concat": (_I, [_VP, _I64, _I, _I, _I, _VP, _VP]),
    "otb_layernorm_fwd_f32": (_I, [_VP, _I64, _VP, _VP, _VP, _I64, _I, _I, _F, _VP]),
    "otb_add_rowbias_f32": (_I, [_VP, _VP, _I, _I, _VP, _I, _I, _VP]),
    "otb_attn_fwd_f32": (_I, [C.POINTER(AttnDesc), _VP]),
    "otb_epilogue_f32": (_I, [_VP, _VP, _I, _VP, _I, _VP, _VP, _I, _I, _VP]),
    "otb_layernorm_bwd_f32": (_I, [_VP, _I64, _VP, _I64, _VP, _VP, _I64, _VP, _VP, _VP, _I, _I, _F, _VP]),
    "otb_act_bwd_f32": (_I, [_VP, _VP, _I, _VP, _I64, _VP]),
    "otb_gate_grad_f32": (_I, [_VP, _VP, _I64, _VP, _VP, _VP]),
    "otb_rowbias_grad_f32": (_I, [_VP, _I, _I, _I, _I, _I, _VP, _VP]),
    "otb_attn_bwd_f32": (_I, [C.POINTER(AttnDesc), C.POINTER(AttnGrads), _VP]),
    "otb_label_mask": (_I, [_VP, _I, _I, _I64, _I64, _I64, _I64, _VP, _VP]),
    "otb_shifted_cross_entropy": (_I, [_VP, _I, _I64, _VP, _I, _I, _I, _VP, _VP, _I64, _VP, _VP]),
    "otb_scale_by_scalar": (_I, [_VP, _I, _I64, _VP, _VP]),
    "otb_im2col_patches": (_I, [_VP, _I, _I, _I, _I, _I, _VP, _I, _VP]),
    "otb_clip_assemble": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "otb_media_from_clip": (_I, [_VP, _VP, _I, _VP, _I, _I, _I, _VP]),
    "otb_rmsnorm_fwd": (_I, [_VP, _I64, _VP, _VP, _I64, _VP, _I, _I, _F, _VP]),
    "otb_rmsnorm_bwd": (_I, [_VP, _I64, _VP, _I64, _VP, _VP, _VP, _I64, _VP, _I64, _I, _I, _VP]),
    "otb_rmsnorm_bwd_chunks": (_I, [_I, _I]),
    "otb_rmsnorm_bwd_params": (_I, [_VP, _I64, _VP, _I64, _VP, _VP, _VP, _I64, _VP, _I64, _VP, _I, _VP, _I, _I, _VP]),
    "otb_rope128": (_I, [_VP, _I64, _I64, _I, _I, _I, _F, _I, _VP]),
    "otb_rope128_freqs": (_I, [_VP, _I64, _I64, _I, _I, _I, _VP, _F, _I, _VP]),
    "otb_swiglu_fwd": (_I, [_VP, _I64, _VP, _I64, _VP, _I64, _I64, _I, _VP]),
    "otb_swiglu_bwd": (_I, [_VP, _I64, _VP, _I64, _VP, _I64, _VP, _I64, _VP, _I64, _I64, _I, _VP]),
    "otb_lora_dropout_fwd": (_I, [_VP, _VP, _I64, _I, _I64, _F, C.c_uint64, C.c_uint32, _VP]),
    "otb_lora_dropout_bwd_add": (_I, [_VP, _VP, _I64, _I, _I64, _F, C.c_uint64, C.c_uint32, _VP]),
    "otb_qkln_rope_ws_floats": (_I, []),
    "otb_qkln_rope_fwd": (_I, [_VP, _I64, _VP, _VP, _VP, _VP, _VP, _I64, _VP, _I64, _I, _I, _I, _F, _F, _VP]),
    "otb_qkln_rope_bwd": (_I, [_VP, _I64, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _VP, _VP, _VP, _VP, _I, _VP, _I64, _I, _I,
                               _I, _F, _VP]),
    "otb_preprocess_images": (_I, [_VP, _VP, _I, _I, _I, _VP, _F, _F, _F, _F, _F, _F, _VP, _I, _VP]),
    "otb_fuyu_scatter": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
}

_lib = None


def load():
    """Load libotter_b200.so (once). Raises OtbError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise OtbError(f"{LIB_PATH} not found — run `python -c 'import __graft_entry__ as g; g.build()'` first; "
                       "otter_b200 has no CPU/PyTorch fallback")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    for i, st in enumerate((GemmEpilogue, AttnDesc, AttnGrads, LmAttnDesc, LmAttnGrads, LmAttnDecodeDesc)):
        if lib.otb_abi_sizeof(i) != C.sizeof(st):
            raise OtbError(f"ABI mismatch: {st.__name__} is {C.sizeof(st)} bytes in ctypes, "
                           f"{lib.otb_abi_sizeof(i)} in the library")
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().otb_last_error()
        raise OtbError(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")
