"""ctypes binding of libcambrian_b200.so (the C ABI declared in include/cambrian_b200.h).

There is NO fallback: if the shared library is missing or an entry point fails, the caller gets an
exception.  PyTorch is used only for device memory and streams (tensor.data_ptr(), current stream).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import torch

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libcambrian_b200.so"

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float
_vpp = C.POINTER(C.c_void_p)
_ip = C.POINTER(C.c_int)

# name -> (restype, argtypes); must list every symbol include/cambrian_b200.h declares
SIGNATURES = {
    "cb_version": (_i, []),
    "cb_last_error": (C.c_char_p, []),
    "cb_sm_count": (_i, []),
    "cb_launch_count": (_i64, []),
    "cb_gemm_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i64, _i64, _i64, _i64, _i64, _i64, _i, _i,
                          _vp, _vp, _vp, _i64, _i64, _f, _i, _i, _i, _i, _vp]),
    "cb_sva_window_attn_fwd": (_i, [_vp, _vp, _vp, _i, _vpp, _vpp, _vpp, _ip, _i, _i, _i, _i, _vp]),
    "cb_sva_window_attn_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vpp, _vpp, _vpp, _vpp, _vpp, _ip,
                                    _i, _i, _i, _i, _vp]),
    "cb_layernorm_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _vp, _i, _i, _vp]),
    "cb_layernorm_bwd": (_i, [_vp] * 10 + [_i64, _i64, _i, _vp, _i, _i, _vp]),
    "cb_rmsnorm_fwd": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _f, _i, _vp]),
    "cb_rmsnorm_bwd": (_i, [_vp] * 8 + [_i64, _i64, _i, _vp]),
    "cb_norm_bwd_workspace_floats": (_i64, [_i64, _i]),
    "cb_attn_fwd": (_i, [_vp] * 6 + [_i] * 6 + [_i64] * 8 + [_f, _i, _vp]),
    "cb_attn_fwd_window": (_i, [_vp] * 6 + [_i] * 6 + [_i64] * 8 + [_f, _i, _i, _vp]),
    "cb_attn_bwd": (_i, [_vp] * 11 + [_i] * 6 + [_i64] * 16 + [_f, _i, _vp]),
    "cb_attn_bwd_window": (_i, [_vp] * 11 + [_i] * 6 + [_i64] * 16 + [_f, _i, _i, _vp]),
    "cb_act_fwd": (_i, [_vp, _vp, _i64, _i, _vp]),
    "cb_act_bwd": (_i, [_vp, _vp, _vp, _i64, _i, _vp]),
    "cb_swiglu_fwd": (_i, [_vp, _vp, _vp, _i64, _i, _i64, _i64, _vp]),
    "cb_swiglu_bwd": (_i, [_vp] * 5 + [_i64, _i, _i64, _i64, _i64, _vp]),
    "cb_rope": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _i64, _i, _i, _vp]),
    "cb_embed_splice": (_i, [_vp] * 6 + [_i, _i, _i, _i, _i64, _vp]),
    "cb_embed_splice_bwd": (_i, [_vp] * 6 + [_i, _i, _i, _i, _i64, _vp]),
    "cb_add_pos_tokens": (_i, [_vp] * 4 + [_i, _i, _i, _vp]),
    "cb_bilinear": (_i, [_vp, _vp] + [_i] * 6 + [_i64, _i64, _i, _i, _vp]),
    "cb_patchify_nchw": (_i, [_vp, _vp] + [_i] * 5 + [_vp]),
    "cb_patchify_nhwc": (_i, [_vp, _vp] + [_i] * 5 + [_vp]),
    "cb_dwconv7": (_i, [_vp] * 4 + [_i] * 4 + [_vp]),
    "cb_add_inplace": (_i, [_vp, _vp, _i64, _vp]),
    "cb_group_colsum": (_i, [_vp, _vp, _vp, _i, _i64, _i, _f, _i, _vp]),
    "cb_group_broadcast": (_i, [_vp, _vp, _i, _i64, _i, _f, _i, _vp]),
    "cb_pos_grad": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "cb_f32_to_bf16": (_i, [_vp, _vp, _i64, _i, _i64, _f, _vp]),
    "cb_cross_entropy": (_i, [_vp] * 4 + [_i64, _i64, _i64, _f, _i, _i64, _vp]),
    "cb_cross_entropy_ex": (_i, [_vp] * 4 + [_i64, _i64, _i64, _f, _vp, _i, _i64, _vp]),
    "cb_adamw": (_i, [_vp] * 5 + [_i64] + [_f] * 5 + [_i, _f, _vp]),
    "cb_adamw_ex": (_i, [_vp] * 5 + [_i64] + [_f] * 5 + [_i, _f, _vp, _i, _vp]),
    "cb_adamw_host": (_i, [_vp] * 5 + [_i64] + [_f] * 5 + [_i, _f, _vp, _i, _vp]),
    "cb_adamw8": (_i, [_vp] * 7 + [_i64] + [_f] * 5 + [_i, _f, _vp, _i, _vp]),
    "cb_adamw8_host": (_i, [_vp] * 7 + [_i64] + [_f] * 5 + [_i, _f, _vp, _i, _vp]),
    "cb_gemv_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _i64, _i64, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_allreduce_symm_bf16": (_i, [C.c_uint64, _vp, _vp, _i64, _i64, _i, _i, C.c_uint32, _i, _vp]),
    "cb_embed_grad_sorted": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i64, _vp]),
    "cb_sumsq_bf16": (_i, [_vp, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_clip_coef": (_i, [_vp, _f, _f, _vp, _vp]),
    "cb_span_gather": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "cb_span_scatter": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "cb_span_gather_hw": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "cb_span_scatter_hw": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "cb_window_gather": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "cb_gemm_swiglu_bf16": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i64, _i64, _i64, _i64, _vp]),
    "cb_resample_ksize": (_i, [_i, _i]),
    "cb_resample_coeffs": (_i, [_i, _i, _vp, _vp]),
    "cb_preprocess_workspace_bytes": (_i64, [_i, _i, _i]),
    "cb_preprocess_image": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "cb_embed_splice_ragged": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i, _vp]),
    "cb_tower_combine_fwd": (_i, [_vp, _i, _vpp, _vp, _vp, _i64, _i, _i, _vp]),
    "cb_tower_combine_bwd": (_i, [_vp, _i, _vpp, _vp, _vpp, _vp, _i64, _i, _i, _vp]),
    "cb_bilinear_bwd": (_i, [_vp, _vp] + [_i] * 6 + [_vp]),
    "cb_nf4_quantize": (_i, [_vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "cb_gemv_nf4": (_i, [_vp, _vp, _i, _i, _i, _i64, _i64, _i, _ip, _vpp, _vpp, _vpp, _vpp, _vp, _vp, _i64, _i, _vp]),
    "cb_nf4_dequant": (_i, [_vp, _i, _i, _i, _ip, _vpp, _vpp, _vpp, _vpp, _vp]),
    "cb_int8_quantize_weight": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp]),
    "cb_int8_quantize_act": (_i, [_vp, _i, _i, _i64, _f, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cb_gemv_int8": (_i, [_vp] * 5 + [_i64, _vp, _vp, _vp, _i, _i, _i, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_gemm_int8": (_i, [_vp] * 5 + [_i64, _vp, _vp, _vp, _i, _i, _i, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_fp8_quantize_weight": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp]),
    "cb_fp8_quantize_act": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp]),
    "cb_gemv_fp8": (_i, [_vp] * 5 + [_i, _i, _i, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_gemm_fp8": (_i, [_vp] * 5 + [_i, _i, _i, _i64, _vp, _vp, _i64, _i, _vp]),
    "cb_kv_fp8_append": (_i, [_vp, _vp, _i64] + [_vp] * 4 + [_i] * 5 + [_i64, _vp, _vp]),
    "cb_attn_decode_fp8_workspace_floats": (_i64, [_i] * 5),
    "cb_attn_decode_fp8": (_i, [_vp, _i64] + [_vp] * 5 + [_i64, _vp, _vp, _i64] + [_i] * 6 + [_i64, _vp, _f, _vp]),
    "cb_fp8_quantize_weight_t_workspace_floats": (_i64, [_i, _i]),
    "cb_fp8_quantize_weight_t": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _i64, _vp]),
    "cb_rmsnorm_fwd_fp8": (_i, [_vp] * 5 + [_i64, _i, _f, _i, _vp]),
    "cb_swiglu_bwd_fp8": (_i, [_vp] * 7 + [_i64, _i, _i64, _i64, _i64, _vp]),
    "cb_paged_kv_append": (_i, [_vp, _vp, _i64] + [_vp] * 4 + [_i, _vp, _i64, _vp] + [_i] * 7 + [_i64, _i, _vp]),
    "cb_attn_decode_paged_workspace_floats": (_i64, [_i] * 5),
    "cb_attn_decode_paged": (_i, [_vp, _i64] + [_vp] * 4 + [_i, _vp, _i64, _vp, _i, _vp, _vp, _i64] + [_i] * 7 + [_f, _vp]),
    "cb_paged_kv_gather": (_i, [_vp] * 4 + [_i, _vp] + [_i] * 5 + [_i64, _vp, _vp, _i64, _vp]),
}

_lib = None


class CambrianB200Error(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the shared library (once).  Fails loudly: the product has no CPU / eager fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise CambrianB200Error(
            f"{LIB_PATH} not found — build it with `python -m cambrian_b200.build` "
            "(there is no PyTorch/CPU fallback for the hot path)")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    msg = load().cb_last_error().decode(errors="replace")
    if rc == 1:
        raise ValueError(f"{what}: {msg}")
    raise CambrianB200Error(f"{what} failed (code {rc}): {msg}")


def ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return arr


def int_array(vals):
    return (C.c_int * len(vals))(*vals)
