"""ctypes binding of the C ABI declared in include/lvb200.h.

Loading is lazy and loud: `lib()` raises RuntimeError if liblvb200.so is missing (run
`python -c "import __graft_entry__ as g; g.build()"` or `python long-vita_b200/build.py`).
There is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liblvb200.so")

_lock = threading.Lock()
_lib = None

c_i64 = C.c_int64
c_i32 = C.c_int32
c_f32 = C.c_float
c_ptr = C.c_void_p


class AttnParams(C.Structure):
    """Mirror of `lv_attn_params` (include/lvb200.h)."""

    _fields_ = [
        ("q", c_ptr), ("k", c_ptr), ("v", c_ptr), ("out", c_ptr), ("lse", c_ptr),
        ("batch", c_i64), ("sq", c_i64), ("sk", c_i64), ("hq", c_i64), ("hkv", c_i64), ("d", c_i64),
        ("q_strides", c_i64 * 3), ("k_strides", c_i64 * 3), ("v_strides", c_i64 * 3), ("o_strides", c_i64 * 3),
        ("scale", c_f32), ("causal", c_i32),
        ("q_seg_len", c_i64), ("q_seg_pos", c_i64 * 2), ("kv_pos0", c_i64),
    ]


class AttnBwdParams(C.Structure):
    """Mirror of `lv_attn_bwd_params` (include/lvb200.h)."""

    _fields_ = [
        ("fwd", AttnParams), ("d_out", c_ptr), ("dq", c_ptr), ("dk", c_ptr), ("dv", c_ptr),
        ("do_strides", c_i64 * 3), ("dq_strides", c_i64 * 3), ("dk_strides", c_i64 * 3), ("dv_strides", c_i64 * 3),
        ("delta_ws", c_ptr),
    ]


class AttnDocs(C.Structure):
    """Mirror of `lv_attn_docs` (include/lvb200.h)."""

    _fields_ = [("cu_seqlens", c_ptr), ("n_docs", c_i64)]


class AttnFp8Kv(C.Structure):
    """Mirror of `lv_attn_fp8_kv` (include/lvb200.h)."""

    _fields_ = [("k8", c_ptr), ("vt8", c_ptr), ("k_scale", c_ptr), ("v_scale", c_ptr)]


class CpParams(C.Structure):
    """Mirror of `lv_cp_params` (include/lvb200.h)."""

    _fields_ = [
        ("rank", c_i32), ("cp", c_i32), ("seq_total", c_i64), ("epoch", C.c_uint32), ("peer_tok_stride", c_i64),
        ("peer_kv", c_ptr * 8), ("peer_ready", c_ptr * 8), ("my_ready", c_ptr),
        ("k_full", c_ptr), ("v_full", c_ptr), ("blk_flags", c_ptr), ("fault", c_ptr),
    ]


# name -> (restype, argtypes); every symbol include/lvb200.h declares
SIGNATURES = {
    "lv_version": (c_i32, []),
    "lv_last_error": (C.c_char_p, []),
    "lv_launch_count": (c_i64, []),
    "lv_attn_fwd": (c_i32, [C.POINTER(AttnParams), c_ptr]),
    "lv_attn_bwd_ws_bytes": (c_i64, [c_i64, c_i64, c_i64]),
    "lv_attn_bwd": (c_i32, [C.POINTER(AttnBwdParams), c_ptr]),
    "lv_attn_docs_fwd": (c_i32, [C.POINTER(AttnParams), C.POINTER(AttnDocs), c_ptr]),
    "lv_attn_docs_bwd": (c_i32, [C.POINTER(AttnBwdParams), C.POINTER(AttnDocs), c_ptr]),
    "lv_attn_fp8_quant_kv": (c_i32, [C.POINTER(AttnParams), C.POINTER(AttnFp8Kv), c_ptr]),
    "lv_attn_fwd_fp8": (c_i32, [C.POINTER(AttnParams), C.POINTER(AttnFp8Kv), c_ptr]),
    "lv_attn_cp_fwd": (c_i32, [C.POINTER(AttnParams), C.POINTER(CpParams), c_ptr]),
    "lv_cp_check_fault": (c_i32, [c_ptr, c_ptr]),
    "lv_ipc_alloc": (c_i32, [c_i64, C.POINTER(c_ptr)]),
    "lv_ipc_free": (c_i32, [c_ptr]),
    "lv_ipc_get_handle": (c_i32, [c_ptr, c_ptr]),
    "lv_ipc_open_handle": (c_i32, [c_ptr, C.POINTER(c_ptr)]),
    "lv_ipc_close_handle": (c_i32, [c_ptr]),
    "lv_rmsnorm": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_f32, c_ptr]),
    "lv_layernorm": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_f32, c_ptr]),
    "lv_rope_table": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_rope": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_ptr]),
    "lv_swiglu": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_bias_gelu": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i32, c_ptr]),
    "lv_ls_residual": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_pixel_shuffle": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i32, c_ptr]),
    "lv_embed_scatter": (c_i32, [c_ptr, c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_i64, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_row_gather": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_row_scatter_zero": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_row_scatter": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_rmsnorm_bwd_partials": (c_i64, [c_i64, c_i64]),
    "lv_rmsnorm_bwd": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_f32, c_ptr]),
    "lv_swiglu_bwd": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_layernorm_bwd_partials": (c_i64, [c_i64, c_i64]),
    "lv_layernorm_bwd": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_f32, c_ptr]),
    "lv_gelu_bwd": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i32, c_ptr]),
    "lv_ls_residual_bwd_partials": (c_i64, [c_i64, c_i64]),
    "lv_ls_residual_bwd": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_ptr]),
    "lv_pixel_shuffle_bwd": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i32, c_ptr]),
    "lv_patch_im2col": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr]),
    "lv_frame_preprocess_ws_bytes": (c_i64, [c_i64, c_i64, c_i64, c_i64]),
    "lv_frame_preprocess": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr, c_ptr]),
    "lv_image_tiles_ws_bytes": (c_i64, [c_i64, c_i64]),
    "lv_image_tiles_preprocess": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_i64,
                                          c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_ptr, c_ptr, c_ptr]),
    "lv_ce_accumulate": (c_i32, [c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_ce_grad": (c_i32, [c_ptr, c_i64, c_ptr, c_i64, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_attn_decode_merge": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr]),
    "lv_attn_decode_host": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f32,
                                    c_ptr]),
    "lv_host_alloc": (c_i32, [c_i64, C.POINTER(c_ptr)]),
    "lv_host_free": (c_i32, [c_ptr]),
    "lv_rows_to_host": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_rows_to_host_fp8": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr]),
    "lv_attn_decode_host_fp8": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f32,
                                        c_ptr]),
    "lv_kv_rows_dequant_fp8": (c_i32, [c_ptr, c_ptr, c_i64, c_i64, c_i64, c_ptr]),
    "lv_gemm_bias_act": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i32, c_ptr]),
    "lv_gemm_ex": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i32, c_i32, c_i32,
                           c_ptr]),
    "lv_gemm_wgrad_acc_f32": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i32, c_i32, c_ptr]),
    "lv_quant_rows_fp8_fmt": (c_i32, [c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i32, c_ptr]),
    "lv_gemm_fp8": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i32,
                            c_ptr]),
    "lv_quant_cols_fp8_t": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i32, c_ptr]),
    "lv_gemm_fp8_grad": (c_i32, [c_ptr, c_i32, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                                 c_i32, c_ptr]),
    "lv_patch_embed_ws_bytes": (c_i64, [c_i64, c_i64, c_i64, c_i64]),
    "lv_patch_embed": (c_i32, [c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_ptr, c_i64, c_i64, c_i64, c_i64, c_ptr]),
}


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(
                    f"CUDA extension {LIB_PATH} is missing: build it with `python long-vita_b200/build.py`. "
                    "long_vita_b200 has no CPU / PyTorch fallback."
                )
            handle = C.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(handle, name)  # AttributeError if the .so does not export it
                fn.restype = res
                fn.argtypes = args
            _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().lv_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")
