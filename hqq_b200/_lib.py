"""ctypes binding of ``libhqq_b200.so`` (the C ABI declared in ``include/hqq_b200.h``).

There is no CPU fallback and no second backend: if the library is missing or cannot be
loaded, or a call is made without a CUDA device, this module raises -- loudly.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p

import torch

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libhqq_b200.so")

HQQ_F32, HQQ_F16, HQQ_BF16, HQQ_U8, HQQ_I32, HQQ_I64 = range(6)
HQQ_OK, HQQ_E_INVALID, HQQ_E_UNSUPPORTED, HQQ_E_WORKSPACE, HQQ_E_CUDA = 0, -1, -2, -3, -4

DTYPE_CODE = {
    torch.float32: HQQ_F32, torch.float16: HQQ_F16, torch.bfloat16: HQQ_BF16,
    torch.uint8: HQQ_U8, torch.int32: HQQ_I32, torch.int64: HQQ_I64,
}

# symbol -> (restype, argtypes); must list every function include/hqq_b200.h declares
SIGNATURES = {
    "hqq_b200_abi_version": (c_int, []),
    "hqq_b200_last_error": (c_char_p, []),
    "hqq_b200_pack": (c_int, [c_int, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p]),
    "hqq_b200_unpack": (c_int, [c_int, c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p]),
    "hqq_b200_dequantize": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_quantize_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "hqq_b200_quantize_shard_begin": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p,
                                              c_void_p, c_size_t, c_void_p]),
    "hqq_b200_quantize_shard_finish": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p,
                                               c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "hqq_b200_quantize": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "hqq_b200_quantize_ex": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float,
                                     c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_size_t, c_void_p]),
    "hqq_b200_linear_fwd_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "hqq_b200_dense_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "hqq_b200_lm_logprob_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "hqq_b200_lm_logprob": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p]),
    "hqq_b200_linear_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                    c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "hqq_b200_linear_fwd_multi": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
                                          c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "hqq_b200_linear_fwd_route": (c_int, [c_int64, c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "hqq_b200_linear_fwd_grouped": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                            c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_moe_route": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int] + [c_void_p] * 7 + [c_int, c_void_p]),
    "hqq_b200_glue_moe_combine": (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
    "hqq_b200_decode_linear_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_decode_linear_fwd_desc": (c_int, [c_void_p, c_void_p]),
    "hqq_b200_glue_add_rmsnorm_tp": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p]),
    "hqq_b200_glue_add_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p]),
    "hqq_b200_glue_add_rmsnorm_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_void_p]),
    "hqq_b200_glue_silu_mul": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                     c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                     c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "hqq_b200_glue_rope_append_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                               c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv8": (c_int, [c_void_p] * 14 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv8": (c_int, [c_void_p] * 14 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_attn_prefill": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "hqq_b200_glue_rope_attn_decode_batch_seqpos": (c_int, [c_void_p] * 9 + [c_int] * 6 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_seqpos": (c_int, [c_void_p] * 10 + [c_int] * 6 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv8_seqpos": (c_int, [c_void_p] * 14 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_varlen": (c_int, [c_void_p] * 10 + [c_int] * 6 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv8_varlen": (c_int, [c_void_p] * 16 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_attn_prefill_varlen": (c_int, [c_void_p] * 6 + [c_int] * 6 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_batch_paged": (c_int, [c_void_p] * 10 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_paged": (c_int, [c_void_p] * 11 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv8_paged": (c_int, [c_void_p] * 15 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_paged": (c_int, [c_void_p] * 11 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv8_paged": (c_int, [c_void_p] * 17 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_kv8_stage_paged": (c_int, [c_void_p] * 11 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_attn_prefill_paged": (c_int, [c_void_p] * 7 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_devpos": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_devpos_paged": (c_int, [c_void_p] * 10 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_workspace_bytes": (c_size_t, [c_int] * 5),
    "hqq_b200_glue_rope_append_rows_kv8_devpos": (c_int, [c_void_p] * 13 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv8_devpos_paged": (c_int, [c_void_p] * 14 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_kv8": (c_int, [c_void_p] * 10 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_kv8_paged": (c_int, [c_void_p] * 11 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv4": (c_int, [c_void_p] * 14 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv4_seqpos": (c_int, [c_void_p] * 14 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_attn_decode_split_kv4_paged": (c_int, [c_void_p] * 15 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv4": (c_int, [c_void_p] * 14 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv4_varlen": (c_int, [c_void_p] * 16 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv4_paged": (c_int, [c_void_p] * 17 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_kv4_stage": (c_int, [c_void_p] * 10 + [c_int] * 6 + [c_void_p]),
    "hqq_b200_glue_kv4_stage_paged": (c_int, [c_void_p] * 11 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv4_devpos": (c_int, [c_void_p] * 13 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_rope_append_rows_kv4_devpos_paged": (c_int, [c_void_p] * 14 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_kv4": (c_int, [c_void_p] * 10 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_kv4_paged": (c_int, [c_void_p] * 11 + [c_int] * 9 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split": (c_int, [c_void_p] * 6 + [c_int] * 7 + [c_void_p]),
    "hqq_b200_glue_attn_verify_split_paged": (c_int, [c_void_p] * 7 + [c_int] * 8 + [c_void_p]),
    "hqq_b200_glue_ngram_draft": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "hqq_b200_glue_spec_accept": (c_int, [c_void_p] * 8 + [c_int] * 3 + [c_void_p]),
    "hqq_b200_glue_argmax": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "hqq_b200_glue_argmax_key": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_void_p]),
    "hqq_b200_glue_argmax_tp": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "hqq_b200_glue_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64, c_void_p, c_void_p, c_int, c_void_p]),
    "hqq_b200_glue_sample_pos": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_int, c_float, ctypes.c_uint64, c_int, c_void_p, c_void_p, c_void_p,
                                         c_int, c_void_p]),
    "hqq_b200_glue_sample_slots": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, ctypes.c_uint64, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_int, c_void_p]),
    "hqq_b200_glue_penalize": (c_int, [c_void_p, c_int, c_int, c_int, c_int] + [c_void_p] * 7 + [c_int, c_int, c_void_p]),
    "hqq_b200_launch_count": (c_int64, []),
    "hqq_b200_launch_count_reset": (None, []),
    "hqq_b200_reload_env": (None, []),
}


ABI_VERSION = 2  # HQQ_B200_ABI_VERSION of include/hqq_b200.h this binding was written against


class DecodeDesc(ctypes.Structure):
    """Mirror of `hqq_b200_decode_desc` (include/hqq_b200.h)."""
    _fields_ = [("x", c_void_p), ("x_op", c_int), ("x2", c_void_p), ("x_weight", c_void_p), ("h_out", c_void_p), ("eps", c_float),
                ("count", c_int), ("W_q", c_void_p), ("scale", c_void_p), ("zero", c_void_p), ("bias", c_void_p), ("y", c_void_p),
                ("N", c_void_p), ("K", c_int64), ("group_size", c_int), ("nbits", c_int), ("dtype", c_int), ("tp", c_int), ("rank", c_int),
                ("peer_data", c_void_p), ("red_data", c_void_p), ("y_tagged", c_void_p), ("x_tagged", c_void_p), ("x2_tagged", c_void_p),
                ("step_ctr", c_void_p), ("x_index", c_int), ("x_per_step", c_int)]


class HQQB200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code


_lib = None


def load(path: str | None = None) -> ctypes.CDLL:
    """Load the shared library (once) and declare every prototype."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(
            f"hqq_b200: {p} not found. Build it with `python -m hqq_b200.build` (needs nvcc, sm_90a). "
            "There is no CPU or PyTorch fallback for this package.")
    lib = ctypes.CDLL(p)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means the .so is stale -> fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.hqq_b200_abi_version() != ABI_VERSION:
        raise RuntimeError("hqq_b200: ABI version mismatch between libhqq_b200.so and the Python layer; rebuild")
    if path is None:
        _lib = lib
    return lib


def last_error() -> str:
    return load().hqq_b200_last_error().decode("utf-8", "replace")


def check(rc: int) -> None:
    if rc == HQQ_OK:
        return
    msg = last_error()
    raise HQQB200Error(rc, msg or f"hqq_b200 call failed with code {rc}")


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"hqq_b200: {what} must live on a CUDA device (got {t.device}); there is no CPU path")


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()
