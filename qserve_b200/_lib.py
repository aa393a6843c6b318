"""ctypes binding of libqserve_b200.so (the C ABI declared in include/qserve_b200.h).

There is deliberately NO fallback: if the shared library is missing the import fails loudly, and every op
raises RuntimeError when the CUDA launch fails (for example on a machine without a GPU).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libqserve_b200.so")

# name -> (restype, argtypes); mirrors include/qserve_b200.h one to one
_P, _I, _F, _L, _Z = c_void_p, c_int, c_float, c_int64, c_size_t
SIGNATURES = {
    "qs_abi_version": (c_int, []),
    "qs_last_error": (c_char_p, []),
    "qs_set_pdl": (c_int, [_I]),
    "qs_w4a8_gemm_per_chn": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _Z, _P]),
    "qs_w4a8_gemm_per_group": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _Z, _P]),
    "qs_w8a8_gemm": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _Z, _P]),
    "qs_gemm_workspace_bytes": (c_size_t, []),
    "qs_argmax_rows": (c_int, [_P, _P, _I, _I, _P]),
    "qs_gemm_force_split": (c_int, [_I]),
    "qs_gemm_force_tile_tokens": (c_int, [_I]),
    "qs_gemm_set_profile_buffer": (c_int, [_P]),
    "qs_set_trace_buffer": (c_int, [_P, ctypes.c_uint]),
    "qs_single_query_attention": (c_int, [_P, _P, _P, _L, _L, _L, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _P, _Z, _P]),
    "qs_attention_workspace_bytes": (c_size_t, [_I, _I, _I]),
    "qs_single_query_attention_quant": (c_int, [_P, _P, _P, _L, _L, _L, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _P, c_size_t, _P]),
    "qs_apply_bias_rope_update_kv_cache": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _I, _P]),
    "qs_compute_padding_offsets": (c_int, [_P, _P, _I, _I, _P]),
    "qs_prefill_attention": (c_int, [_P, _P, _P, _L, _L, _L, _P, _L, _P, _I, _I, _I, _I, _I, _I, _F, _P]),
    "qs_apply_bias_rope_update_kv_cache_at": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _I, _P]),
    "qs_prefix_prefill_attention": (c_int, [_P, _P, _P, _L, _L, _L, _P, _L, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "qs_multi_token_decode_attention": (c_int, [_P, _P, _P, _L, _L, _L, _P, _L, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P, _Z, _P]),
    "qs_multi_token_attention_workspace_bytes": (c_size_t, [_I, _I, _I, _I, _I, _I, _I]),
    "qs_apply_bias_rope_update_kv_cache_tree": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _I, _P]),
    "qs_tree_decode_attention": (c_int, [_P, _P, _P, _L, _L, _L, _P, _L, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P, _Z, _P]),
    "qs_tree_accept_greedy": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "qs_kv_cache_compact": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "qs_kv_cache_fork": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "qs_sample_rows": (c_int, [_P, _P, _P, _P, _P, ctypes.c_uint64, _P, _I, _I, _P]),
    "qs_tree_accept_sampling": (c_int, [_P, _P, _P, _P, _P, _P, _P, ctypes.c_uint64, _P, _P, _P, _P, _I, _I, _I, _P]),
    "qs_apply_penalties": (c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "qs_logprobs_rows": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "qs_apply_penalties_tree": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "qs_logprobs_accepted": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "qs_ngram_propose": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "qs_spec_commit": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "qs_spec_commit_stops": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _P]),
    "qs_rms_norm": (c_int, [_P, _P, _P, _F, _I, _I, _I, _P]),
    "qs_rms_norm_general": (c_int, [_P, _P, _P, _P, _F, _I, _I, _I, _P]),
    "qs_rms_norm_general_fuse_sum": (c_int, [_P, _P, _P, _P, _P, _F, _I, _I, _I, _P]),
    "qs_dequant_add_residual_rms_norm_quant": (c_int, [_P, _P, _P, _P, _P, _F, _F, _I, _I, _P]),
    "qs_invoke_quant": (c_int, [_P, _P, _P, _I, _I, _P]),
    "qs_invoke_quant_scalar": (c_int, [_P, _P, _F, _I, _I, _P]),
    "qs_invoke_quant_fuse_sum": (c_int, [_P, _P, _P, _P, _I, _I, _P]),
    "qs_add_rms_norm_general_peer": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _F, _I, _I, _P]),
    "qs_row_absmax": (c_int, [_P, _P, _I, _I, _P]),
    "qs_invoke_quant_given_amax": (c_int, [_P, _P, _P, _P, _P, _I, _I, _P]),
    "qs_invoke_dequant_add_residual": (c_int, [_P, _P, _P, _P, _F, _I, _I, _P]),
    "qs_invoke_dequant": (c_int, [_P, _P, _F, _I, _I, _I, _I, _P]),
    "qs_silu_and_mul": (c_int, [_P, _P, _I, _I, _P]),
    "qs_silu_and_mul_quant": (c_int, [_P, _P, _P, _P, _I, _I, _P]),
    "qs_add_rms_norm_general": (c_int, [_P, _P, _P, _P, _P, _P, _P, _F, _I, _I, _P]),
    "qs_gelu_new": (c_int, [_P, _P, _I, _I, _P]),
    "qs_gelu_fast": (c_int, [_P, _P, _I, _I, _P]),
    "qs_dequant_silu_and_mul_quant": (c_int, [_P, _P, _F, _F, _F, _P, _P, _I, _I, _P]),
}

ABI_VERSION = 2


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found. Build it with `python -m qserve_b200.build` (needs nvcc). "
            "qserve_b200 has no CPU or PyTorch fallback path."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    got = lib.qs_abi_version()
    if got != ABI_VERSION:
        raise ImportError(f"libqserve_b200.so ABI version {got}, python binding expects {ABI_VERSION}: rebuild")
    return lib


lib = _load()


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError(f"qserve_b200 [{rc}]: {lib.qs_last_error().decode(errors='replace')}")
