"""Host-side mirror of the reference's `qserve_backend` operator API on top of the C ABI.

Every public function has the name, positional argument order, argument meaning, ownership rules and error
behaviour (RuntimeError) of the pybind11 function it replaces (reference file:line in each docstring), so that
`qserve/modeling/layers/*` and `qserve/modeling/models/llama_w4a8_unpad.py` run unchanged against it.
PyTorch is used only for what the reference uses it for at this boundary: tensor metadata, the current CUDA
stream and the two outputs the reference ops allocate themselves.
"""
from __future__ import annotations

from typing import Optional

import torch

from ._lib import check, lib

_HALF = torch.float16


# --------------------------------------------------------------------------------------------------
# plumbing
# --------------------------------------------------------------------------------------------------


def _call(t: torch.Tensor, fn, *args) -> None:
    """Launch `fn(*args, stream)` on the current stream of t's device, with that device current (the reference ops hold an
    at::cuda::CUDAGuard on the input's device, fused_attention.cpp:203); raises RuntimeError on failure."""
    idx = t.device.index
    cur = torch.cuda.current_device()
    if idx is None or idx == cur:
        check(fn(*args, torch._C._cuda_getCurrentRawStream(cur)))
    else:
        with torch.cuda.device(idx):
            check(fn(*args, torch._C._cuda_getCurrentRawStream(idx)))


def _require(cond: bool, msg: str) -> None:
    if not cond:
        raise RuntimeError(msg)


def _cuda(t: torch.Tensor, name: str) -> None:
    _require(t.is_cuda, f"{name} must be on CUDA")  # CHECK_DEVICE, fused_attention.cpp:22


_workspaces: dict = {}
_retired: list = []  # outgrown workspaces, kept alive for graphs captured with them


def gemm_workspace(device: torch.device) -> torch.Tensor:
    """Zero-initialised once per device; afterwards owned by the library (self-cleaning split-K counters)."""
    key = ("gemm", device.index)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(lib.qs_gemm_workspace_bytes(), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def attention_workspace(device: torch.device, batch: int, num_heads: int, head_dim: int) -> torch.Tensor:
    key = ("attn", device.index)
    need = lib.qs_attention_workspace_bytes(batch, num_heads, head_dim)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < need:
        # a workspace that was handed out is never freed: a captured CUDA graph may still hold its address (the self-cleaning
        # counters inside must not alias reused memory on replay)
        if ws is not None:
            _retired.append(ws)
        with torch.cuda.device(device):
            ws = torch.zeros(need, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def set_pdl(enabled: bool) -> bool:
    """Toggle programmatic dependent launch for all subsequently launched kernels; returns the previous setting."""
    return bool(lib.qs_set_pdl(1 if enabled else 0))


# --------------------------------------------------------------------------------------------------
# qgemm_w4a8_per_chn / qgemm_w4a8_per_group / qgemm_w8a8
# --------------------------------------------------------------------------------------------------


def _gemm_common(in_feats, kernel, out_feats, k_div: int):
    _cuda(in_feats, "in_feats"); _cuda(kernel, "kernel"); _cuda(out_feats, "out_feats")
    _require(in_feats.dtype == torch.int8 and kernel.dtype == torch.int8, "in_feats and kernel must be int8")
    _require(out_feats.dtype == _HALF, "out_feats must be float16")
    _require(in_feats.is_contiguous() and kernel.is_contiguous() and out_feats.is_contiguous(), "GEMM operands must be contiguous")
    M, K = in_feats.size(0), in_feats.size(1)  # gemm_cuda.cu:604-605
    N = out_feats.size(-1)                     # gemm_cuda.cu:613
    _require(out_feats.size(-2) == M, "out_feats rows must match in_feats rows")
    _require(kernel.size(0) == N and kernel.size(1) * k_div == K, f"kernel shape {tuple(kernel.shape)} does not match N={N}, K={K}")
    return M, N, K


def w4a8_per_chn_gemm_forward_cuda(in_feats, kernel, wscales, ascales, w_szs, a_ssums, out_feats, _acc_out=None) -> None:
    """qserve_backend.qgemm_w4a8_per_chn.gemm_forward_cuda (w4a8_per_chn/gemm_cuda.cu:596-652, pybind.cpp:13-16).

    out_feats[M,N] (fp16, caller allocated) = (in_feats s8 [M,K] . kernel u4 [N,K/2]) * wscales[n] * ascales[m] - w_szs[n] * a_ssums[m].
    """
    M, N, K = _gemm_common(in_feats, kernel, out_feats, 2)
    if M == 0:
        return
    ws = gemm_workspace(in_feats.device)
    _call(in_feats, lib.qs_w4a8_gemm_per_chn, in_feats.data_ptr(), kernel.data_ptr(), wscales.data_ptr(), ascales.data_ptr(), w_szs.data_ptr(),
                                   a_ssums.data_ptr(), out_feats.data_ptr(), _acc_out.data_ptr() if _acc_out is not None else None,
                                   M, N, K, ws.data_ptr(), ws.numel())


def w4a8_per_group_gemm_forward_cuda(in_feats, kernel, zeros, scales_i8, wscales, ascales, out_feats, _acc_out=None) -> None:
    """qserve_backend.qgemm_w4a8_per_group.gemm_forward_cuda (w4a8_per_group/gemm_cuda.cu:630-702).

    Argument order as called by w4a8_linear.py:123-131: (x, qweight, s2_zeros, s2_scales, s1_scales, input_scales, out).
    """
    M, N, K = _gemm_common(in_feats, kernel, out_feats, 2)
    _require(zeros.dtype == torch.int8 and scales_i8.dtype == torch.int8, "zeros and scales_i8 must be int8")
    _require(tuple(zeros.shape) == (K // 128, N) and tuple(scales_i8.shape) == (K // 128, N), "level-2 params must be [K/128, N]")
    if M == 0:
        return
    ws = gemm_workspace(in_feats.device)
    _call(in_feats, lib.qs_w4a8_gemm_per_group, in_feats.data_ptr(), kernel.data_ptr(), zeros.data_ptr(), scales_i8.data_ptr(), wscales.data_ptr(),
                                     ascales.data_ptr(), out_feats.data_ptr(), _acc_out.data_ptr() if _acc_out is not None else None,
                                     M, N, K, ws.data_ptr(), ws.numel())


def w8a8_gemm_forward_cuda(in_feats, kernel, wscales, ascales, out_feats, _acc_out=None) -> None:
    """qserve_backend.qgemm_w8a8.w8a8_gemm_forward_cuda (w8a8/w8a8_gemm_cuda.cu:532-577, pybind.cpp:13-17)."""
    M, N, K = _gemm_common(in_feats, kernel, out_feats, 1)
    _require(wscales.dtype == _HALF and ascales.dtype == _HALF, "wscales and ascales must be float16 (w8a8_linear.py:99-101 casts them)")
    if M == 0:
        return
    ws = gemm_workspace(in_feats.device)
    _call(in_feats, lib.qs_w8a8_gemm, in_feats.data_ptr(), kernel.data_ptr(), wscales.data_ptr(), ascales.data_ptr(), out_feats.data_ptr(),
                           _acc_out.data_ptr() if _acc_out is not None else None, M, N, K, ws.data_ptr(), ws.numel())


# --------------------------------------------------------------------------------------------------
# fused_attention
# --------------------------------------------------------------------------------------------------


def single_query_attention(q, k, v, kv_pointers, length_per_sample_: Optional[torch.Tensor], alibi_slopes_: Optional[torch.Tensor],
                           memory_max_seqlen: int, tokens_per_block: int, size_per_token: int, timestep: int,
                           rotary_embedding_dim: int, rotary_base: float, neox_rotary_style: bool, int4_kv_cache: bool,
                           kv_cache_with_zeros: bool) -> torch.Tensor:
    """qserve_backend.fused_attention.single_query_attention (fused_attention.cpp:150-240).

    Returns a NEW tensor shaped like q (the reference returns torch::empty_like(q), :205).  Mutates the KV pages.
    """
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (kv_pointers, "kv_pointers")):
        _cuda(t, n)
    _require(q.dtype == _HALF and k.dtype == _HALF and v.dtype == _HALF, "single_query_attention: only float16 is supported (fused_attention.cpp:24-30)")
    batch = kv_pointers.size(0)
    nheads, nheads_kv, headdim = q.size(1), k.size(1), k.size(-1)
    _require(k.stride(2) == 1 and k.stride(1) == headdim, "k must have stride(2) == 1 and stride(1) == head_dim")  # :179
    _require(v.stride(2) == 1 and v.stride(1) == headdim, "v must have stride(2) == 1 and stride(1) == head_dim")  # :180
    _require(q.stride(2) == 1 and q.stride(1) == headdim, "q must have stride(2) == 1 and stride(1) == head_dim")
    _require(kv_pointers.is_contiguous() and kv_pointers.dtype == torch.int64, "kv_pointers must be contiguous int64")  # :182
    lens_ptr = None
    if length_per_sample_ is not None:
        _cuda(length_per_sample_, "length_per_sample")
        _require(tuple(length_per_sample_.shape) == (batch,), "length_per_sample must have shape (batch_size)")
        _require(length_per_sample_.is_contiguous(), "length_per_sample must be contiguous")
        _require(length_per_sample_.dtype == torch.int32, "length_per_sample must be int32")  # :189
        lens_ptr = length_per_sample_.data_ptr()
    if alibi_slopes_ is not None:  # accepted, validated and ignored, exactly like the reference (:192-199, :91)
        _cuda(alibi_slopes_, "alibi_slopes")
        _require(tuple(alibi_slopes_.shape) == (nheads,) and alibi_slopes_.dtype == torch.float32, "alibi_slopes must be float32 [nheads]")
    out = torch.empty((q.size(0), nheads, headdim), dtype=q.dtype, device=q.device)
    ws = attention_workspace(q.device, batch, nheads, headdim)
    _call(q, lib.qs_single_query_attention, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), kv_pointers.data_ptr(),
                                        lens_ptr, out.data_ptr(), batch, nheads, nheads_kv, headdim, kv_pointers.size(-1), int(memory_max_seqlen),
                                        int(tokens_per_block), int(size_per_token), int(timestep), int(rotary_embedding_dim), float(rotary_base),
                                        int(bool(neox_rotary_style)), int(bool(int4_kv_cache)), int(bool(kv_cache_with_zeros)), ws.data_ptr(),
                                        ws.numel())
    return out


def apply_bias_rope_update_kv_cache(qkv, seq_lens, padding_offset, kv_pointers: Optional[torch.Tensor], head_num: int, kv_head_num: int,
                                    seq_len: int, tokens_per_block: int, size_per_token: int, rotary_embedding_dim: int,
                                    rotary_embedding_base: float, rotary_embedding_max_positions: int, neox_rotary_style: bool,
                                    int4_kv_cache: bool, kv_cache_with_zeros: bool) -> None:
    """qserve_backend.fused_attention.apply_bias_rope_update_kv_cache (update_kv_cache.cu:20-108): in-place RoPE on the
    packed qkv [T,(Hq+2Hkv)*D] and per-token-per-head asymmetric quantisation of K/V into the pages."""
    _cuda(qkv, "qkv")
    _require(qkv.dtype == _HALF and qkv.is_contiguous(), "qkv must be contiguous float16")
    _require(seq_lens.dtype == torch.int32 and padding_offset.dtype == torch.int32, "seq_lens and padding_offset must be int32")
    head_dim = int(rotary_embedding_dim)  # size_per_head = rotary_embedding_dim (update_kv_cache.cu:54)
    _require(qkv.size(-1) == (head_num + 2 * kv_head_num) * head_dim, "qkv width does not match (head_num + 2*kv_head_num) * head_dim")
    kvp, max_blocks = None, 0
    if kv_pointers is not None:
        _require(kv_pointers.is_contiguous() and kv_pointers.dtype == torch.int64, "kv_pointers must be contiguous int64")
        kvp, max_blocks = kv_pointers.data_ptr(), kv_pointers.size(-1)
    _call(qkv, lib.qs_apply_bias_rope_update_kv_cache, qkv.data_ptr(), seq_lens.data_ptr(), padding_offset.data_ptr(), kvp, seq_lens.size(0), qkv.size(0),
                                                 max_blocks, int(head_num), int(kv_head_num), head_dim, int(seq_len), int(tokens_per_block),
                                                 int(size_per_token), int(rotary_embedding_dim), float(rotary_embedding_base),
                                                 int(rotary_embedding_max_positions), int(bool(neox_rotary_style)), int(bool(int4_kv_cache)),
                                                 int(bool(kv_cache_with_zeros)))


def compute_padding_offsets(cu_seqlens, max_seqlen: int, tot_num_tokens: int) -> torch.Tensor:
    """qserve_backend.fused_attention.compute_padding_offsets (input_metadata_helper.cu:33-45): returns int32 [tot_num_tokens]."""
    _cuda(cu_seqlens, "cu_seqlens")
    _require(cu_seqlens.dtype == torch.int32, "cu_seqlens must be int32")
    out = torch.empty((tot_num_tokens,), dtype=torch.int32, device=cu_seqlens.device)
    _call(cu_seqlens, lib.qs_compute_padding_offsets, out.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.size(0) - 1, int(max_seqlen))
    return out


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q: int, max_seqlen_k: int, dropout_p: float = 0.0,
                           softmax_scale: Optional[float] = None, causal: bool = False, **unsupported) -> torch.Tensor:
    """Drop-in for the ONE way the reference calls flash_attn.flash_attn_varlen_func (llama_w4a8_unpad.py:232-242): causal self-attention over a
    batch of prompts, q [T,Hq,128], k / v [T,Hkv,128] fp16 (strided views of the rotated qkv buffer are fine), the same cu_seqlens for queries
    and keys, no dropout.  Returns fp16 [T,Hq,128].  Anything else raises: this is not a general flash-attention."""
    _cuda(q, "q")
    _require(not unsupported or all(val in (None, False, 0, 0.0, (-1, -1)) for val in unsupported.values()), f"unsupported arguments {sorted(unsupported)}")
    _require(causal and float(dropout_p) == 0.0, "only causal=True, dropout_p=0.0 is implemented")
    _require(q.dtype == _HALF and k.dtype == _HALF and v.dtype == _HALF, "q, k, v must be float16")
    _require(q.dim() == 3 and k.dim() == 3 and v.dim() == 3 and q.size(2) == 128 and k.size(2) == 128 and v.size(2) == 128, "q, k, v must be [T, H, 128]")
    _require(k.shape == v.shape and q.size(0) == k.size(0), "q, k, v must cover the same tokens; k and v the same heads")
    _require(cu_seqlens_q.dtype == torch.int32 and cu_seqlens_q.is_contiguous(), "cu_seqlens must be contiguous int32")
    _require(cu_seqlens_k is cu_seqlens_q or (cu_seqlens_k.shape == cu_seqlens_q.shape and cu_seqlens_k.data_ptr() == cu_seqlens_q.data_ptr())
             or bool(torch.equal(cu_seqlens_k, cu_seqlens_q)), "queries and keys must share cu_seqlens (prompt self-attention)")
    _require(int(max_seqlen_q) == int(max_seqlen_k), "max_seqlen_q and max_seqlen_k must agree")
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        _require(t.stride(2) == 1 and t.stride(1) == 128, f"{name}: heads must be contiguous rows of 128 halfs")
    T, hq, hkv = q.size(0), q.size(1), k.size(1)
    out = torch.empty((T, hq, 128), dtype=_HALF, device=q.device)
    if T == 0:
        return out
    scale = float(softmax_scale) if softmax_scale is not None else 128 ** -0.5
    _call(q, lib.qs_prefill_attention, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), out.data_ptr(), out.stride(0),
          cu_seqlens_q.data_ptr(), cu_seqlens_q.size(0) - 1, T, int(max_seqlen_q), hq, hkv, 128, scale)
    return out


# --------------------------------------------------------------------------------------------------
# layernorm_ops
# --------------------------------------------------------------------------------------------------


def _rows(t: torch.Tensor):
    hidden = t.size(-1)
    return (t.numel() // hidden if hidden else 0), hidden


def _noop(t: torch.Tensor) -> bool:
    """Empty batches are a no-op (the reference launches a zero-sized grid); data_ptr() of an empty tensor is NULL."""
    return t.numel() == 0


def _half_only(t: torch.Tensor, op: str) -> None:
    _require(t.dtype == _HALF, f"{op}: only float16 activations are supported by qserve_b200 (models run .half(), model_runner.py:148)")


def rms_norm(out, input, weight, epsilon: float, use_quant: bool = False) -> None:
    """layernorm_ops.rms_norm (layernorm.cpp:48-50, layernorm_kernels.cu:404-425)."""
    _cuda(input, "input"); _half_only(input, "rms_norm")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_rms_norm, out.data_ptr(), input.data_ptr(), weight.data_ptr(), float(epsilon), int(bool(use_quant)), tokens, hidden)


def rms_norm_general(out, input, weight, scaling, epsilon: float, use_per_token_quant: bool = False) -> None:
    """layernorm_ops.rms_norm_general (layernorm.cpp:52-54, layernorm_kernels.cu:427-464)."""
    _cuda(input, "input"); _half_only(input, "rms_norm_general")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_rms_norm_general, out.data_ptr(), input.data_ptr(), weight.data_ptr(), scaling.data_ptr(), float(epsilon),
                                  int(bool(use_per_token_quant)), tokens, hidden)


def rms_norm_general_fuse_sum(out, input, weight, input_sum, scaling, epsilon: float, use_per_token_quant: bool = False) -> None:
    """layernorm_ops.rms_norm_general_fuse_sum (layernorm.cpp:56-58, layernorm_kernels.cu:466-508)."""
    _cuda(input, "input"); _half_only(input, "rms_norm_general_fuse_sum")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_rms_norm_general_fuse_sum, out.data_ptr(), input.data_ptr(), weight.data_ptr(), input_sum.data_ptr(), scaling.data_ptr(),
                                           float(epsilon), int(bool(use_per_token_quant)), tokens, hidden)


def invoke_dequant_add_residual_rms_norm_quant(out, input, residual, gamma, scale, epsilon: float) -> None:
    """layernorm_ops.invoke_dequant_add_residual_rms_norm_quant, scalar-Half and Tensor scale overloads (layernorm.cpp:60-71)."""
    _cuda(input, "input"); _half_only(residual, "invoke_dequant_add_residual_rms_norm_quant")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    if isinstance(scale, torch.Tensor):
        _call(input, lib.qs_dequant_add_residual_rms_norm_quant, out.data_ptr(), input.data_ptr(), residual.data_ptr(), gamma.data_ptr(), scale.data_ptr(), 0.0,
                                                         float(epsilon), tokens, hidden)
    else:
        s = float(torch.tensor(float(scale), dtype=_HALF))  # at::Half argument
        _call(input, lib.qs_dequant_add_residual_rms_norm_quant, out.data_ptr(), input.data_ptr(), residual.data_ptr(), gamma.data_ptr(), None, s,
                                                         float(epsilon), tokens, hidden)


# --------------------------------------------------------------------------------------------------
# fused_kernels
# --------------------------------------------------------------------------------------------------


def invoke_quant(out, input, scale) -> None:
    """fused_kernels.invoke_quant: Tensor scale [tokens] (written) or scalar Half scale (read)  (fused.cpp:52-58)."""
    _cuda(input, "input"); _half_only(input, "invoke_quant")
    _require(input.is_contiguous() and out.is_contiguous(), "invoke_quant: input and out must be contiguous")  # asserts, fused_kernels.cu:202-203
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    if isinstance(scale, torch.Tensor):
        _call(input, lib.qs_invoke_quant, out.data_ptr(), input.data_ptr(), scale.data_ptr(), tokens, hidden)
    else:
        s = float(torch.tensor(float(scale), dtype=_HALF))
        _call(input, lib.qs_invoke_quant_scalar, out.data_ptr(), input.data_ptr(), s, tokens, hidden)


def invoke_quant_fuse_sum(out, input, input_sum, scale) -> None:
    """fused_kernels.invoke_quant_fuse_sum (fused.cpp:59-69, fused_kernels.cu:234-265)."""
    _cuda(input, "input"); _half_only(input, "invoke_quant_fuse_sum")
    _require(input.is_contiguous() and out.is_contiguous(), "invoke_quant_fuse_sum: input and out must be contiguous")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    if isinstance(scale, torch.Tensor):
        _call(input, lib.qs_invoke_quant_fuse_sum, out.data_ptr(), input.data_ptr(), input_sum.data_ptr(), scale.data_ptr(), tokens, hidden)
    else:  # scalar overload: static scale, the sum argument is unused by the reference kernel (fused_kernels.cu:131-136)
        s = float(torch.tensor(float(scale), dtype=_HALF))
        _call(input, lib.qs_invoke_quant_scalar, out.data_ptr(), input.data_ptr(), s, tokens, hidden)


def invoke_dequant_add_residual(out, input, residual, scale) -> None:
    """fused_kernels.invoke_dequant_add_residual, both overloads (fused.cpp:48-55)."""
    _cuda(input, "input"); _half_only(residual, "invoke_dequant_add_residual")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    if isinstance(scale, torch.Tensor):
        _call(input, lib.qs_invoke_dequant_add_residual, out.data_ptr(), input.data_ptr(), residual.data_ptr(), scale.data_ptr(), 0.0, tokens, hidden)
    else:
        s = float(torch.tensor(float(scale), dtype=_HALF))
        _call(input, lib.qs_invoke_dequant_add_residual, out.data_ptr(), input.data_ptr(), residual.data_ptr(), None, s, tokens, hidden)


def invoke_dequant(out, input, scale) -> None:
    """fused_kernels.invoke_dequant (fused.cpp:56, fused_kernels.cu:179-196)."""
    _cuda(input, "input"); _half_only(out, "invoke_dequant")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    s = float(torch.tensor(float(scale), dtype=_HALF))
    _call(input, lib.qs_invoke_dequant, out.data_ptr(), input.data_ptr(), s, tokens, hidden, input.stride(-2), out.stride(-2))


# --------------------------------------------------------------------------------------------------
# activation_ops
# --------------------------------------------------------------------------------------------------


def silu_and_mul(out, input) -> None:
    """activation_ops.silu_and_mul (activation.cpp:26, activation_kernels.cu:84-97): out[..., d] = silu(x[..., :d]) * x[..., d:]."""
    _cuda(input, "input"); _half_only(input, "silu_and_mul")
    if _noop(input):
        return
    d = input.size(-1) // 2
    tokens = input.numel() // input.size(-1) if input.size(-1) else 0
    _call(input, lib.qs_silu_and_mul, out.data_ptr(), input.data_ptr(), tokens, d)


def gelu_new(out, input) -> None:
    """activation_ops.gelu_new (activation.cpp:27)."""
    _cuda(input, "input"); _half_only(input, "gelu_new")
    tokens, d = _rows(input)
    _call(input, lib.qs_gelu_new, out.data_ptr(), input.data_ptr(), tokens, d)


def gelu_fast(out, input) -> None:
    """activation_ops.gelu_fast (activation.cpp:28)."""
    _cuda(input, "input"); _half_only(input, "gelu_fast")
    tokens, d = _rows(input)
    _call(input, lib.qs_gelu_fast, out.data_ptr(), input.data_ptr(), tokens, d)


def invoke_dequant_silu_and_mul_quant(out, input, scale_gate: float, scale_up: float, scale_out, tmp: Optional[torch.Tensor] = None) -> None:
    """activation_ops.invoke_dequant_silu_and_mul_quant, scalar and per-token overloads (activation.cpp:29-38)."""
    _cuda(input, "input")
    d = input.size(-1) // 2
    tokens = input.numel() // input.size(-1) if input.size(-1) else 0
    if isinstance(scale_out, torch.Tensor):
        _require(tmp is not None, "per-token overload needs the tmp buffer")
        _call(input, lib.qs_dequant_silu_and_mul_quant, out.data_ptr(), input.data_ptr(), float(scale_gate), float(scale_up), 0.0, scale_out.data_ptr(),
                                                tmp.data_ptr(), tokens, d)
    else:
        _call(input, lib.qs_dequant_silu_and_mul_quant, out.data_ptr(), input.data_ptr(), float(scale_gate), float(scale_up), float(scale_out), None, None,
                                                tokens, d)


# --------------------------------------------------------------------------------------------------
# fused extensions (not part of the reference surface; bit-identical to the op sequences they replace)
# --------------------------------------------------------------------------------------------------


def add_rms_norm_general(out, hidden_out, x, delta, weight, input_sum: Optional[torch.Tensor], scaling, epsilon: float) -> None:
    """hidden_out = x + delta (fp16, as torch computes `residual + out_buf`), then rms_norm_general[_fuse_sum](out, hidden_out, ...)."""
    _cuda(x, "x"); _half_only(x, "add_rms_norm_general"); _half_only(delta, "add_rms_norm_general")
    if _noop(x):
        return
    tokens, hidden = _rows(x)
    _call(x, lib.qs_add_rms_norm_general, out.data_ptr(), hidden_out.data_ptr(), x.data_ptr(), delta.data_ptr(), weight.data_ptr(),
                                      input_sum.data_ptr() if input_sum is not None else None, scaling.data_ptr(), float(epsilon), tokens, hidden)


def silu_and_mul_quant(out, input, input_sum: Optional[torch.Tensor], scale) -> None:
    """silu_and_mul(input) followed by invoke_quant[_fuse_sum]; the fp16 activation never leaves the SM."""
    _cuda(input, "input"); _half_only(input, "silu_and_mul_quant")
    if _noop(input):
        return
    d = input.size(-1) // 2
    tokens = input.numel() // input.size(-1)
    _call(input, lib.qs_silu_and_mul_quant, out.data_ptr(), input.data_ptr(), input_sum.data_ptr() if input_sum is not None else None, scale.data_ptr(),
                                    tokens, d)


def single_query_attention_quant(q, k, v, kv_pointers, length_per_sample, memory_max_seqlen: int, tokens_per_block: int, size_per_token: int,
                                 timestep: int, rotary_embedding_dim: int, rotary_base: float, int4_kv_cache: bool, kv_cache_with_zeros: bool,
                                 out_q, out_scale, out_sum: Optional[torch.Tensor]) -> None:
    """single_query_attention + invoke_quant[_fuse_sum] in one launch: out_q int8 [B, Hq*D], out_scale / out_sum fp16 [B].
    Bit-identical to the two reference ops run back to back (llama_w4a8_unpad.py:265-283)."""
    batch = kv_pointers.size(0)
    if batch == 0:
        return
    nheads, nheads_kv, headdim = q.size(1), k.size(1), k.size(-1)
    _require(q.dtype == _HALF and q.stride(2) == 1 and q.stride(1) == headdim, "q must be float16 with stride(1) == head_dim")
    _require(k.stride(1) == headdim and v.stride(1) == headdim and kv_pointers.is_contiguous(), "k, v, kv_pointers layout")
    _require(out_q.dtype == torch.int8 and out_q.is_contiguous() and out_q.numel() == batch * nheads * headdim, "out_q must be int8 [B, Hq*D]")
    ws = attention_workspace(q.device, batch, nheads, headdim)
    _call(q, lib.qs_single_query_attention_quant, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), kv_pointers.data_ptr(),
                                              length_per_sample.data_ptr(), out_q.data_ptr(), out_scale.data_ptr(),
                                              out_sum.data_ptr() if out_sum is not None else None, batch, nheads, nheads_kv, headdim,
                                              kv_pointers.size(-1), int(memory_max_seqlen), int(tokens_per_block), int(size_per_token), int(timestep),
                                              int(rotary_embedding_dim), float(rotary_base), int(bool(int4_kv_cache)), int(bool(kv_cache_with_zeros)),
                                              ws.data_ptr(), ws.numel())


def apply_bias_rope_update_kv_cache_at(qkv, seq_lens, padding_offset, start_pos, kv_pointers: Optional[torch.Tensor], head_num: int,
                                       kv_head_num: int, seq_len: int, tokens_per_block: int, size_per_token: int, rotary_embedding_dim: int,
                                       rotary_embedding_base: float, rotary_embedding_max_positions: int, neox_rotary_style: bool,
                                       int4_kv_cache: bool, kv_cache_with_zeros: bool) -> None:
    """apply_bias_rope_update_kv_cache for prompt CHUNKS that continue sequences whose first start_pos[b] tokens (int32 [B], device) are
    already cached: seq_lens are the chunk lengths, token pos of chunk b is rotated at position start_pos[b] + pos and appended there.
    Appending a prompt in chunks leaves the same bytes as one apply_bias_rope_update_kv_cache call over the whole prompt."""
    for t, n in ((qkv, "qkv"), (seq_lens, "seq_lens"), (padding_offset, "padding_offset"), (start_pos, "start_pos")):
        _cuda(t, n)
    _require(qkv.dtype == _HALF and qkv.is_contiguous(), "qkv must be contiguous float16")
    _require(seq_lens.dtype == torch.int32 and padding_offset.dtype == torch.int32, "seq_lens and padding_offset must be int32")
    _require(start_pos.dtype == torch.int32 and start_pos.is_contiguous() and tuple(start_pos.shape) == (seq_lens.size(0),),
             "start_pos must be contiguous int32 [batch]")
    head_dim = int(rotary_embedding_dim)
    _require(head_dim == 128, "apply_bias_rope_update_kv_cache_at: head_dim must be 128")
    _require(qkv.size(-1) == (head_num + 2 * kv_head_num) * head_dim, "qkv width does not match (head_num + 2*kv_head_num) * head_dim")
    kvp, max_blocks = None, 0
    if kv_pointers is not None:
        _cuda(kv_pointers, "kv_pointers")
        _require(kv_pointers.is_contiguous() and kv_pointers.dtype == torch.int64, "kv_pointers must be contiguous int64")
        kvp, max_blocks = kv_pointers.data_ptr(), kv_pointers.size(-1)
    _call(qkv, lib.qs_apply_bias_rope_update_kv_cache_at, qkv.data_ptr(), seq_lens.data_ptr(), padding_offset.data_ptr(), start_pos.data_ptr(), kvp,
          seq_lens.size(0), qkv.size(0), max_blocks, int(head_num), int(kv_head_num), head_dim, int(seq_len), int(tokens_per_block),
          int(size_per_token), int(rotary_embedding_dim), float(rotary_embedding_base), int(rotary_embedding_max_positions),
          int(bool(neox_rotary_style)), int(bool(int4_kv_cache)), int(bool(kv_cache_with_zeros)))


def prefix_prefill_attention(q, k, v, cu_seqlens, max_seqlen: int, prefix_lens, max_prefix_len: int, kv_pointers, tokens_per_block: int,
                             size_per_token: int, int4_kv_cache: bool, softmax_scale: Optional[float] = None) -> torch.Tensor:
    """Causal attention of a batch of prompt chunks over their cached prefix.  q [T,Hq,128], k / v [T,Hkv,128] fp16 (strided views of the qkv
    buffer apply_bias_rope_update_kv_cache_at has rotated), cu_seqlens int32 [B+1] chunk offsets, prefix_lens int32 [B] cached tokens,
    kv_pointers int64 [B,2,max_blocks] page addresses (the block table covers the prefix and the chunk).  Query i of sequence b attends to the
    prefix keys dequantised from the ZINT4 / ZINT8 pages and to chunk keys 0..i in fp16.  max_prefix_len bounds prefix_lens (it is not checked
    on the device).  Returns fp16 [T,Hq,128]."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (cu_seqlens, "cu_seqlens"), (prefix_lens, "prefix_lens"), (kv_pointers, "kv_pointers")):
        _cuda(t, n)
    _require(q.dtype == _HALF and k.dtype == _HALF and v.dtype == _HALF, "q, k, v must be float16")
    _require(q.dim() == 3 and k.dim() == 3 and v.dim() == 3 and q.size(2) == 128 and k.size(2) == 128 and v.size(2) == 128, "q, k, v must be [T, H, 128]")
    _require(k.shape == v.shape and q.size(0) == k.size(0), "q, k, v must cover the same tokens; k and v the same heads")
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        _require(t.stride(2) == 1 and t.stride(1) == 128, f"{name}: heads must be contiguous rows of 128 halfs")
    _require(cu_seqlens.dtype == torch.int32 and cu_seqlens.is_contiguous() and cu_seqlens.dim() == 1, "cu_seqlens must be contiguous int32")
    batch = cu_seqlens.size(0) - 1
    _require(prefix_lens.dtype == torch.int32 and prefix_lens.is_contiguous() and tuple(prefix_lens.shape) == (batch,), "prefix_lens must be contiguous int32 [batch]")
    _require(kv_pointers.dtype == torch.int64 and kv_pointers.is_contiguous() and kv_pointers.dim() == 3 and kv_pointers.size(0) == batch
             and kv_pointers.size(1) == 2, "kv_pointers must be contiguous int64 [batch, 2, max_blocks]")
    _require(int(tokens_per_block) == 64, "tokens_per_block must be 64")
    T, hq, hkv = q.size(0), q.size(1), k.size(1)
    _require(hq % hkv == 0, "num_heads must be a multiple of num_kv_heads")
    _require(int(size_per_token) == hkv * 128 * (4 if int4_kv_cache else 8) // 8, "size_per_token does not match the kv heads and the cache type")
    _require(int(max_prefix_len) >= 0 and int(max_seqlen) >= 0, "negative max_prefix_len / max_seqlen")
    _require(int(max_prefix_len) + int(max_seqlen) <= kv_pointers.size(-1) * 64, "the page table is too short for max_prefix_len + max_seqlen")
    out = torch.empty((T, hq, 128), dtype=_HALF, device=q.device)
    if T == 0 or batch == 0:
        return out
    scale = float(softmax_scale) if softmax_scale is not None else 128 ** -0.5
    _call(q, lib.qs_prefix_prefill_attention, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), out.data_ptr(), out.stride(0),
          cu_seqlens.data_ptr(), prefix_lens.data_ptr(), kv_pointers.data_ptr(), batch, T, int(max_seqlen), int(max_prefix_len), kv_pointers.size(-1),
          hq, hkv, 128, int(tokens_per_block), int(size_per_token), int(bool(int4_kv_cache)), scale)
    return out


class PeerContext:
    """Peer-mapped buffers of a tensor-parallel group for the fused all-reduce (qs_add_rms_norm_general_peer): built once from
    torch.distributed._symmetric_memory (device memory + NVLink peer mappings are torch's plumbing; the kernel is ours).
    Layout of the symmetric allocation on every rank: [2 phases][tokens, hidden] fp16 partial outputs, then a 256-byte flag pad."""

    def __init__(self, tokens: int, hidden: int, device: torch.device, group):
        import ctypes

        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        _require(self.world <= 8, "PeerContext: at most 8 ranks")
        self.tokens, self.hidden = tokens, hidden
        phase_bytes = tokens * hidden * 2
        with torch.cuda.device(device):
            self.buf = symm.empty(2 * phase_bytes + 256, dtype=torch.uint8, device=device)
            self.buf.zero_()
            self.handle = symm.rendezvous(self.buf, group.group_name if hasattr(group, "group_name") else group)
            self.state = torch.zeros(4, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group)  # every rank's pad is zeroed before anyone signals
        base = [int(p) for p in self.handle.buffer_ptrs]
        self.partial = [self.buf[p * phase_bytes:(p + 1) * phase_bytes].view(torch.float16).view(tokens, hidden) for p in range(2)]  # local GEMM outputs
        arr = ctypes.c_void_p * self.world
        self._delta = [arr(*[b + p * phase_bytes for b in base]) for p in range(2)]
        self._flags = arr(*[b + 2 * phase_bytes for b in base])


def add_rms_norm_general_peer(out, hidden_out, x, ctx: "PeerContext", phase: int, weight, input_sum: Optional[torch.Tensor], scaling, epsilon: float) -> None:
    """add_rms_norm_general with delta = the sum over the tensor-parallel ranks of ctx.partial[phase] (fused all-reduce over peer memory)."""
    _cuda(x, "x"); _half_only(x, "add_rms_norm_general_peer")
    if _noop(x):
        return
    tokens, hidden = _rows(x)
    _require(tokens == ctx.tokens and hidden == ctx.hidden, "add_rms_norm_general_peer: shape does not match the PeerContext")
    _call(x, lib.qs_add_rms_norm_general_peer, out.data_ptr(), hidden_out.data_ptr(), x.data_ptr(), ctx._delta[phase], ctx._flags, ctx.state.data_ptr(),
          ctx.world, ctx.rank, int(phase), weight.data_ptr(), input_sum.data_ptr() if input_sum is not None else None, scaling.data_ptr(), float(epsilon),
          tokens, hidden)


def row_absmax(amax_out: torch.Tensor, input: torch.Tensor) -> None:
    """Tensor-parallel extension: amax_out[t] (fp32) = max |input[t, :]| of this rank's shard (then max-all-reduced by the caller)."""
    _cuda(input, "input"); _half_only(input, "row_absmax")
    _require(input.is_contiguous() and amax_out.dtype == torch.float32, "row_absmax: contiguous fp16 input, fp32 output")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_row_absmax, amax_out.data_ptr(), input.data_ptr(), tokens, hidden)


def invoke_quant_given_amax(out, input, amax: torch.Tensor, input_sum: Optional[torch.Tensor], scale) -> None:
    """Tensor-parallel extension: invoke_quant[_fuse_sum] with a caller-supplied (global) per-token amax, fp32 [tokens]."""
    _cuda(input, "input"); _half_only(input, "invoke_quant_given_amax")
    _require(input.is_contiguous() and out.is_contiguous() and amax.dtype == torch.float32, "invoke_quant_given_amax: contiguous tensors, fp32 amax")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_invoke_quant_given_amax, out.data_ptr(), input.data_ptr(), amax.data_ptr(), input_sum.data_ptr() if input_sum is not None else None,
          scale.data_ptr(), tokens, hidden)


def argmax_rows(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torch.argmax(logits, dim=-1) for fp16 logits [rows, vocab] in one launch (greedy sampling of the decode runner)."""
    _cuda(logits, "logits")
    _require(logits.dtype == _HALF and logits.dim() == 2 and logits.is_contiguous(), "logits must be contiguous float16 [rows, vocab]")
    if out is None:
        out = torch.empty(logits.size(0), dtype=torch.int64, device=logits.device)
    if logits.size(0) == 0:
        return out
    _call(logits, lib.qs_argmax_rows, out.data_ptr(), logits.data_ptr(), logits.size(0), logits.size(1))
    return out
