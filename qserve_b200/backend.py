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


def _tensor(t: torch.Tensor, name: str, dtype: torch.dtype, shape: Optional[tuple] = None, device: Optional[torch.device] = None) -> torch.Tensor:
    """Require t to be a contiguous CUDA tensor of dtype, of exactly `shape` if given (a None entry leaves that dimension free) and on
    `device` if given; returns t."""
    _cuda(t, name)
    if t.dtype != dtype or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous {dtype} tensor, got {t.dtype}")
    if shape is not None and (t.dim() != len(shape) or any(s is not None and s != d for s, d in zip(shape, t.shape))):
        raise RuntimeError(f"{name} must have shape {tuple('*' if s is None else s for s in shape)}, got {tuple(t.shape)}")
    if device is not None and t.device != device:
        raise RuntimeError(f"{name} is on {t.device}, the other tensors on {device}")
    return t


def _out(t: Optional[torch.Tensor], name: str, dtype: torch.dtype, shape: tuple, device: torch.device) -> torch.Tensor:
    """An output: a new tensor if t is None, else t checked by _tensor (written in place, e.g. inside a CUDA graph capture)."""
    return torch.empty(shape, dtype=dtype, device=device) if t is None else _tensor(t, name, dtype, shape, device)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """The device address of an optional tensor argument (None: NULL)."""
    return None if t is None else t.data_ptr()


def _half_scalar(x) -> float:
    """A scalar scale rounded to fp16, as the reference's at::Half overloads receive it."""
    return float(torch.tensor(float(x), dtype=_HALF))


_workspaces: dict = {}
# A workspace that was handed out is never freed: a captured CUDA graph may still hold its address, and the self-cleaning counters inside
# must not alias reused memory on replay.  Outgrown workspaces are kept alive here.
_retired: list = []


def _workspace(kind: str, device: torch.device, nbytes: int) -> torch.Tensor:
    """The zero-initialised workspace `kind` of `device`, replaced by a larger one when it holds fewer than nbytes bytes; once handed out
    it is owned by the library (self-cleaning counters)."""
    key = (kind, device.index)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        if ws is not None:
            _retired.append(ws)
        with torch.cuda.device(device):
            ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


_GEMM_WORKSPACE_BYTES = lib.qs_gemm_workspace_bytes()


def gemm_workspace(device: torch.device) -> torch.Tensor:
    return _workspace("gemm", device, _GEMM_WORKSPACE_BYTES)


def attention_workspace(device: torch.device, batch: int, num_heads: int, head_dim: int) -> torch.Tensor:
    return _workspace("attn", device, lib.qs_attention_workspace_bytes(batch, num_heads, head_dim))


def set_pdl(enabled: bool) -> bool:
    """Toggle programmatic dependent launch for all subsequently launched kernels; returns the previous setting."""
    return bool(lib.qs_set_pdl(1 if enabled else 0))


# --------------------------------------------------------------------------------------------------
# qgemm_w4a8_per_chn / qgemm_w4a8_per_group / qgemm_w8a8
# --------------------------------------------------------------------------------------------------


def _gemm_common(in_feats, kernel, out_feats, k_div: int):
    _tensor(in_feats, "in_feats", torch.int8); _tensor(kernel, "kernel", torch.int8); _tensor(out_feats, "out_feats", _HALF)
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
                                   a_ssums.data_ptr(), out_feats.data_ptr(), _ptr(_acc_out), M, N, K, ws.data_ptr(), ws.numel())


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
                                     ascales.data_ptr(), out_feats.data_ptr(), _ptr(_acc_out), M, N, K, ws.data_ptr(), ws.numel())


def w8a8_gemm_forward_cuda(in_feats, kernel, wscales, ascales, out_feats, _acc_out=None) -> None:
    """qserve_backend.qgemm_w8a8.w8a8_gemm_forward_cuda (w8a8/w8a8_gemm_cuda.cu:532-577, pybind.cpp:13-17)."""
    M, N, K = _gemm_common(in_feats, kernel, out_feats, 1)
    _require(wscales.dtype == _HALF and ascales.dtype == _HALF, "wscales and ascales must be float16 (w8a8_linear.py:99-101 casts them)")
    if M == 0:
        return
    ws = gemm_workspace(in_feats.device)
    _call(in_feats, lib.qs_w8a8_gemm, in_feats.data_ptr(), kernel.data_ptr(), wscales.data_ptr(), ascales.data_ptr(), out_feats.data_ptr(),
                           _ptr(_acc_out), M, N, K, ws.data_ptr(), ws.numel())


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
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _cuda(t, n)
    _tensor(kv_pointers, "kv_pointers", torch.int64)  # :182
    _require(q.dtype == _HALF and k.dtype == _HALF and v.dtype == _HALF, "single_query_attention: only float16 is supported (fused_attention.cpp:24-30)")
    batch = kv_pointers.size(0)
    nheads, nheads_kv, headdim = q.size(1), k.size(1), k.size(-1)
    _require(k.stride(2) == 1 and k.stride(1) == headdim, "k must have stride(2) == 1 and stride(1) == head_dim")  # :179
    _require(v.stride(2) == 1 and v.stride(1) == headdim, "v must have stride(2) == 1 and stride(1) == head_dim")  # :180
    _require(q.stride(2) == 1 and q.stride(1) == headdim, "q must have stride(2) == 1 and stride(1) == head_dim")
    if length_per_sample_ is not None:
        _tensor(length_per_sample_, "length_per_sample", torch.int32, (batch,))  # :184-189
    if alibi_slopes_ is not None:  # accepted, validated and ignored, exactly like the reference (:192-199, :91)
        _cuda(alibi_slopes_, "alibi_slopes")
        _require(tuple(alibi_slopes_.shape) == (nheads,) and alibi_slopes_.dtype == torch.float32, "alibi_slopes must be float32 [nheads]")
    out = torch.empty((q.size(0), nheads, headdim), dtype=q.dtype, device=q.device)
    ws = attention_workspace(q.device, batch, nheads, headdim)
    _call(q, lib.qs_single_query_attention, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), kv_pointers.data_ptr(),
                                        _ptr(length_per_sample_), out.data_ptr(), batch, nheads, nheads_kv, headdim, kv_pointers.size(-1),
                                        int(memory_max_seqlen), int(tokens_per_block), int(size_per_token), int(timestep), int(rotary_embedding_dim),
                                        float(rotary_base), int(bool(neox_rotary_style)), int(bool(int4_kv_cache)), int(bool(kv_cache_with_zeros)),
                                        ws.data_ptr(), ws.numel())
    return out


def apply_bias_rope_update_kv_cache(qkv, seq_lens, padding_offset, kv_pointers: Optional[torch.Tensor], head_num: int, kv_head_num: int,
                                    seq_len: int, tokens_per_block: int, size_per_token: int, rotary_embedding_dim: int,
                                    rotary_embedding_base: float, rotary_embedding_max_positions: int, neox_rotary_style: bool,
                                    int4_kv_cache: bool, kv_cache_with_zeros: bool) -> None:
    """qserve_backend.fused_attention.apply_bias_rope_update_kv_cache (update_kv_cache.cu:20-108): in-place RoPE on the
    packed qkv [T,(Hq+2Hkv)*D] and per-token-per-head asymmetric quantisation of K/V into the pages."""
    _tensor(qkv, "qkv", _HALF)
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


def _qkv_heads(q, k, v):
    """The layout of the prompt attentions' q [T,Hq,128] and k / v [T,Hkv,128]: fp16, heads as contiguous rows of 128 halfs (strided views of
    the qkv buffer are fine), one token count.  Returns (T, Hq, Hkv).  The device checks are the caller's."""
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        _require(t.dtype == _HALF and t.dim() == 3 and t.size(2) == 128, f"{name} must be float16 [T, H, 128]")
        _require(t.stride(2) == 1 and t.stride(1) == 128, f"{name}: heads must be contiguous rows of 128 halfs")
    _require(k.shape == v.shape and q.size(0) == k.size(0), "q, k, v must cover the same tokens; k and v the same heads")
    return q.size(0), q.size(1), k.size(1)


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q: int, max_seqlen_k: int, dropout_p: float = 0.0,
                           softmax_scale: Optional[float] = None, causal: bool = False, **unsupported) -> torch.Tensor:
    """Drop-in for the ONE way the reference calls flash_attn.flash_attn_varlen_func (llama_w4a8_unpad.py:232-242): causal self-attention over a
    batch of prompts, q [T,Hq,128], k / v [T,Hkv,128] fp16 (strided views of the rotated qkv buffer are fine), the same cu_seqlens for queries
    and keys, no dropout.  Returns fp16 [T,Hq,128].  Anything else raises: this is not a general flash-attention."""
    _cuda(q, "q")
    _require(not unsupported or all(val in (None, False, 0, 0.0, (-1, -1)) for val in unsupported.values()), f"unsupported arguments {sorted(unsupported)}")
    _require(causal and float(dropout_p) == 0.0, "only causal=True, dropout_p=0.0 is implemented")
    T, hq, hkv = _qkv_heads(q, k, v)
    _require(cu_seqlens_q.dtype == torch.int32 and cu_seqlens_q.is_contiguous(), "cu_seqlens must be contiguous int32")
    _require(cu_seqlens_k is cu_seqlens_q or (cu_seqlens_k.shape == cu_seqlens_q.shape and cu_seqlens_k.data_ptr() == cu_seqlens_q.data_ptr())
             or bool(torch.equal(cu_seqlens_k, cu_seqlens_q)), "queries and keys must share cu_seqlens (prompt self-attention)")
    _require(int(max_seqlen_q) == int(max_seqlen_k), "max_seqlen_q and max_seqlen_k must agree")
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
        _call(input, lib.qs_dequant_add_residual_rms_norm_quant, out.data_ptr(), input.data_ptr(), residual.data_ptr(), gamma.data_ptr(), None,
                                                         _half_scalar(scale), float(epsilon), tokens, hidden)


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
        _call(input, lib.qs_invoke_quant_scalar, out.data_ptr(), input.data_ptr(), _half_scalar(scale), tokens, hidden)


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
        _call(input, lib.qs_invoke_quant_scalar, out.data_ptr(), input.data_ptr(), _half_scalar(scale), tokens, hidden)


def invoke_dequant_add_residual(out, input, residual, scale) -> None:
    """fused_kernels.invoke_dequant_add_residual, both overloads (fused.cpp:48-55)."""
    _cuda(input, "input"); _half_only(residual, "invoke_dequant_add_residual")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    if isinstance(scale, torch.Tensor):
        _call(input, lib.qs_invoke_dequant_add_residual, out.data_ptr(), input.data_ptr(), residual.data_ptr(), scale.data_ptr(), 0.0, tokens, hidden)
    else:
        _call(input, lib.qs_invoke_dequant_add_residual, out.data_ptr(), input.data_ptr(), residual.data_ptr(), None, _half_scalar(scale), tokens, hidden)


def invoke_dequant(out, input, scale) -> None:
    """fused_kernels.invoke_dequant (fused.cpp:56, fused_kernels.cu:179-196)."""
    _cuda(input, "input"); _half_only(out, "invoke_dequant")
    if _noop(input):
        return
    tokens, hidden = _rows(input)
    _call(input, lib.qs_invoke_dequant, out.data_ptr(), input.data_ptr(), _half_scalar(scale), tokens, hidden, input.stride(-2), out.stride(-2))


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
                                      _ptr(input_sum), scaling.data_ptr(), float(epsilon), tokens, hidden)


def silu_and_mul_quant(out, input, input_sum: Optional[torch.Tensor], scale) -> None:
    """silu_and_mul(input) followed by invoke_quant[_fuse_sum]; the fp16 activation never leaves the SM."""
    _cuda(input, "input"); _half_only(input, "silu_and_mul_quant")
    if _noop(input):
        return
    d = input.size(-1) // 2
    tokens = input.numel() // input.size(-1)
    _call(input, lib.qs_silu_and_mul_quant, out.data_ptr(), input.data_ptr(), _ptr(input_sum), scale.data_ptr(), tokens, d)


def single_query_attention_quant(q, k, v, kv_pointers, length_per_sample, memory_max_seqlen: int, tokens_per_block: int, size_per_token: int,
                                 timestep: int, rotary_embedding_dim: int, rotary_base: float, int4_kv_cache: bool, kv_cache_with_zeros: bool,
                                 out_q, out_scale, out_sum: Optional[torch.Tensor]) -> None:
    """single_query_attention + invoke_quant[_fuse_sum] in one launch: out_q int8 [B, Hq*D], out_scale / out_sum fp16 [B].
    Bit-identical to the two reference ops run back to back (llama_w4a8_unpad.py:265-283)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _cuda(t, n)
    dev = q.device
    _tensor(kv_pointers, "kv_pointers", torch.int64, device=dev)
    batch = kv_pointers.size(0)
    if batch == 0:
        return
    nheads, nheads_kv, headdim = q.size(1), k.size(1), k.size(-1)
    _require(q.dtype == _HALF and k.dtype == _HALF and v.dtype == _HALF, "q, k, v must be float16")
    _require(q.stride(2) == 1 and q.stride(1) == headdim and k.stride(1) == headdim and v.stride(1) == headdim, "q, k, v: stride(1) must be head_dim")
    _tensor(length_per_sample, "length_per_sample", torch.int32, (batch,), dev)
    _tensor(out_q, "out_q", torch.int8, device=dev)
    _require(out_q.numel() == batch * nheads * headdim, "out_q must be int8 [B, Hq*D]")
    _tensor(out_scale, "out_scale", _HALF, (batch,), dev)
    if out_sum is not None:
        _tensor(out_sum, "out_sum", _HALF, (batch,), dev)
    ws = attention_workspace(dev, batch, nheads, headdim)
    _call(q, lib.qs_single_query_attention_quant, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), kv_pointers.data_ptr(),
                                              length_per_sample.data_ptr(), out_q.data_ptr(), out_scale.data_ptr(), _ptr(out_sum), batch, nheads,
                                              nheads_kv, headdim, kv_pointers.size(-1), int(memory_max_seqlen), int(tokens_per_block), int(size_per_token),
                                              int(timestep), int(rotary_embedding_dim), float(rotary_base), int(bool(int4_kv_cache)),
                                              int(bool(kv_cache_with_zeros)), ws.data_ptr(), ws.numel())


def apply_bias_rope_update_kv_cache_at(qkv, seq_lens, padding_offset, start_pos, kv_pointers: Optional[torch.Tensor], head_num: int,
                                       kv_head_num: int, seq_len: int, tokens_per_block: int, size_per_token: int, rotary_embedding_dim: int,
                                       rotary_embedding_base: float, rotary_embedding_max_positions: int, neox_rotary_style: bool,
                                       int4_kv_cache: bool, kv_cache_with_zeros: bool, tree_mask: Optional[torch.Tensor] = None) -> None:
    """apply_bias_rope_update_kv_cache for prompt CHUNKS that continue sequences whose first start_pos[b] tokens (int32 [B], device) are
    already cached: seq_lens are the chunk lengths, token pos of chunk b is rotated at position start_pos[b] + pos and appended there.
    Appending a prompt in chunks leaves the same bytes as one apply_bias_rope_update_kv_cache call over the whole prompt.

    tree_mask (int32 [T], one ancestor word per row, see tree_decode_attention in multi_token_decode_attention): the rows are draft-tree
    nodes (seq_len <= 16); node i is rotated at position start_pos[b] + depth(i) and stored in slot start_pos[b] + i.  None: the call above."""
    _tensor(qkv, "qkv", _HALF)
    for t, n in ((seq_lens, "seq_lens"), (padding_offset, "padding_offset")):
        _cuda(t, n)
        _require(t.dtype == torch.int32, f"{n} must be int32")
    _tensor(start_pos, "start_pos", torch.int32, (seq_lens.size(0),))
    head_dim = int(rotary_embedding_dim)
    _require(head_dim == 128, "apply_bias_rope_update_kv_cache_at: head_dim must be 128")
    _require(qkv.size(-1) == (head_num + 2 * kv_head_num) * head_dim, "qkv width does not match (head_num + 2*kv_head_num) * head_dim")
    if kv_pointers is not None:
        _tensor(kv_pointers, "kv_pointers", torch.int64)
    fn, mask = lib.qs_apply_bias_rope_update_kv_cache_at, ()
    if tree_mask is not None:
        _tensor(tree_mask, "tree_mask", torch.int32, device=qkv.device)
        _require(tree_mask.numel() == qkv.size(0), "tree_mask must hold one word per draft row")
        _require(1 <= int(seq_len) <= 16, "apply_bias_rope_update_kv_cache_at: a draft tree has at most 16 nodes per sequence (seq_len)")
        fn, mask = lib.qs_apply_bias_rope_update_kv_cache_tree, (tree_mask.data_ptr(),)
    _call(qkv, fn, qkv.data_ptr(), seq_lens.data_ptr(), padding_offset.data_ptr(), start_pos.data_ptr(), *mask, _ptr(kv_pointers), seq_lens.size(0),
          qkv.size(0), 0 if kv_pointers is None else kv_pointers.size(-1), int(head_num), int(kv_head_num), head_dim, int(seq_len), int(tokens_per_block),
          int(size_per_token), int(rotary_embedding_dim), float(rotary_embedding_base), int(rotary_embedding_max_positions),
          int(bool(neox_rotary_style)), int(bool(int4_kv_cache)), int(bool(kv_cache_with_zeros)))


def _paged_prompt(q, k, v, cu_seqlens, max_seqlen, prefix_lens, max_prefix_len, kv_pointers, tokens_per_block, size_per_token, int4_kv_cache):
    """The checks prefix_prefill_attention and multi_token_decode_attention share: q / k / v as _qkv_heads, every tensor on q's CUDA device,
    cu_seqlens int32 [B+1], prefix_lens int32 [B], kv_pointers int64 [B, 2, max_blocks] of 64-token pages covering max_prefix_len + max_seqlen
    tokens, and size_per_token of the KV heads and the cache type.  Returns (B, T, Hq, Hkv).  The callers bound max_seqlen."""
    _cuda(q, "q")
    dev = q.device
    for t, n in ((k, "k"), (v, "v")):
        _require(t.device == dev, f"{n} is on {t.device}, q on {dev}")
    T, hq, hkv = _qkv_heads(q, k, v)
    batch = _tensor(cu_seqlens, "cu_seqlens", torch.int32, (None,), dev).size(0) - 1
    _tensor(prefix_lens, "prefix_lens", torch.int32, (batch,), dev)
    _tensor(kv_pointers, "kv_pointers", torch.int64, (batch, 2, None), dev)
    _require(int(tokens_per_block) == 64, "tokens_per_block must be 64")
    _require(hq % hkv == 0, "num_heads must be a multiple of num_kv_heads")
    _require(int(size_per_token) == hkv * 128 * (4 if int4_kv_cache else 8) // 8, "size_per_token does not match the kv heads and the cache type")
    _require(int(max_prefix_len) >= 0, "negative max_prefix_len")
    _require(int(max_prefix_len) + int(max_seqlen) <= kv_pointers.size(-1) * 64, "the page table is too short for max_prefix_len + max_seqlen")
    return batch, T, hq, hkv


def prefix_prefill_attention(q, k, v, cu_seqlens, max_seqlen: int, prefix_lens, max_prefix_len: int, kv_pointers, tokens_per_block: int,
                             size_per_token: int, int4_kv_cache: bool, softmax_scale: Optional[float] = None) -> torch.Tensor:
    """Causal attention of a batch of prompt chunks over their cached prefix.  q [T,Hq,128], k / v [T,Hkv,128] fp16 (strided views of the qkv
    buffer apply_bias_rope_update_kv_cache_at has rotated), cu_seqlens int32 [B+1] chunk offsets, prefix_lens int32 [B] cached tokens,
    kv_pointers int64 [B,2,max_blocks] page addresses (the block table covers the prefix and the chunk).  Query i of sequence b attends to the
    prefix keys dequantised from the ZINT4 / ZINT8 pages and to chunk keys 0..i in fp16.  max_prefix_len bounds prefix_lens (it is not checked
    on the device).  Returns fp16 [T,Hq,128].  Every chunk key is used un-quantised: this is prompt attention, not n decode steps (for those,
    e.g. speculative-decoding verification, use multi_token_decode_attention, which reads the earlier chunk tokens back from the pages)."""
    _require(int(max_seqlen) >= 0, "negative max_seqlen")
    batch, T, hq, hkv = _paged_prompt(q, k, v, cu_seqlens, max_seqlen, prefix_lens, max_prefix_len, kv_pointers, tokens_per_block, size_per_token,
                                      int4_kv_cache)
    out = torch.empty((T, hq, 128), dtype=_HALF, device=q.device)
    if T == 0 or batch == 0:
        return out
    scale = float(softmax_scale) if softmax_scale is not None else 128 ** -0.5
    _call(q, lib.qs_prefix_prefill_attention, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), out.data_ptr(), out.stride(0),
          cu_seqlens.data_ptr(), prefix_lens.data_ptr(), kv_pointers.data_ptr(), batch, T, int(max_seqlen), int(max_prefix_len), kv_pointers.size(-1),
          hq, hkv, 128, int(tokens_per_block), int(size_per_token), int(bool(int4_kv_cache)), scale)
    return out


def multi_token_workspace(device: torch.device, batch: int, num_tokens: int, max_seqlen: int, max_prefix_len: int, num_heads: int,
                          num_kv_heads: int, int4_kv_cache: bool) -> torch.Tensor:
    return _workspace("mtok", device, max(1, lib.qs_multi_token_attention_workspace_bytes(batch, num_tokens, max_seqlen, max_prefix_len, num_heads,
                                                                                         num_kv_heads, int(bool(int4_kv_cache)))))


def multi_token_decode_attention(q, k, v, cu_seqlens, max_seqlen: int, prefix_lens, max_prefix_len: int, kv_pointers, tokens_per_block: int,
                                 size_per_token: int, int4_kv_cache: bool, softmax_scale: Optional[float] = None,
                                 tree_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decode attention of n_b <= 16 draft tokens per sequence in one launch (speculative-decoding verification).  Arguments as for
    prefix_prefill_attention: q [T,Hq,128], k / v [T,Hkv,128] fp16, the draft rows apply_bias_rope_update_kv_cache_at has rotated and appended
    at positions prefix_lens[b] .. prefix_lens[b] + n_b - 1; cu_seqlens int32 [B+1]; prefix_lens int32 [B]; kv_pointers int64 [B,2,max_blocks].

    Query token i of sequence b is computed as single_query_attention computes that decode step: it attends to the cache positions
    0 .. prefix_lens[b] + i - 1 dequantised from the ZINT4 / ZINT8 pages (the earlier draft tokens included, read back quantised) and to its own
    key and value un-quantised.  So a greedy verify gives the numbers of n sequential decode steps up to the fp32 summation order.  This differs
    from prefix_prefill_attention, which uses every chunk key un-quantised.  1 <= max_seqlen <= 16; max_prefix_len bounds prefix_lens (it is
    not checked on the device).  The default softmax scale is the decode kernel's 1/sqrt(128).  Returns fp16 [T,Hq,128].

    tree_mask (int32 [T], one word per draft row): the draft tokens of a sequence are the nodes 0 .. n_b - 1 of a token tree in topological
    order, appended by apply_bias_rope_update_kv_cache_at(..., tree_mask=tree_mask); bit j of node i's word means "node j is an ancestor of
    node i" (bits >= i are ignored; a chain is (1 << i) - 1).  Node i attends to the cache positions 0 .. prefix_lens[b] - 1, to the slots of
    its ancestors and to its own key / value, i.e. it gets the decode step at position prefix_lens[b] + depth(i) after sequential decoding
    along its root path.  The mask contents are not validated (that would need a host synchronisation); whatever they hold, the kernels never
    read a slot >= prefix_lens[b] + i for node i.  A chain mask gives this function's result without a mask bit for bit.  None: no mask."""
    _require(1 <= int(max_seqlen) <= 16, "max_seqlen must be 1 .. 16 draft tokens")
    batch, T, hq, hkv = _paged_prompt(q, k, v, cu_seqlens, max_seqlen, prefix_lens, max_prefix_len, kv_pointers, tokens_per_block, size_per_token,
                                      int4_kv_cache)
    out = torch.empty((T, hq, 128), dtype=_HALF, device=q.device)
    if T == 0 or batch == 0:
        return out
    fn, mask = lib.qs_multi_token_decode_attention, ()
    if tree_mask is not None:
        _tensor(tree_mask, "tree_mask", torch.int32, device=q.device)
        _require(tree_mask.numel() == T, "tree_mask must hold one word per draft row")
        fn, mask = lib.qs_tree_decode_attention, (tree_mask.data_ptr(),)
    ws = multi_token_workspace(q.device, batch, T, int(max_seqlen), int(max_prefix_len), hq, hkv, int4_kv_cache)
    scale = float(softmax_scale) if softmax_scale is not None else 0.0
    _call(q, fn, q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(0), k.stride(0), v.stride(0), out.data_ptr(), out.stride(0), cu_seqlens.data_ptr(),
          prefix_lens.data_ptr(), *mask, kv_pointers.data_ptr(), batch, T, int(max_seqlen), int(max_prefix_len), kv_pointers.size(-1), hq, hkv, 128,
          int(tokens_per_block), int(size_per_token), int(bool(int4_kv_cache)), scale, ws.data_ptr(), ws.numel())
    return out


def tree_accept_greedy(draft_tokens, tree_mask, target_tokens, accept_len: Optional[torch.Tensor] = None, path: Optional[torch.Tensor] = None,
                       bonus: Optional[torch.Tensor] = None):
    """Greedy acceptance of a draft tree, one warp per sequence and no host synchronisation.  draft_tokens int64 [B, n] (node 0 is the root:
    the token emitted by the previous step; padding nodes carry -1, which never matches), tree_mask int32 [B, n] (ancestor words as for
    multi_token_decode_attention), target_tokens int64 [B, n] (the target model's greedy token after each node), n <= 16.  From the root the
    walk moves to the lowest-index child c of the current node with draft[c] == target[current] until no child matches.  Returns
    (accept_len int32 [B] >= 1, path int32 [B, n] with path[:, 0] = 0 and -1 past accept_len, bonus int64 [B] = target[last accepted node]);
    the optional out tensors are written in place (CUDA-graph capture)."""
    B, n = _tensor(draft_tokens, "draft_tokens", torch.int64, (None, None)).shape
    dev = draft_tokens.device
    _tensor(tree_mask, "tree_mask", torch.int32, (B, n), dev)
    _tensor(target_tokens, "target_tokens", torch.int64, (B, n), dev)
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    accept_len = _out(accept_len, "accept_len", torch.int32, (B,), dev)
    path = _out(path, "path", torch.int32, (B, n), dev)
    bonus = _out(bonus, "bonus", torch.int64, (B,), dev)
    if B:
        _call(draft_tokens, lib.qs_tree_accept_greedy, draft_tokens.data_ptr(), tree_mask.data_ptr(), target_tokens.data_ptr(), accept_len.data_ptr(),
              path.data_ptr(), bonus.data_ptr(), B, n)
    return accept_len, path, bonus


def kv_cache_compact(kv_pointers, start_pos, path, accept_len, num_kv_heads: int, tokens_per_block: int, size_per_token: int,
                     int4_kv_cache: bool) -> None:
    """Move the accepted path of a draft tree into consecutive cache slots, for every layer in one launch: for k < accept_len[b] the slot
    bytes (codes, scale, zero; K and V; every KV head) of start_pos[b] + path[b, k] are copied to slot start_pos[b] + k.  Node path[b, k] has
    depth k and was rotated at that position, so afterwards slots start_pos[b] .. start_pos[b] + accept_len[b] - 1 hold exactly what sequential
    decoding of the accepted tokens writes; the engine then advances the context by accept_len.  kv_pointers int64 [L, B, 2, max_blocks] or
    [B, 2, max_blocks]; start_pos int32 [B]; path int32 [B, n] and accept_len int32 [B] as tree_accept_greedy returns them (n <= 16).
    The page table must cover start_pos[b] + n slots (not checked on the device: slots outside the table are left alone)."""
    _tensor(kv_pointers, "kv_pointers", torch.int64)
    _require(kv_pointers.dim() in (3, 4) and kv_pointers.size(-2) == 2, "kv_pointers must be int64 [L, B, 2, max_blocks] or [B, 2, max_blocks]")
    L = kv_pointers.size(0) if kv_pointers.dim() == 4 else 1
    B = kv_pointers.size(-3)
    dev = kv_pointers.device
    _tensor(start_pos, "start_pos", torch.int32, (B,), dev)
    n = _tensor(path, "path", torch.int32, (B, None), dev).size(1)
    _tensor(accept_len, "accept_len", torch.int32, (B,), dev)
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    _require(int(tokens_per_block) == 64, "tokens_per_block must be 64")
    _require(int(num_kv_heads) >= 1 and int(size_per_token) == int(num_kv_heads) * 128 * (4 if int4_kv_cache else 8) // 8,
             "size_per_token does not match the kv heads and the cache type")
    _require(n <= kv_pointers.size(-1) * 64, "the page table is too short for the draft nodes")
    if B == 0 or L == 0:
        return
    _call(kv_pointers, lib.qs_kv_cache_compact, kv_pointers.data_ptr(), start_pos.data_ptr(), path.data_ptr(), accept_len.data_ptr(), L, B, n,
          kv_pointers.size(-1), int(num_kv_heads), int(tokens_per_block), int(size_per_token), int(bool(int4_kv_cache)))


def fork_pairs(parents, children, batch: int):
    """The (parent, child) rows of a fork as two lists of ints, checked on the host: in [0, batch), equally long, no child twice, no row both
    parent and child (its pages would be read and written by the same copy)."""
    parents, children = [int(x) for x in parents], [int(x) for x in children]
    _require(len(parents) == len(children), f"{len(parents)} parents but {len(children)} children")
    _require(all(0 <= r < batch for r in parents + children), f"parent and child rows must lie in [0, {batch})")
    _require(len(set(children)) == len(children), "a child row appears twice")
    both = set(parents) & set(children)
    _require(not both, f"rows {sorted(both)}: a parent row is also a child")
    return parents, children


def kv_cache_fork(kv_pointers, parents, children, lens, num_kv_heads: int, tokens_per_block: int, size_per_token: int, int4_kv_cache: bool) -> None:
    """Copy-on-write fork of cached prompts (SamplingParams.n / best_of), every layer in one launch: for each pair (parents[p], children[p]) with
    P = lens[parents[p]] cached tokens, the bytes of slots 0 .. P % 64 - 1 (codes, scale, zero; K and V; every KV head) of the parent's page at
    block P // 64 are copied into the child's page at the same block index (nothing when P % 64 == 0).  The caller points the child's entries
    for blocks 0 .. P // 64 - 1 at the parent's pages first; the child's entry at block P // 64 must be its own page.  kv_pointers int64
    [L, B, 2, max_blocks] or [B, 2, max_blocks]; parents / children: host sequences of row indices (checked here: in [0, B), equally long, no
    child twice, no row both parent and child); lens int32 [B] on the device (trusted)."""
    _require(kv_pointers.dim() in (3, 4) and kv_pointers.size(-2) == 2, "kv_pointers must be int64 [L, B, 2, max_blocks] or [B, 2, max_blocks]")
    L = kv_pointers.size(0) if kv_pointers.dim() == 4 else 1
    B = kv_pointers.size(-3)
    parents, children = fork_pairs(parents, children, B)
    _tensor(kv_pointers, "kv_pointers", torch.int64)
    dev = kv_pointers.device
    _tensor(lens, "lens", torch.int32, (B,), dev)
    _require(int(tokens_per_block) == 64, "tokens_per_block must be 64")
    _require(int(num_kv_heads) >= 1 and int(size_per_token) == int(num_kv_heads) * 128 * (4 if int4_kv_cache else 8) // 8,
             "size_per_token does not match the kv heads and the cache type")
    if not parents or L == 0:
        return
    rows = torch.tensor(parents + children, dtype=torch.int32, device=dev)
    _call(kv_pointers, lib.qs_kv_cache_fork, kv_pointers.data_ptr(), rows.data_ptr(), rows[len(parents):].data_ptr(), lens.data_ptr(), L, B, len(parents),
          kv_pointers.size(-1), int(num_kv_heads), int(tokens_per_block), int(size_per_token), int(bool(int4_kv_cache)))


def _row_vec(v, n: int, dev, dt, name: str, ok, what: str) -> torch.Tensor:
    """A per-row parameter as a device tensor: a scalar broadcasts (and is checked on the host); a tensor is used as given (its values are
    trusted: checking them would synchronise with the device)."""
    if isinstance(v, torch.Tensor):
        return _tensor(v, name, dt, (n,), dev)
    _require(ok(v), f"{name}={v}: {what}")
    return torch.full((n,), v, dtype=dt, device=dev)


def _row_params(n: int, dev, temperature, top_k, top_p, offsets):
    """Per-row sampling parameters as device tensors (see _row_vec)."""
    def vec(v, dt, name, ok, what):
        return _row_vec(v, n, dev, dt, name, ok, what)
    T = vec(temperature, torch.float32, "temperature", lambda v: float(v) >= 0, "must be >= 0")
    K = vec(top_k, torch.int32, "top_k", lambda v: int(v) == -1 or int(v) >= 1, "must be -1 (off) or >= 1")
    P = vec(top_p, torch.float32, "top_p", lambda v: 0 < float(v) <= 1, "must lie in (0, 1]")
    _tensor(offsets, "offsets", torch.int64, (n,), dev)
    return T, K, P


def _logit_rows(logits) -> tuple:
    rows, V = _tensor(logits, "logits", _HALF, (None, None)).shape
    _require(V % 8 == 0 and 8 <= V <= 196608, f"vocab={V}: a multiple of 8 up to 196608")
    return rows, V


def _seed(seed) -> int:
    _require(0 <= int(seed) < (1 << 64), "seed must be an unsigned 64-bit integer")
    return int(seed)


def sample_rows(logits, temperature, top_k, top_p, seed: int, offsets, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Temperature / top-p / top-k sampling, one token per row of fp16 logits [rows, V] in one launch: the GPU work of the reference's
    `Sampler.forward` (qserve/modeling/layers/sampler.py:24-93).  temperature (fp32), top_k (int32, -1 disables) and top_p (fp32) are
    per-row tensors or scalars; seed is a uint64; offsets int64 [rows] (device) is read and advanced by one per call, so CUDA-graph
    replays draw fresh numbers.  Greedy rows (T < 1e-5 or top_p < 1e-8) return exactly argmax_rows.  Otherwise the kept set is
    {z >= max(tau_p, tau_k)} of z = x / T: what TopPLogitsWarper then TopKLogitsWarper keep, stated independently of tie order, and the
    token is the inverse CDF of the kept softmax at the Philox draw u (see include/qserve_b200.h).  Differences from the reference: the
    reference divides by T and runs softmax().cumsum() over the row in fp16 and draws with torch's RNG, so the distribution agrees up to its
    fp16 rounding but the same seed does not give the same tokens.  V % 8 == 0, V <= 196608.  Returns out int64 [rows]."""
    rows, V = _logit_rows(logits)
    dev = logits.device
    T, K, P = _row_params(rows, dev, temperature, top_k, top_p, offsets)
    out = _out(out, "out", torch.int64, (rows,), dev)
    if rows:
        _call(logits, lib.qs_sample_rows, out.data_ptr(), logits.data_ptr(), T.data_ptr(), K.data_ptr(), P.data_ptr(), _seed(seed), offsets.data_ptr(),
              rows, V)
    return out


def tree_accept_sampling(draft_tokens, tree_mask, logits, temperature, top_k, top_p, seed: int, offsets, draft_probs: Optional[torch.Tensor] = None,
                         accept_len: Optional[torch.Tensor] = None, path: Optional[torch.Tensor] = None, bonus: Optional[torch.Tensor] = None):
    """Sampled acceptance of a draft tree that keeps the target distribution exactly (SpecInfer multi-step speculative sampling; for a chain,
    Leviathan / Chen rejection sampling): the counterpart of tree_accept_greedy with the same draft_tokens int64 [B, n], tree_mask int32
    [B, n] and outputs.  logits fp16 [B, n, V] are the verify logits; temperature / top_k / top_p per sequence as for sample_rows; offsets
    int64 [B] advanced by one; draft_probs fp32 [B, n, V] or None: row c is the distribution q_c node c's token was drawn from (None: one-hot
    at the draft, for deterministic drafters such as Medusa / EAGLE top-k candidates or greedy draft models; i.i.d. siblings pass the same q,
    siblings drawn without replacement the renormalised q each came from).  From the root with p = the warped logits of node 0, child c with
    token d is accepted iff u_c q_c(d) < p(d) (u_c: Philox draw j = c); rejection sets p <- max(p - q_c, 0) renormalised (kept if the mass is
    0); with no child accepted the bonus is drawn from p with draw j = 0.  Greedy rows (T < 1e-5 or top_p < 1e-8) give exactly
    tree_accept_greedy(draft, mask, argmax_rows(logits)).  Returns (accept_len int32 [B], path int32 [B, n], bonus int64 [B]), ready for
    kv_cache_compact; the optional out tensors are written in place (CUDA-graph capture)."""
    B, n = _tensor(draft_tokens, "draft_tokens", torch.int64, (None, None)).shape
    dev = draft_tokens.device
    _tensor(tree_mask, "tree_mask", torch.int32, (B, n), dev)
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    V = _tensor(logits, "logits", _HALF, (B, n, None), dev).size(2)
    _require(V % 8 == 0 and 8 <= V <= 196608, f"vocab={V}: a multiple of 8 up to 196608")
    if draft_probs is not None:
        _tensor(draft_probs, "draft_probs", torch.float32, (B, n, V), dev)
    T, K, P = _row_params(B, dev, temperature, top_k, top_p, offsets)
    accept_len = _out(accept_len, "accept_len", torch.int32, (B,), dev)
    path = _out(path, "path", torch.int32, (B, n), dev)
    bonus = _out(bonus, "bonus", torch.int64, (B,), dev)
    if B:
        _call(draft_tokens, lib.qs_tree_accept_sampling, draft_tokens.data_ptr(), tree_mask.data_ptr(), logits.data_ptr(), _ptr(draft_probs), T.data_ptr(),
              K.data_ptr(), P.data_ptr(), _seed(seed), offsets.data_ptr(), accept_len.data_ptr(), path.data_ptr(), bonus.data_ptr(), B, n, V)
    return accept_len, path, bonus


MAX_PENALTY_HISTORY = 32768  # history tokens per row apply_penalties supports
MAX_TOP_LOGPROBS = 20


def apply_penalties(logits, history, prompt_lens, seq_lens, repetition, presence, frequency) -> torch.Tensor:
    """Repetition / presence / frequency penalties (SamplingParams.repetition_penalty / presence_penalty / frequency_penalty, vLLM's
    semantics) applied in place to fp16 logits [rows, V] before sample_rows / argmax_rows; returns logits.  history int64 [rows, H] holds
    the prompt at [0, prompt_lens[r]) and the generated tokens at [prompt_lens[r], seq_lens[r]) (prompt_lens / seq_lens int32 [rows], clamped
    to 0 <= prompt_lens <= seq_lens <= H on the device; -1 and other out-of-range ids are ignored), H <= 32768.  repetition (in (0, 2]),
    presence and frequency (in [-2, 2]) are fp32 per-row tensors (trusted) or scalars (checked).  For each token t of the history, with c its
    count among the generated tokens, in fp32: x = x / rep if x > 0 else x * rep (rep != 1); if c > 0: x = (x - frequency * c) - presence;
    one rounding to fp16.  Only history tokens whose value changes are written: neutral rows (1, 0, 0) and NaN logits stay as they are, and
    the call is bitwise deterministic.  See include/qserve_b200.h."""
    rows, V = _logit_rows(logits)
    dev = logits.device
    H = _tensor(history, "history", torch.int64, (rows, None), dev).size(1)
    _require(H <= MAX_PENALTY_HISTORY, f"history of {H} tokens per row: at most {MAX_PENALTY_HISTORY}")
    _tensor(prompt_lens, "prompt_lens", torch.int32, (rows,), dev)
    _tensor(seq_lens, "seq_lens", torch.int32, (rows,), dev)
    R = _row_vec(repetition, rows, dev, torch.float32, "repetition", lambda v: 0 < float(v) <= 2, "must lie in (0, 2]")
    P = _row_vec(presence, rows, dev, torch.float32, "presence", lambda v: -2 <= float(v) <= 2, "must lie in [-2, 2]")
    F = _row_vec(frequency, rows, dev, torch.float32, "frequency", lambda v: -2 <= float(v) <= 2, "must lie in [-2, 2]")
    if rows and H:
        _call(logits, lib.qs_apply_penalties, logits.data_ptr(), history.data_ptr(), prompt_lens.data_ptr(), seq_lens.data_ptr(), R.data_ptr(),
              P.data_ptr(), F.data_ptr(), rows, V, H)
    return logits


def logprobs_rows(logits, tokens, n: int, logprob: Optional[torch.Tensor] = None, top_ids: Optional[torch.Tensor] = None,
                  top_logprobs: Optional[torch.Tensor] = None):
    """Log-probabilities for SamplingParams.logprobs / prompt_logprobs in one launch: for fp16 logits [rows, V] and tokens int64 [rows] (the
    sampled token, or the next prompt token), returns (logprob fp32 [rows], top_ids int64 [rows, n], top_logprobs fp32 [rows, n]) with
    0 <= n <= 20, the top tokens ordered by logit descending, ties by ascending index.  The distribution is the row's softmax at T = 1 with the
    sampler's conventions (NaN and -inf weigh 0, +inf logits share the mass); pass the penalised logits to get the distribution before the
    temperature / top-k / top-p warpers.  A row without weight gives NaN and top_ids -1; an out-of-range token gives NaN; with fewer than n
    non-NaN logits the remaining slots are -1 / -inf.  The optional out tensors are written in place (CUDA-graph capture).  Deterministic."""
    rows, V = _logit_rows(logits)
    dev = logits.device
    n = int(n)
    _require(0 <= n <= MAX_TOP_LOGPROBS, f"n={n}: 0 .. {MAX_TOP_LOGPROBS} top log-probabilities")
    _tensor(tokens, "tokens", torch.int64, (rows,), dev)
    logprob = _out(logprob, "logprob", torch.float32, (rows,), dev)
    top_ids = _out(top_ids, "top_ids", torch.int64, (rows, n), dev)
    top_logprobs = _out(top_logprobs, "top_logprobs", torch.float32, (rows, n), dev)
    if rows:
        _call(logits, lib.qs_logprobs_rows, logprob.data_ptr(), _ptr(top_ids if n else None), _ptr(top_logprobs if n else None),
              logits.data_ptr(), tokens.data_ptr(), rows, V, n)
    return logprob, top_ids, top_logprobs


def apply_penalties_tree(logits, draft_tokens, tree_mask, history, prompt_lens, seq_lens, repetition, presence, frequency) -> torch.Tensor:
    """apply_penalties on every node row of a draft tree, in place on the verify logits fp16 [B, n, V] before greedy or sampled acceptance;
    returns logits.  draft_tokens int64 [B, n] and tree_mask int32 [B, n] as ngram_propose returns them (n <= 16).  Row b's history follows
    the generation loop: h[0 .. L) with L = seq_lens[b], h[L - 1] the root (node 0).  Node i's row is, bit for bit, what apply_penalties
    writes for it given the expanded history h[0 .. L), the tokens of node i's ancestors j >= 1 in index order, node i's own token (i >= 1),
    with the row's prompt_lens and parameters; the expanded history is not clipped at H.  So node i's row is the distribution the sequential
    step at that position samples from, and greedy or sampled acceptance stays exact under penalties.  Other arguments and rules as
    apply_penalties (history int64 [B, H], H <= 32768).  See include/qserve_b200.h."""
    B, n = _tensor(draft_tokens, "draft_tokens", torch.int64, (None, None)).shape
    dev = draft_tokens.device
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    _tensor(tree_mask, "tree_mask", torch.int32, (B, n), dev)
    V = _tensor(logits, "logits", _HALF, (B, n, None), dev).size(2)
    _require(V % 8 == 0 and 8 <= V <= 196608, f"vocab={V}: a multiple of 8 up to 196608")
    H = _tensor(history, "history", torch.int64, (B, None), dev).size(1)
    _require(H <= MAX_PENALTY_HISTORY, f"history of {H} tokens per row: at most {MAX_PENALTY_HISTORY}")
    _tensor(prompt_lens, "prompt_lens", torch.int32, (B,), dev)
    _tensor(seq_lens, "seq_lens", torch.int32, (B,), dev)
    R = _row_vec(repetition, B, dev, torch.float32, "repetition", lambda v: 0 < float(v) <= 2, "must lie in (0, 2]")
    P = _row_vec(presence, B, dev, torch.float32, "presence", lambda v: -2 <= float(v) <= 2, "must lie in [-2, 2]")
    F = _row_vec(frequency, B, dev, torch.float32, "frequency", lambda v: -2 <= float(v) <= 2, "must lie in [-2, 2]")
    if B:
        _call(logits, lib.qs_apply_penalties_tree, logits.data_ptr(), draft_tokens.data_ptr(), tree_mask.data_ptr(), history.data_ptr(),
              prompt_lens.data_ptr(), seq_lens.data_ptr(), R.data_ptr(), P.data_ptr(), F.data_ptr(), B, n, V, H)
    return logits


def logprobs_accepted(logits, draft_tokens, path, accept_len, bonus, seq_lens, finished, n_top: int, logprob, top_ids: Optional[torch.Tensor] = None,
                      top_logprobs: Optional[torch.Tensor] = None) -> None:
    """Log-probabilities of the tokens a speculative step emits, in history columns, in place and before spec_commit commits them.  For every
    unfinished row (finished int32 [B] == 0) with acc = accept_len[b] clamped to [1, n] as spec_commit clamps it: emitted token k < acc
    (draft_tokens[b, path[b, k + 1]] for k < acc - 1, else bonus[b]) is scored by node row path[b, k] of logits fp16 [B, n, V] with exactly
    the logprobs_rows arithmetic and written at column seq_lens[b] + k (seq_lens int32 [B] before the commit: where spec_commit puts the
    token) of logprob fp32 [B, W] and, for 1 <= n_top <= 20, top_ids int64 / top_logprobs fp32 [B, W, n_top].  Columns >= W are dropped;
    finished rows and tokens past acc are not written.  After the commit, column c holds the entry of history token c for
    prompt_lens[b] <= c < seq_lens[b]; entries of tokens the commit cut are unspecified.  A plain step passes n = 1, path = 0, accept_len = 1
    and bonus = its token.  See include/qserve_b200.h."""
    B, n = _tensor(draft_tokens, "draft_tokens", torch.int64, (None, None)).shape
    dev = draft_tokens.device
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    n_top = int(n_top)
    _require(0 <= n_top <= MAX_TOP_LOGPROBS, f"n_top={n_top}: 0 .. {MAX_TOP_LOGPROBS} top log-probabilities")
    V = _tensor(logits, "logits", _HALF, (B, n, None), dev).size(2)
    _require(V % 8 == 0 and 8 <= V <= 196608, f"vocab={V}: a multiple of 8 up to 196608")
    _tensor(path, "path", torch.int32, (B, n), dev)
    for t, nm, dt in ((accept_len, "accept_len", torch.int32), (bonus, "bonus", torch.int64), (seq_lens, "seq_lens", torch.int32),
                      (finished, "finished", torch.int32)):
        _tensor(t, nm, dt, (B,), dev)
    W = _tensor(logprob, "logprob", torch.float32, (B, None), dev).size(1)
    _require(W >= 1, "logprob must have at least one column")
    if n_top:
        _require(top_ids is not None and top_logprobs is not None, f"n_top={n_top} needs top_ids and top_logprobs")
        _tensor(top_ids, "top_ids", torch.int64, (B, W, n_top), dev)
        _tensor(top_logprobs, "top_logprobs", torch.float32, (B, W, n_top), dev)
    if B:
        _call(logits, lib.qs_logprobs_accepted, logprob.data_ptr(), _ptr(top_ids if n_top else None), _ptr(top_logprobs if n_top else None),
              logits.data_ptr(), draft_tokens.data_ptr(), path.data_ptr(), accept_len.data_ptr(), bonus.data_ptr(), seq_lens.data_ptr(),
              finished.data_ptr(), B, n, V, n_top, W)


MAX_DRAFT_NGRAM = 8
MAX_DRAFT_BRANCHES = 8


def ngram_propose(history, seq_lens, num_nodes: int, n_min: int = 1, n_max: int = 4, branches: int = 1, tokens: Optional[torch.Tensor] = None,
                  tree_mask: Optional[torch.Tensor] = None):
    """Prompt-lookup draft trees (n-gram drafting) from each row's own token history, one CTA per row and no host synchronisation.
    history int64 [B, H] (H <= 32768), seq_lens int32 [B] = L (clamped to [0, H] on the device); the last token h[L - 1] is the root.  For
    every end position j <= L - 2, m(j) is the longest g <= min(n_max, j + 1) with h[j - g + 1 .. j] == h[L - g .. L - 1] (ids < 0 never
    match); the j with m(j) >= n_min, ranked by (m, j) descending, give up to `branches` continuations h[j + 1 .. min(j + n - 1, L - 1)],
    inserted in rank order into a trie below the root until num_nodes = n nodes exist.  Returns (tokens int64 [B, n], tree_mask int32 [B, n])
    ready for verify_forward / tree_accept_*: node 0 is the root (mask 0), padding nodes have token -1 and mask 1.  1 <= n <= 16,
    1 <= n_min <= n_max <= 8, 1 <= branches <= 8.  The optional out tensors are written in place (CUDA-graph capture).  See
    include/qserve_b200.h."""
    n, n_min, n_max, branches = int(num_nodes), int(n_min), int(n_max), int(branches)
    _require(1 <= n <= 16, f"num_nodes={n}: a draft tree has 1 .. 16 nodes")
    _require(1 <= n_min <= n_max <= MAX_DRAFT_NGRAM, f"n_min={n_min}, n_max={n_max}: need 1 <= n_min <= n_max <= {MAX_DRAFT_NGRAM}")
    _require(1 <= branches <= MAX_DRAFT_BRANCHES, f"branches={branches}: 1 .. {MAX_DRAFT_BRANCHES}")
    B, H = _tensor(history, "history", torch.int64, (None, None)).shape
    _require(1 <= H <= MAX_PENALTY_HISTORY, f"history of {H} tokens per row: 1 .. {MAX_PENALTY_HISTORY}")
    dev = history.device
    _tensor(seq_lens, "seq_lens", torch.int32, (B,), dev)
    tokens = _out(tokens, "tokens", torch.int64, (B, n), dev)
    tree_mask = _out(tree_mask, "tree_mask", torch.int32, (B, n), dev)
    if B:
        _call(history, lib.qs_ngram_propose, history.data_ptr(), seq_lens.data_ptr(), tokens.data_ptr(), tree_mask.data_ptr(), B, H, n, n_min, n_max,
              branches)
    return tokens, tree_mask


MAX_STOP_TOKENS = 8  # stop tokens per row besides eos


def spec_commit(draft_tokens, path, accept_len, bonus, history, seq_lens, prompt_lens, budget, eos, finished, start_pos,
                context_lens: Optional[torch.Tensor] = None, roots: Optional[torch.Tensor] = None, stop_ids: Optional[torch.Tensor] = None) -> None:
    """Advance every unfinished row by what its speculative step accepted, in place and without host synchronisation: the tokens
    draft_tokens[b, path[b, 1 .. acc - 1]] and bonus[b] (acc = accept_len[b]; draft_tokens int64 [B, n], path int32 [B, n], accept_len int32 [B]
    and bonus int64 [B] as tree_accept_greedy / tree_accept_sampling return them) are cut after the first eos[b] (int64 [B], -1: none), then
    to budget[b] - (L - prompt_lens[b]) tokens (int32 [B]), and appended to history int64 [B, H] at L = seq_lens[b] (columns >= H dropped);
    seq_lens advances by the count.  start_pos (int32 [B]) = L - 1, the optional context_lens (int32 [B]) = L and roots (int64 [B]) = the last
    token: what the next verify step (start_pos) or decode step (context_lens, tokens = roots) reads.  finished int32 [B] is set when a row
    appends eos or reaches its budget; finished rows are left untouched.  A plain decode step commits with n = 1, path = 0, accept_len = 1 and
    bonus = its token.  stop_ids int64 [B, S] (S <= 8, -1 pads; SamplingParams.stop_token_ids): any token of {eos[b]} and stop_ids[b] ends
    the row as eos does (appended, cut after, finished; the budget cut still wins), in the qs_spec_commit_stops launch.  See
    include/qserve_b200.h."""
    B, n = _tensor(draft_tokens, "draft_tokens", torch.int64, (None, None)).shape
    _require(1 <= n <= 16, "a draft tree has 1 .. 16 nodes per sequence")
    dev = draft_tokens.device
    H = _tensor(history, "history", torch.int64, (B, None), dev).size(1)
    _require(1 <= H <= MAX_PENALTY_HISTORY, f"history of {H} tokens per row: 1 .. {MAX_PENALTY_HISTORY}")
    _tensor(path, "path", torch.int32, (B, n), dev)
    for t, nm, dt in ((accept_len, "accept_len", torch.int32), (bonus, "bonus", torch.int64), (seq_lens, "seq_lens", torch.int32),
                      (prompt_lens, "prompt_lens", torch.int32), (budget, "budget", torch.int32), (eos, "eos", torch.int64),
                      (finished, "finished", torch.int32), (start_pos, "start_pos", torch.int32)):
        _tensor(t, nm, dt, (B,), dev)
    for t, nm, dt in ((context_lens, "context_lens", torch.int32), (roots, "roots", torch.int64)):
        if t is not None:
            _tensor(t, nm, dt, (B,), dev)
    if stop_ids is not None:
        S = _tensor(stop_ids, "stop_ids", torch.int64, (B, None), dev).size(1)
        _require(S <= MAX_STOP_TOKENS, f"{S} stop tokens per row: at most {MAX_STOP_TOKENS}")
    if not B:
        return
    if stop_ids is None:
        _call(history, lib.qs_spec_commit, draft_tokens.data_ptr(), path.data_ptr(), accept_len.data_ptr(), bonus.data_ptr(), history.data_ptr(),
              seq_lens.data_ptr(), prompt_lens.data_ptr(), budget.data_ptr(), eos.data_ptr(), finished.data_ptr(), start_pos.data_ptr(),
              _ptr(context_lens), _ptr(roots), B, n, H)
    else:
        _call(history, lib.qs_spec_commit_stops, draft_tokens.data_ptr(), path.data_ptr(), accept_len.data_ptr(), bonus.data_ptr(),
              history.data_ptr(), seq_lens.data_ptr(), prompt_lens.data_ptr(), budget.data_ptr(), eos.data_ptr(), _ptr(stop_ids if S else None), S,
              finished.data_ptr(), start_pos.data_ptr(), _ptr(context_lens), _ptr(roots), B, n, H)


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
          ctx.world, ctx.rank, int(phase), weight.data_ptr(), _ptr(input_sum), scaling.data_ptr(), float(epsilon),
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
    _call(input, lib.qs_invoke_quant_given_amax, out.data_ptr(), input.data_ptr(), amax.data_ptr(), _ptr(input_sum),
          scale.data_ptr(), tokens, hidden)


def argmax_rows(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torch.argmax(logits, dim=-1) for fp16 logits [rows, vocab] in one launch (greedy sampling of the decode runner)."""
    _tensor(logits, "logits", _HALF, (None, None))
    if out is None:
        out = torch.empty(logits.size(0), dtype=torch.int64, device=logits.device)
    if logits.size(0) == 0:
        return out
    _call(logits, lib.qs_argmax_rows, out.data_ptr(), logits.data_ptr(), logits.size(0), logits.size(1))
    return out
