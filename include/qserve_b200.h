/* qserve_b200 -- C ABI of the Hopper (sm_90a) W4A8KV4 kernel library.
 *
 * Drop-in boundary for the seven `qserve_backend.*` torch-extension modules of mit-han-lab/qserve
 * (kernels/setup.py:158-245).  The reference has no C ABI: its boundary is pybind11 functions taking
 * torch::Tensor.  Every entry point below is the plain-pointer form of one such function; the reference-side
 * binding (a ten-line pybind11 / ctypes stub per function) is shown in INTEGRATION.md, and the shipped Python
 * package `qserve_backend/` is exactly that stub written with ctypes.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless stated otherwise; `stream` is a cudaStream_t (0 = legacy default);
 *   - fp16 tensors are passed as `const void*` / `void*` to IEEE binary16 data ("half");
 *   - every function returns 0 on success and a negative qs_status otherwise; qs_last_error() returns a
 *     thread-local, NUL-terminated description of the last failure (the Python layer raises RuntimeError with it,
 *     matching the reference's TORCH_CHECK behaviour, fused_attention.cpp:168-199);
 *   - nothing here allocates device memory: outputs and workspaces are caller-owned, so every call is
 *     CUDA-graph capturable; launches go to the caller's stream (the reference GEMMs use the legacy default
 *     stream, gemm_cuda.cu:53 -- using the current stream is a superset);
 *   - there is no CPU fallback: without a CUDA device the launches fail with QS_ERR_CUDA.
 */
#ifndef QSERVE_B200_H_
#define QSERVE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QS_ABI_VERSION 1
#if defined(__GNUC__)
#define QS_API __attribute__((visibility("default")))
#else
#define QS_API
#endif

typedef enum qs_status {
  QS_OK = 0,
  QS_ERR_INVALID = -1,
  QS_ERR_CUDA = -2,
  QS_ERR_WORKSPACE = -3,
  QS_ERR_UNSUPPORTED = -4
} qs_status;

QS_API int qs_abi_version(void);
QS_API const char* qs_last_error(void);
/* Enable (1) / disable (0) programmatic dependent launch for all subsequent launches; returns the previous value.
 * With PDL on (default) every kernel runs `griddepcontrol.launch_dependents` at entry and reads STATIC operands -- weights, weight scales,
 * level-2 parameters, the page-pointer table, length_per_sample -- BEFORE `griddepcontrol.wait`, so that its prologue overlaps the previous
 * kernel.  Those tensors must therefore not be written by a kernel of the same stream inside a chain of back-to-back library calls (update block
 * tables / context lengths from the host, as the reference's ModelRunner does, or behind a non-library kernel).  The controls of this header
 * (qs_set_pdl, qs_gemm_force_*, ...) are process-wide and unsynchronised; qs_last_error() is thread-local.  Host-side caches (kernel
 * attributes, SM count, tensor maps) are keyed by the CURRENT device: make the tensors' device current before calling (the Python mirror does). */
QS_API int qs_set_pdl(int enabled);

/* ---------------------------------------------------------------------------------------------------------
 * qserve_backend.qgemm_w4a8_per_chn.gemm_forward_cuda           kernels/csrc/qgemm/w4a8_per_chn/gemm_cuda.cu:596-652
 *   out[m,n] = half( float(sum_k in[m,k]*q[n,k]) * wscales[n] * ascales[m] - w_szs[n] * a_ssums[m] )
 *   in_feats int8 [M,K]; kernel packed uint4 [N,K/2] in the checkpoint layout (w4a8_linear.py:292-322);
 *   wscales, w_szs fp16 [N]; ascales, a_ssums fp16 [M]; out fp16 [M,N].  N % 128 == 0, K % 128 == 0.
 *   workspace: reserved (split-K partial tiles are exchanged through distributed shared memory inside a thread-block
 *   cluster, no global scratch is needed); pass NULL / 0 or a buffer of qs_gemm_workspace_bytes() bytes.
 *   acc_out (optional, may be NULL): raw INT32 accumulators [M,N] for bit-exact parity checks.
 * --------------------------------------------------------------------------------------------------------- */
QS_API int qs_w4a8_gemm_per_chn(const int8_t* in_feats, const int8_t* kernel, const void* wscales, const void* ascales, const void* w_szs,
                         const void* a_ssums, void* out_feats, int32_t* acc_out, int M, int N, int K, void* workspace,
                         size_t workspace_bytes, void* stream);

/* qserve_backend.qgemm_w4a8_per_group.gemm_forward_cuda         kernels/csrc/qgemm/w4a8_per_group/gemm_cuda.cu:630-702
 *   w8[n,k] = (q[n,k]*s2[k/128,n] + z2[k/128,n]) mod 256 as int8 ;  out = half( float(acc) * (wscales[n]*ascales[m]) )
 *   zeros, scales_i8: int8 [K/128, N] with the checkpoint's per-32-column shuffle (w4a8_linear.py:231-277).          */
QS_API int qs_w4a8_gemm_per_group(const int8_t* in_feats, const int8_t* kernel, const int8_t* zeros, const int8_t* scales_i8,
                           const void* wscales, const void* ascales, void* out_feats, int32_t* acc_out, int M, int N, int K,
                           void* workspace, size_t workspace_bytes, void* stream);

/* qserve_backend.qgemm_w8a8.w8a8_gemm_forward_cuda              kernels/csrc/qgemm/w8a8/w8a8_gemm_cuda.cu:532-577
 *   kernel int8 [N,K] row-major;  out = half( float(acc) * (wscales[n]*ascales[m]) )                                  */
QS_API int qs_w8a8_gemm(const int8_t* in_feats, const int8_t* kernel, const void* wscales, const void* ascales, void* out_feats,
                 int32_t* acc_out, int M, int N, int K, void* workspace, size_t workspace_bytes, void* stream);

QS_API size_t qs_gemm_workspace_bytes(void);
/* test hook: force the cluster split-K factor (1, 2, 4 or 8) of the next GEMM calls; 0 = automatic */
QS_API int qs_gemm_force_split(int split);
/* test / tuning hook: force the tokens-per-tile of the GEMMs (32, 64, 128; 0 = automatic: 32 / 64 / 128 by M);
 * returns the previous value */
QS_API int qs_gemm_force_tile_tokens(int nt);
/* profiling hook: device buffer of 16 x uint64 per CTA receiving %globaltimer stamps of the GEMM phases; NULL disables */
QS_API int qs_gemm_set_profile_buffer(void* dev_buffer);
/* step tracing: u64 buffer [0] = record count (zero it), then `capacity_records` x (kernel_id << 8 | phase, %globaltimer);
 * block 0 of every kernel logs entry (0), dependency resolved (1) and exit (2); NULL disables (tools/step_timeline.py) */
QS_API int qs_set_trace_buffer(void* dev_buffer, unsigned capacity_records);

/* ---------------------------------------------------------------------------------------------------------
 * qserve_backend.fused_attention.single_query_attention         kernels/csrc/fused_attention/fused_attention.cpp:150-240
 *   q fp16 [B,Hq,D] with row stride q_stride (elements); k, v fp16 [B,Hkv,D] with row strides k_stride, v_stride
 *   (stride(1) == D, stride(2) == 1, fused_attention.cpp:179-180); kv_pointers int64 [B,2,max_blocks] absolute
 *   device addresses of the K then V pages (kvCacheUtils.h:84-90); length_per_sample int32 [B] = context length
 *   INCLUDING the token being decoded (may be NULL: then `timestep` is used); out fp16 [B,Hq,D] contiguous.
 *   Side effect: RoPE(k) and v of the new token are quantised and appended at index length-1.
 *   D must be 128, kv_cache_with_zeros must be 1 (ZINT4 / ZINT8), rotary_embedding_dim must equal D.
 *   workspace (optional): qs_attention_workspace_bytes(...) bytes, zero-initialised once; enables context splits.  */
QS_API int qs_single_query_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                              const int64_t* kv_pointers, const int32_t* length_per_sample, void* out, int batch, int num_heads,
                              int num_kv_heads, int head_dim, int max_blocks_per_seq, int memory_max_seqlen, int tokens_per_block,
                              int size_per_token, int timestep, int rotary_embedding_dim, float rotary_base, int neox_rotary_style,
                              int int4_kv_cache, int kv_cache_with_zeros, void* workspace, size_t workspace_bytes, void* stream);
QS_API size_t qs_attention_workspace_bytes(int batch, int num_heads, int head_dim);

/* qserve_backend.fused_attention.apply_bias_rope_update_kv_cache    kernels/csrc/fused_attention/update_kv_cache.cu:20-108
 *   qkv fp16 [T,(Hq+2Hkv)*D]: q and k are rotated IN PLACE (NeoX), K/V quantised per (token, kv head) into the pages.
 *   kv_pointers may be NULL (rotate only).                                                                          */
QS_API int qs_apply_bias_rope_update_kv_cache(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int64_t* kv_pointers,
                                       int batch, int num_tokens, int max_blocks_per_seq, int head_num, int kv_head_num, int head_dim,
                                       int seq_len, int tokens_per_block, int size_per_token, int rotary_embedding_dim,
                                       float rotary_embedding_base, int rotary_embedding_max_positions, int neox_rotary_style,
                                       int int4_kv_cache, int kv_cache_with_zeros, void* stream);

/* Prompt-phase attention: replaces the third-party call flash_attn.flash_attn_varlen_func(q, k, v, cu_seqlens, cu_seqlens, max_seqlen,
 *   max_seqlen, dropout_p=0.0, causal=True) at qserve/modeling/models/llama_w4a8_unpad.py:232-242 (SURVEY.md section 8, row f-3).
 *   q [T,Hq,128], k / v [T,Hkv,128] fp16: strided views of the qkv buffer apply_bias_rope_update_kv_cache has rotated in place (row strides in
 *   halfs, multiples of 8); cu_seqlens int32 [batch+1] shared by queries and keys; out fp16 [T,Hq,128].  Causal, no dropout, GQA by
 *   Hq / Hkv.  fp32 softmax, P rounded to fp16 before the second MMA (as flash-attn does); wgmma, sm_90a only.
 *   max_seqlen must be >= the longest sequence (as for flash-attn: query blocks beyond it are not launched).                          */
QS_API int qs_prefill_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                         int64_t out_stride, const int32_t* cu_seqlens, int batch, int num_tokens, int max_seqlen, int num_heads,
                         int num_kv_heads, int head_dim, float softmax_scale, void* stream);

/* qserve_backend.fused_attention.compute_padding_offsets         kernels/csrc/fused_attention/input_metadata_helper.cu:33-45 */
QS_API int qs_compute_padding_offsets(int32_t* padding_offsets, const int32_t* cu_seqlens, int batch, int max_seqlen, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * qserve_backend.layernorm_ops                                   kernels/csrc/layernorm.cpp:47-72
 * --------------------------------------------------------------------------------------------------------- */
/* rms_norm(out, input, weight, epsilon, use_quant): out fp16 (use_quant=0) or int8 (use_quant=1)                   */
QS_API int qs_rms_norm(void* out, const void* input, const void* weight, float epsilon, int use_quant, int tokens, int hidden, void* stream);
/* rms_norm_general(out int8, input, weight, scaling fp16 [tokens] (out) | [1] (in), epsilon, use_per_token_quant)   */
QS_API int qs_rms_norm_general(int8_t* out, const void* input, const void* weight, void* scaling, float epsilon, int use_per_token_quant,
                        int tokens, int hidden, void* stream);
/* rms_norm_general_fuse_sum(out, input, weight, input_sum fp16 [tokens] (out), scaling, epsilon, use_per_token_quant) */
QS_API int qs_rms_norm_general_fuse_sum(int8_t* out, const void* input, const void* weight, void* input_sum, void* scaling, float epsilon,
                                 int use_per_token_quant, int tokens, int hidden, void* stream);
/* invoke_dequant_add_residual_rms_norm_quant: scale_vec fp16 [tokens] or NULL (then scalar `scale`); residual updated in place */
QS_API int qs_dequant_add_residual_rms_norm_quant(int8_t* out, const int32_t* input, void* residual, const void* gamma, const void* scale_vec,
                                           float scale, float epsilon, int tokens, int hidden, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * qserve_backend.fused_kernels                                   kernels/csrc/fused.cpp:47-70
 * --------------------------------------------------------------------------------------------------------- */
QS_API int qs_invoke_quant(int8_t* out, const void* input, void* scale /* fp16 [tokens] out */, int tokens, int hidden, void* stream);
QS_API int qs_invoke_quant_scalar(int8_t* out, const void* input, float scale, int tokens, int hidden, void* stream);
QS_API int qs_invoke_quant_fuse_sum(int8_t* out, const void* input, void* input_sum, void* scale, int tokens, int hidden, void* stream);
/* Tensor-parallel extension (no reference counterpart: the reference has tp_size = 1 hard-coded, llama_w4a8_unpad.py:115).
 * SURVEY.md 8e parity rule: all ranks quantise their K shard of a token with the same scale.  qs_row_absmax writes the local
 * per-token max |x| (fp32 [tokens]); the caller max-all-reduces it; qs_invoke_quant_given_amax then does the arithmetic of
 * invoke_quant[_fuse_sum] with that amax (input_sum, may be null, is the LOCAL shard's row sum). */
/* Tensor-parallel extension: the sum-all-reduce of a row-parallel GEMM output fused into its consumer (SURVEY.md 5 / 8e: "fused into
 * the GEMM epilogue ... over NVLink").  delta_ptrs[r] = address, valid in THIS process, of rank r's fp16 partial [tokens, hidden] of this
 * phase (peer-mapped symmetric memory); flag_ptrs[r] = rank r's flag pad (16 x u32, zero-initialised, peer-mapped); state = 4 x u32 of
 * local device memory, zero-initialised, owned by the library afterwards.  phase 0 / 1 = o_proj / down_proj (two buffers: see DESIGN.md 6).
 * Semantics: delta = fp16(sum over ranks, fp32, rank order) ; then exactly qs_add_rms_norm_general(out, hidden_out, x, delta, ...).
 * All ranks must issue the same sequence of peer calls. */
QS_API int qs_add_rms_norm_general_peer(int8_t* out, void* hidden_out, const void* x, const void* const* delta_ptrs, void* const* flag_ptrs, void* state,
                                        int world, int rank, int phase, const void* gamma, void* input_sum, void* scaling, float epsilon, int tokens,
                                        int hidden, void* stream);
QS_API int qs_row_absmax(float* amax_out, const void* input, int tokens, int hidden, void* stream);
QS_API int qs_invoke_quant_given_amax(int8_t* out, const void* input, const float* amax, void* input_sum, void* scale, int tokens, int hidden,
                                      void* stream);
QS_API int qs_invoke_dequant_add_residual(void* out, const int32_t* input, const void* residual, const void* scale_vec, float scale, int tokens,
                                   int hidden, void* stream);
QS_API int qs_invoke_dequant(void* out, const int32_t* input, float scale, int tokens, int hidden, int input_stride, int out_stride, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * qserve_backend.activation_ops                                  kernels/csrc/activation.cpp:25-39
 * --------------------------------------------------------------------------------------------------------- */
QS_API int qs_silu_and_mul(void* out, const void* input, int tokens, int d, void* stream);
QS_API int qs_gelu_new(void* out, const void* input, int tokens, int d, void* stream);
QS_API int qs_gelu_fast(void* out, const void* input, int tokens, int d, void* stream);
/* scale_out_vec float [tokens] (out) and tmp float [tokens,d] select the per-token overload; both NULL = scalar scale_out */
QS_API int qs_dequant_silu_and_mul_quant(int8_t* out, const int32_t* input, float scale_gate, float scale_up, float scale_out,
                                  float* scale_out_vec, float* tmp, int tokens, int d, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused extensions (NOT part of the reference surface; bit-identical to the op sequences they replace).
 * Used by qserve_b200/decode.py to cut the launch count of the decode step (SURVEY.md section 8f-2).
 * --------------------------------------------------------------------------------------------------------- */
/* hidden_out = half(x + delta)   [the torch `residual + out_buf` of llama_w4a8_unpad.py:348,360]
 * followed by rms_norm_general[_fuse_sum](out, hidden_out, weight, input_sum | NULL, scaling, epsilon, per_token=1)      */
QS_API int qs_add_rms_norm_general(int8_t* out, void* hidden_out, const void* x, const void* delta, const void* weight, void* input_sum,
                                   void* scaling, float epsilon, int tokens, int hidden, void* stream);
/* single_query_attention followed by invoke_quant[_fuse_sum] of the [B, Hq*D] result: out_q int8 [B, Hq*D], out_scale fp16 [B],
 * out_sum fp16 [B] or NULL.  The fp16 attention row stays in `workspace` (>= qs_attention_workspace_bytes, zero-initialised
 * once, L2 resident); the last CTA of a token to finish quantises it, so the result is bit-identical to the two-op sequence. */
QS_API int qs_single_query_attention_quant(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                                           const int64_t* kv_pointers, const int32_t* length_per_sample, int8_t* out_q, void* out_scale,
                                           void* out_sum, int batch, int num_heads, int num_kv_heads, int head_dim, int max_blocks_per_seq,
                                           int memory_max_seqlen, int tokens_per_block, int size_per_token, int timestep,
                                           int rotary_embedding_dim, float rotary_base, int int4_kv_cache, int kv_cache_with_zeros, void* workspace,
                                           size_t workspace_bytes, void* stream);
/* silu_and_mul(input [tokens, 2d]) followed by invoke_quant[_fuse_sum](out, act, input_sum | NULL, scale)                 */
/* greedy sampling helper for the decode runner: out[r] = index of the first maximum of logits[r, :] (fp16, NaN = maximum), as
 * torch.argmax(logits, -1) does in the reference's sampler */
QS_API int qs_argmax_rows(int64_t* out, const void* logits, int rows, int vocab, void* stream);
QS_API int qs_silu_and_mul_quant(int8_t* out, const void* input, void* input_sum, void* scale, int tokens, int d, void* stream);

/* Prompt chunks over a cached prefix (chunked prefill, prefix reuse, continuing a conversation).
 *
 * qs_apply_bias_rope_update_kv_cache_at: qs_apply_bias_rope_update_kv_cache for a batch of chunks that continue sequences whose first
 *   start_pos[b] tokens (int32 [batch], device) are already in the pages; seq_lens are the CHUNK lengths.  Token pos of chunk b is rotated at
 *   position start_pos[b] + pos and stored in that position's page and slot; the cyclic window uses the total length start_pos[b] + seq_lens[b].
 *   Appending a prompt in several chunks leaves the same bytes in the pages and in the rotated q / k as appending it in one call.      */
QS_API int qs_apply_bias_rope_update_kv_cache_at(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int32_t* start_pos,
                                                 const int64_t* kv_pointers, int batch, int num_tokens, int max_blocks_per_seq, int head_num,
                                                 int kv_head_num, int head_dim, int seq_len, int tokens_per_block, int size_per_token,
                                                 int rotary_embedding_dim, float rotary_embedding_base, int rotary_embedding_max_positions,
                                                 int neox_rotary_style, int int4_kv_cache, int kv_cache_with_zeros, void* stream);
/* qs_prefix_prefill_attention: causal attention of a batch of chunks.  q [T,Hq,128], k / v [T,Hkv,128] fp16: the chunk rows, strided views of
 *   the qkv buffer qs_apply_bias_rope_update_kv_cache_at has rotated (row strides in halfs, multiples of 8); cu_seqlens int32 [batch+1] chunk
 *   offsets; prefix_lens int32 [batch] cached tokens per sequence; kv_pointers int64 [batch,2,max_blocks_per_seq] as for
 *   qs_single_query_attention; out fp16 [T,Hq,128].  Query i of sequence b (position prefix_lens[b] + i) attends to the prefix keys
 *   0 .. prefix_lens[b]-1, dequantised from the ZINT4 / ZINT8 pages exactly as the reference dequantises them, and to the chunk keys 0 .. i as
 *   the un-quantised fp16 k / v.  GQA by Hq / Hkv, head_dim 128, tokens_per_block 64, fp32 softmax, P rounded to fp16 before the PV product;
 *   wgmma, sm_90a only; deterministic.  max_prefix_len is a host bound (like flash-attn's max_seqlen_k): the call checks
 *   max_prefix_len + max_seqlen <= max_blocks_per_seq * 64, and the kernel TRUSTS prefix_lens[b] <= max_prefix_len.  prefix_lens and the page
 *   table are read before the PDL dependency wait (see qs_set_pdl), the page contents after it.                                          */
QS_API int qs_prefix_prefill_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                                       int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens, const int64_t* kv_pointers,
                                       int batch, int num_tokens, int max_seqlen, int max_prefix_len, int max_blocks_per_seq, int num_heads,
                                       int num_kv_heads, int head_dim, int tokens_per_block, int size_per_token, int int4_kv_cache,
                                       float softmax_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QSERVE_B200_H_ */
