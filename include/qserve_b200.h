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

#define QS_ABI_VERSION 2
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

/* Multi-token decode attention (speculative-decoding verification): n_b = cu_seqlens[b+1] - cu_seqlens[b] <= 16 draft tokens per sequence,
 * rotated and appended at positions prefix_lens[b] .. prefix_lens[b] + n_b - 1 by qs_apply_bias_rope_update_kv_cache_at (start_pos =
 * prefix_lens).  Arguments as for qs_prefix_prefill_attention.  Query token i of sequence b is computed as the decode step
 * qs_single_query_attention would compute it at that position: it attends to the cache positions 0 .. prefix_lens[b] + i - 1 dequantised from
 * the ZINT4 / ZINT8 pages (the earlier draft tokens of the step included, read back quantised) and to its own key and value as the un-quantised
 * fp16 rows of k / v; its own cache slot is not read.  A greedy verify therefore reproduces the numbers of sequential decoding up to the fp32
 * summation order.  (qs_prefix_prefill_attention instead uses every chunk key un-quantised.)  softmax_scale <= 0 selects 1/sqrt(128) as the
 * decode kernel computes it.  Restrictions: fp16, head_dim 128, tokens_per_block 64, 1 <= max_seqlen <= 16, max_prefix_len + max_seqlen <=
 * max_blocks_per_seq * 64; n_b = 0 and prefix_lens[b] = 0 are allowed; the kernel TRUSTS prefix_lens[b] <= max_prefix_len.  The page slots
 * from prefix_lens[b] + n_b - 1 on are never read.  workspace: at least qs_multi_token_attention_workspace_bytes(batch, num_tokens,
 * max_seqlen, max_prefix_len, num_heads, num_kv_heads, int4_kv_cache) bytes, zero-filled once and then owned by the library (its split counters clean
 * themselves up, so the call is CUDA-graph capturable and bitwise deterministic).  cu_seqlens, prefix_lens and the page table are read
 * before the PDL dependency wait, q / k / v and the page contents after it.                                                               */
QS_API int qs_multi_token_decode_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                                           void* out, int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens,
                                           const int64_t* kv_pointers, int batch, int num_tokens, int max_seqlen, int max_prefix_len,
                                           int max_blocks_per_seq, int num_heads, int num_kv_heads, int head_dim, int tokens_per_block,
                                           int size_per_token, int int4_kv_cache, float softmax_scale, void* workspace, size_t workspace_bytes,
                                           void* stream);
QS_API size_t qs_multi_token_attention_workspace_bytes(int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads,
                                                       int num_kv_heads, int int4_kv_cache);

/* Tree-structured drafts (speculative decoding with token trees: Medusa, EAGLE, SpecInfer-style candidate trees).
 *
 * Sequence b has prefix_lens[b] = P_b cached tokens and n_b <= 16 draft NODES 0 .. n_b - 1 in topological order (every ancestor has a smaller
 * index than its descendants).  tree_mask int32 [num_tokens], one word per draft row (aligned with the q rows / cu_seqlens): bit j of node i's
 * word means "node j is an ancestor of node i"; bits >= i are ignored.  A chain is mask_i = (1 << i) - 1.  The depth of node i is
 * d_i = popcount(mask_i & ((1 << i) - 1)).  The mask contents are not validated; whatever they hold, no kernel reads a slot >= P_b + i for
 * node i.  tree_mask is read after the PDL dependency wait (a drafter kernel on the same stream may have just produced it).
 *
 * qs_apply_bias_rope_update_kv_cache_tree: qs_apply_bias_rope_update_kv_cache_at (start_pos = P_b, seq_lens = n_b <= 16) for draft nodes:
 *   node i is rotated (q and k) at position P_b + d_i and quantised into cache slot P_b + i.  The cyclic window uses the slot position and
 *   the total length P_b + n_b.
 * qs_tree_decode_attention: qs_multi_token_decode_attention (same arguments, same workspace) with the tree mask: node i attends to the cache
 *   positions 0 .. P_b - 1, to the slots P_b + j of its ancestors j (read back quantised) and to its own key / value un-quantised; so it gets
 *   what qs_single_query_attention computes at position P_b + d_i after sequential decoding along its root path, up to the fp32 summation
 *   order.  With a chain mask the result is bitwise that of qs_multi_token_decode_attention.
 * qs_tree_accept_greedy: draft_tokens int64 [batch, num_nodes] (padding nodes: -1, which never matches), tree_mask int32 [batch, num_nodes],
 *   target_tokens int64 [batch, num_nodes] (the target model's greedy token after each node).  From the root (node 0) the walk moves to the
 *   lowest-index child c of the current node with draft[c] == target[current] (the parent of c is the highest set bit of mask_c below c) until
 *   no child matches.  Outputs accept_len int32 [batch] (>= 1, root included), path int32 [batch, num_nodes] (path[0] = 0, -1 past
 *   accept_len) and bonus int64 [batch] = target[path[accept_len - 1]].  One warp per sequence; inputs read after the dependency wait.
 * qs_kv_cache_compact: for every layer, sequence, K / V and KV head, copies the slot bytes (codes, scale, zero) of P_b + path[k] to slot P_b + k
 *   for k < accept_len[b].  Node path[k] has depth k, so afterwards slots P_b .. P_b + accept_len - 1 are byte-identical to sequential
 *   decoding of the accepted tokens; the engine then advances the context by accept_len and feeds bonus as the next root.  kv_pointers is
 *   [num_layers, batch, 2, max_blocks_per_seq] (num_layers = 1: one layer's table); start_pos int32 [batch].  The page table and start_pos are
 *   read before the dependency wait, path and accept_len after it.  Slots outside the page table are not touched.  num_nodes <= 16.    */
QS_API int qs_apply_bias_rope_update_kv_cache_tree(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int32_t* start_pos,
                                                   const int32_t* tree_mask, const int64_t* kv_pointers, int batch, int num_tokens,
                                                   int max_blocks_per_seq, int head_num, int kv_head_num, int head_dim, int seq_len,
                                                   int tokens_per_block, int size_per_token, int rotary_embedding_dim, float rotary_embedding_base,
                                                   int rotary_embedding_max_positions, int neox_rotary_style, int int4_kv_cache,
                                                   int kv_cache_with_zeros, void* stream);
QS_API int qs_tree_decode_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                                    int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens, const int32_t* tree_mask,
                                    const int64_t* kv_pointers, int batch, int num_tokens, int max_seqlen, int max_prefix_len,
                                    int max_blocks_per_seq, int num_heads, int num_kv_heads, int head_dim, int tokens_per_block,
                                    int size_per_token, int int4_kv_cache, float softmax_scale, void* workspace, size_t workspace_bytes,
                                    void* stream);
QS_API int qs_tree_accept_greedy(const int64_t* draft_tokens, const int32_t* tree_mask, const int64_t* target_tokens, int32_t* accept_len,
                                 int32_t* path, int64_t* bonus, int batch, int num_nodes, void* stream);
QS_API int qs_kv_cache_compact(const int64_t* kv_pointers, const int32_t* start_pos, const int32_t* path, const int32_t* accept_len, int num_layers,
                               int batch, int num_nodes, int max_blocks_per_seq, int num_kv_heads, int tokens_per_block, int size_per_token,
                               int int4_kv_cache, void* stream);

/* qs_kv_cache_fork: copy-on-write fork of cached prompts (SamplingParams.n / best_of: prefill once, decode n rows).  For every layer, K and V
 *   and every pair p, with P = lens[parents[p]] (the parent's cached tokens): copies the bytes of slots 0 .. P % 64 - 1 (codes, scale and
 *   zero of every KV head) of the parent's page at block P / 64 into the child's page at the same block index.  Nothing is copied when
 *   P % 64 == 0 or block P / 64 lies outside the table.  The caller points the child's entries for blocks 0 .. P / 64 - 1 at the parent's
 *   pages (shared, read-only from then on) before the call; the child's entry at block P / 64 must be its own page.  kv_pointers is
 *   [num_layers, batch, 2, max_blocks_per_seq]; parents, children int32 [num_pairs] and lens int32 [batch] are device arrays, trusted (a child
 *   must not be a parent or appear twice; rows in [0, batch)).  Pages 16-byte aligned.  Everything is read after the dependency wait.      */
QS_API int qs_kv_cache_fork(const int64_t* kv_pointers, const int32_t* parents, const int32_t* children, const int32_t* lens, int num_layers,
                            int batch, int num_pairs, int max_blocks_per_seq, int num_kv_heads, int tokens_per_block, int size_per_token,
                            int int4_kv_cache, void* stream);

/* Sampling on the GPU (the sampler's warpers and draw, and sampled acceptance of draft trees).
 *
 * Per row: temperature T (fp32), top_k (int32, -1 disables) and top_p (fp32), device arrays.  A row is GREEDY if T < 1e-5 or top_p < 1e-8,
 * or if it has no logit other than NaN / -inf: its token is what qs_argmax_rows returns.  Otherwise z = x / T (IEEE fp32), w = exp(z - max z),
 * NaN and -inf logits weigh 0, and the kept set is {z >= max(tau_p, tau_k)}: tau_k is the k-th largest z (top_k > 0, clamped to the count
 * of such logits), tau_p the smallest z whose strictly larger weight is < top_p * sum w (top_p < 1).  This is Hugging Face's TopP then TopK
 * warper (min_tokens_to_keep = 1) independent of tie order.  Draws: Philox4x32-10 with counter (lo(off), hi(off), row, j) and key (lo(seed),
 * hi(seed)), u = (x0 >> 8) * 2^-24, off = offsets[row]; every call advances offsets[row] by one (also for greedy rows).  The token is the
 * smallest index t with sum_{j <= t, kept} w_j > u * sum_kept w.  Weight sums are exact 64-bit fixed-point sums, so a call is bitwise
 * deterministic.  vocab % 8 == 0, vocab <= 196608; logits rows 16-byte aligned.  Parameter arrays are trusted (not read on the host);
 * everything is read after the PDL dependency wait; CUDA-graph capturable.
 *
 * qs_sample_rows: out int64 [rows] (draw j = 0).
 * qs_tree_accept_sampling: the sampled counterpart of qs_tree_accept_greedy (same draft_tokens, tree_mask and outputs), per-sequence
 *   parameters and offsets [batch].  logits fp16 [batch, num_nodes, vocab] are the verify logits; draft_probs fp32 [batch, num_nodes, vocab]
 *   or NULL: row c is the distribution q_c node c's token was drawn from (NULL: one-hot at draft[c]).  From the root with p = the warped
 *   logits of node 0, the children of the current node are tried in index order: child c with token d is accepted iff u_c q_c(d) < p(d)
 *   (u_c: draw j = c); accepting moves to c with p = the warped logits of c, rejecting sets p <- max(p - q_c, 0) renormalised (kept if its
 *   mass is 0).  Padding and out-of-range drafts are never accepted and leave p unchanged.  With no child accepted, bonus is drawn from p
 *   (draw j = 0).  This keeps the target distribution exactly (SpecInfer multi-step speculative sampling).  Greedy rows give exactly
 *   qs_tree_accept_greedy(draft, mask, argmax of every node's logits).  num_nodes <= 16.                                                     */
QS_API int qs_sample_rows(int64_t* out, const void* logits, const float* temperature, const int32_t* top_k, const float* top_p, uint64_t seed,
                          int64_t* offsets, int rows, int vocab, void* stream);
QS_API int qs_tree_accept_sampling(const int64_t* draft_tokens, const int32_t* tree_mask, const void* logits, const float* draft_probs,
                                   const float* temperature, const int32_t* top_k, const float* top_p, uint64_t seed, int64_t* offsets,
                                   int32_t* accept_len, int32_t* path, int64_t* bonus, int batch, int num_nodes, int vocab, void* stream);

/* Penalties and log-probabilities (SamplingParams.repetition_penalty / presence_penalty / frequency_penalty, logprobs / prompt_logprobs).
 * Both read everything after the PDL dependency wait, need no host synchronisation and are CUDA-graph capturable; vocab % 8 == 0,
 * vocab <= 196608.  Parameter arrays are trusted (not read on the host).
 *
 * qs_apply_penalties: fp16 logits [rows, vocab] modified in place before sampling (vLLM's semantics).  history int64 [rows, history_len]:
 *   the prompt at [0, prompt_lens[r]), the generated tokens at [prompt_lens[r], seq_lens[r]); prompt_lens / seq_lens int32 [rows] are clamped
 *   to 0 <= prompt_lens <= seq_lens <= history_len before any read; ids outside [0, vocab) (-1: padding) are ignored.  repetition fp32 (in
 *   (0, 2]), presence and frequency fp32 (in [-2, 2]), [rows].  For every token t that occurs in the row's history, with c = its count among
 *   the generated tokens, x = float(logit[t]) in IEEE fp32 without FMA contraction: (1) if repetition != 1, x = x > 0 ? x / repetition :
 *   x * repetition; (2) if c > 0, x = (x - (frequency * c)) - presence; then one rounding to fp16.  Each distinct token is written once (no
 *   atomics: bitwise deterministic) and only when its bits change; NaN logits and rows with (1, 0, 0) are not written, and no logit outside
 *   the history is touched.  history_len <= 32768.
 * qs_logprobs_rows: for fp16 logits [rows, vocab] and tokens int64 [rows] (the sampled token, or the next prompt token): logprob fp32 [rows]
 *   = the token's log-probability and, for 0 <= n <= 20, top_ids int64 [rows, n] / top_logprobs fp32 [rows, n] = the n largest logits by
 *   (logit descending, index ascending; -0 ties with +0).  The distribution is the sampler's softmax at T = 1: NaN and -inf weigh 0,
 *   w = exp(x - max) with w = 1 where x == max (+inf logits share the mass), the weight sum in 64-bit fixed point.  A row without weight
 *   gives NaN log-probabilities and top_ids -1; an out-of-range token gives NaN; with fewer than n non-NaN logits the remaining slots get -1
 *   and -inf.  top_ids / top_logprobs may be NULL when n = 0.                                                                          */
QS_API int qs_apply_penalties(void* logits, const int64_t* history, const int32_t* prompt_lens, const int32_t* seq_lens, const float* repetition,
                              const float* presence, const float* frequency, int rows, int vocab, int history_len, void* stream);
QS_API int qs_logprobs_rows(float* logprob, int64_t* top_ids, float* top_logprobs, const void* logits, const int64_t* tokens, int rows, int vocab,
                            int n, void* stream);

/* The same penalties and log-probabilities inside a speculative step (same conventions as above).
 *
 * qs_apply_penalties_tree: fp16 verify logits [batch, num_nodes, vocab] of a draft tree (num_nodes <= 16; draft_tokens int64 and tree_mask
 *   int32 [batch, num_nodes], the ancestor words of qs_tree_decode_attention), modified in place before acceptance.  Row b's history follows
 *   the generation loop: h[0 .. L) with L = seq_lens[b] (clamped to [0, history_len]), h[L - 1] is the root, node 0.  Node i's row is, bit for
 *   bit, what qs_apply_penalties writes for that row given the EXPANDED history: h[0 .. L), then the tokens of node i's ancestors j >= 1 (bits
 *   of tree_mask[b, i] below i) in index order, then node i's own token if i >= 1, with the row's prompt_len and parameters.  The expanded
 *   history is not clipped at history_len.  Ids outside [0, vocab) (-1: padding nodes) are ignored; neutral rows and NaN logits are not
 *   written; each (node, token) is written once at most (no atomics).  history_len <= 32768.
 * qs_logprobs_accepted: the log-probabilities of the tokens a speculative step emits, before qs_spec_commit[_stops] commits them.  For every
 *   unfinished row (finished[b] == 0) with acc = accept_len[b] clamped to [1, num_nodes] (path entries to [0, num_nodes - 1], as the commit
 *   clamps them): emitted token k < acc (draft_tokens[b, path[b, k + 1]] for k < acc - 1, else bonus[b]) is scored by node row path[b, k] of
 *   logits fp16 [batch, num_nodes, vocab] with exactly the qs_logprobs_rows arithmetic, and written at column c = min(max(seq_lens[b], 0),
 *   width) + k of logprob fp32 [batch, width] and top_ids int64 / top_logprobs fp32 [batch, width, n] (n <= 20; NULL when n = 0): the column
 *   where the commit puts the token.  Columns >= width are dropped; finished rows and tokens past acc write nothing.  After the commit,
 *   column c is valid for prompt_lens[b] <= c < seq_lens[b]; entries of tokens the commit cut (eos, a stop token, the budget) are
 *   unspecified.  A plain decode step is the call with num_nodes = 1, path = 0, accept_len = 1 and bonus = its token.                     */
QS_API int qs_apply_penalties_tree(void* logits, const int64_t* draft_tokens, const int32_t* tree_mask, const int64_t* history,
                                   const int32_t* prompt_lens, const int32_t* seq_lens, const float* repetition, const float* presence,
                                   const float* frequency, int batch, int num_nodes, int vocab, int history_len, void* stream);
QS_API int qs_logprobs_accepted(float* logprob, int64_t* top_ids, float* top_logprobs, const void* logits, const int64_t* draft_tokens,
                                const int32_t* path, const int32_t* accept_len, const int64_t* bonus, const int32_t* seq_lens,
                                const int32_t* finished, int batch, int num_nodes, int vocab, int n, int width, void* stream);

/* Prompt-lookup speculative decoding: the drafter and the commit that close the loop around the tree verify and acceptance above.  Both read
 * every input after the PDL dependency wait (the previous step's commit writes the history and the lengths), need no host synchronisation,
 * are CUDA-graph capturable and bitwise deterministic.  Row state: history int64 [batch, history_len] holds the prompt and the generated
 * tokens, seq_lens int32 [batch] = L, the last token h[L - 1] (the ROOT) is the latest emitted token and is not yet in the KV cache, so the
 * cache holds L - 1 tokens.
 *
 * qs_ngram_propose: a draft tree of num_nodes = n <= 16 nodes (root included) per row from the row's own history (Saxena 2023 prompt
 *   lookup).  L is clamped to [0, history_len <= 32768].  For every end position j in [0, L - 2], m(j) is the largest g <= min(n_max, j + 1)
 *   with h[j - g + 1 .. j] == h[L - g .. L - 1] and every id of both windows >= 0 (the windows may overlap).  Candidates are the j with
 *   m(j) >= n_min, ranked by (m descending, j descending); the first `branches` are taken.  The continuation of candidate j is
 *   h[j + 1 .. min(j + n - 1, L - 1)].  Node 0 is the root (token h[L - 1], or -1 if L = 0; mask 0).  The continuations are inserted in rank
 *   order into a trie below the root: an existing child with the same token is followed, otherwise node `count` is created (creation order is
 *   topological) with mask = mask[parent] | (1 << parent), until n nodes exist.  Uncreated nodes are padding: token -1, mask 1.  Outputs
 *   tokens int64 [batch, n] and tree_mask int32 [batch, n], the ancestor words of qs_tree_decode_attention.  1 <= n_min <= n_max <= 8,
 *   1 <= branches <= 8.
 * qs_spec_commit: advances every unfinished row (finished[b] == 0; finished rows are not touched) by what its step accepted: draft_tokens
 *   int64 [batch, n], path int32 [batch, n], accept_len int32 [batch] and bonus int64 [batch] as qs_tree_accept_greedy / _sampling return
 *   them (acc = accept_len clamped to [1, n], path entries to [0, n - 1]).  The appended tokens draft[path[1 .. acc - 1]], bonus are cut after
 *   the first eos[b] (eos < 0: none), then to budget[b] - (L - prompt_lens[b]) (at least 0) tokens, written at history[L ..] (columns >=
 *   history_len dropped) and L += count.  Then start_pos = L - 1, context_lens = L and roots = the row's last token (the last appended one,
 *   else h[L - 1]); context_lens and roots may be NULL.  The row becomes finished if it appended eos or L - prompt_lens >= budget.  A plain
 *   decode step is the call with n = 1, path = 0, accept_len = 1 and bonus = the sampled token.                                          */
QS_API int qs_ngram_propose(const int64_t* history, const int32_t* seq_lens, int64_t* tokens, int32_t* tree_mask, int batch, int history_len,
                            int num_nodes, int n_min, int n_max, int branches, void* stream);
QS_API int qs_spec_commit(const int64_t* draft_tokens, const int32_t* path, const int32_t* accept_len, const int64_t* bonus, int64_t* history,
                          int32_t* seq_lens, const int32_t* prompt_lens, const int32_t* budget, const int64_t* eos, int32_t* finished,
                          int32_t* start_pos, int32_t* context_lens, int64_t* roots, int batch, int num_nodes, int history_len, void* stream);
/* qs_spec_commit_stops: qs_spec_commit with a stop-token set per row, stop_ids int64 [batch, num_stops] (num_stops <= 8, entries < 0 pad):
 *   the first appended token in {eos[b]} or the row's set ends the row exactly as eos does (appended, the cut after it, finished; the
 *   budget cut still wins).  stop_ids may be NULL when num_stops = 0, which gives exactly qs_spec_commit.                                */
QS_API int qs_spec_commit_stops(const int64_t* draft_tokens, const int32_t* path, const int32_t* accept_len, const int64_t* bonus,
                                int64_t* history, int32_t* seq_lens, const int32_t* prompt_lens, const int32_t* budget, const int64_t* eos,
                                const int64_t* stop_ids, int num_stops, int32_t* finished, int32_t* start_pos, int32_t* context_lens,
                                int64_t* roots, int batch, int num_nodes, int history_len, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QSERVE_B200_H_ */
