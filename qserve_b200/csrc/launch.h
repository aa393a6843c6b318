// qserve_b200 -- internal host-side launch interfaces shared by the translation units.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace qs {

bool pdl_enabled();
// host-side caches (kernel attributes, SM count) are keyed by the CURRENT device ordinal: one process may drive several GPUs
constexpr int kMaxDevices = 64;
int device_ordinal();
int num_sms();

struct GemmArgs {
  const void* act = nullptr;        // int8 [M, K]
  const void* weight = nullptr;     // W4: packed int4 [N, K/2] (reference layout); W8: int8 [N, K]
  const void* s2_scales = nullptr;  // per-group
  const void* s2_zeros = nullptr;   // per-group
  const void* wscales = nullptr;    // fp16 [N]
  const void* w_szs = nullptr;      // fp16 [N] per-channel
  const void* ascales = nullptr;    // fp16 [M]
  const void* a_ssums = nullptr;    // fp16 [M] per-channel
  void* out = nullptr;              // fp16 [M, N]
  void* acc_out = nullptr;          // optional int32 [M, N]
  int M = 0, N = 0, K = 0;
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  int force_split = 0;          // tests: force the cluster split-K factor (1, 2, 4, 8); 0 = automatic
  int force_nt = 0;             // tests / tuning: force the tokens-per-tile (32, 64, 128); 0 = automatic
  void* prof = nullptr;         // optional device buffer: 16 x uint64 globaltimer stamps per CTA
  void* stream = nullptr;
};

int gemm_w4a8_per_chn(const GemmArgs& a);
int gemm_w4a8_per_group(const GemmArgs& a);
int gemm_w8a8(const GemmArgs& a);
size_t gemm_workspace_bytes();
int gemm_trace_install(void* buf, unsigned cap);
int attention_trace_install(void* buf, unsigned cap);
int elementwise_trace_install(void* buf, unsigned cap);

// elementwise.cu
int rms_norm(void* out, const void* in, const void* weight, float eps, int use_quant, int tokens, int hidden, void* stream);
int layernorm_general_quant(void* out_q, const void* in, const void* gamma, void* input_sum, void* scaling, float eps, int tokens,
                            int hidden, int per_token, void* stream);
int quant_per_token(void* out_q, const void* in, void* input_sum, void* scale, int tokens, int hidden, void* stream);
int quant_scalar(void* out_q, const void* in, float scale, int tokens, int hidden, void* stream);
int row_absmax(void* amax_f32, const void* in, int tokens, int hidden, void* stream);
int quant_given_amax(void* out_q, const void* in, const void* amax_f32, void* input_sum, void* scale, int tokens, int hidden, void* stream);
int silu_and_mul(void* out, const void* in, int tokens, int d, void* stream);
int argmax_rows(void* out_i64, const void* logits_f16, int rows, int vocab, void* stream);
int silu_and_mul_quant(void* out_q, const void* in, void* input_sum, void* scale, int tokens, int d, void* stream);
int add_layernorm_quant(void* out_q, void* hidden_out, const void* x, const void* delta, const void* gamma, void* input_sum, void* scaling, float eps,
                        int tokens, int hidden, void* stream);
int add_layernorm_quant_peer(void* out_q, void* hidden_out, const void* x, const void* const* delta_ptrs, void* const* flag_ptrs, void* state, int world,
                             int rank, int phase, const void* gamma, void* input_sum, void* scaling, float eps, int tokens, int hidden, void* stream);
int gelu(void* out, const void* in, int tokens, int d, int fast, void* stream);
int dequant_add_residual(void* out, const void* in_i32, const void* residual, const void* scale_vec, float scale, int tokens, int hidden,
                         void* stream);
int dequant(void* out, const void* in_i32, float scale, int tokens, int hidden, int in_stride, int out_stride, void* stream);
int dequant_add_residual_rms_norm_quant(void* out_q, const void* in_i32, void* residual, const void* gamma, const void* scale_vec,
                                        float scale, float eps, int tokens, int hidden, void* stream);
int dequant_silu_and_mul_quant(void* out_q, const void* in_i32, float scale_gate, float scale_up, float scale_out, void* scale_out_vec,
                               void* tmp, int tokens, int d, void* stream);

// attention.cu
struct DecodeAttnArgs {
  const void* q = nullptr;  // fp16, row stride q_stride elements
  const void* k = nullptr;
  const void* v = nullptr;
  long long q_stride = 0, k_stride = 0, v_stride = 0;
  const long long* kv_pointers = nullptr;  // [B, 2, max_blocks] absolute device addresses
  const int* lengths = nullptr;            // [B] context length including the new token
  void* out = nullptr;                     // fp16 [B, Hq, D] contiguous
  void* q_out = nullptr;                   // fused-quant extension: int8 [B, Hq*D] (then `out` is not written)
  void* q_scale = nullptr;                 //   fp16 [B]
  void* q_sum = nullptr;                   //   fp16 [B] or null
  void* prof = nullptr;                    // optional: 16 globaltimer stamps per CTA (tools/attn_timeline.py)
  int batch = 0, num_heads = 0, num_kv_heads = 0, head_dim = 0, max_blocks = 0;
  int tokens_per_block = 64, size_per_token = 0, timestep = 0, memory_max_len = 0;
  int rotary_dim = 0;
  float rotary_base = 10000.f;
  int int4_kv = 1, kv_zeros = 1;
  void* workspace = nullptr;
  size_t workspace_bytes = 0;
  void* stream = nullptr;
};
int decode_attention(const DecodeAttnArgs& a);
size_t attention_workspace_bytes(int batch, int num_heads, int head_dim, int max_splits);

struct PrefillAppendArgs {
  void* qkv = nullptr;  // fp16 [T, (Hq + 2 Hkv) * D], q and k rotated in place
  const int* seq_lens = nullptr;
  const int* padding_offset = nullptr;
  const long long* kv_pointers = nullptr;  // may be null: rotate only
  const int* start_pos = nullptr;          // optional [batch]: tokens of each sequence already cached; token pos sits at start_pos[b] + pos
  int batch = 0, num_tokens = 0, max_blocks = 0, num_heads = 0, num_kv_heads = 0, head_dim = 0;
  int seq_len = 0, tokens_per_block = 64, size_per_token = 0, rotary_dim = 0, max_positions = 0;
  float rotary_base = 10000.f;
  int int4_kv = 1, kv_zeros = 1;
  void* stream = nullptr;
};
int prefill_rope_append(const PrefillAppendArgs& a);
int padding_offsets(int* out, const int* cu_seqlens, int batch, int max_seqlen, void* stream);

// prefill_attention.cu: causal variable-length self-attention over the post-RoPE fp16 q / k / v of a prompt batch
struct PrefillAttnArgs {
  const void* q = nullptr;    // fp16 [T, Hq, 128], rows of q_stride halfs
  const void* k = nullptr;    // fp16 [T, Hkv, 128]
  const void* v = nullptr;
  void* out = nullptr;        // fp16 [T, Hq, 128], rows of out_stride halfs
  long long q_stride = 0, k_stride = 0, v_stride = 0, out_stride = 0;
  const int* cu_seqlens = nullptr;  // [batch + 1] token offsets (q and k share them: self-attention over the prompt)
  int batch = 0, num_tokens = 0, max_seqlen = 0, num_heads = 0, num_kv_heads = 0, head_dim = 0;
  float softmax_scale = 0.f;
  void* stream = nullptr;
};
int prefill_attention(const PrefillAttnArgs& a);

// prefix_attention.cu: causal attention of a batch of prompt chunks over their cached prefix (dequantised from the INT4 / INT8 pages) and
// over the chunk itself (fp16 q / k / v)
struct PrefixAttnArgs {
  const void* q = nullptr;    // fp16 [T, Hq, 128] chunk rows, rows of q_stride halfs
  const void* k = nullptr;    // fp16 [T, Hkv, 128]
  const void* v = nullptr;
  void* out = nullptr;        // fp16 [T, Hq, 128], rows of out_stride halfs
  long long q_stride = 0, k_stride = 0, v_stride = 0, out_stride = 0;
  const int* cu_seqlens = nullptr;         // [batch + 1] chunk token offsets
  const int* prefix_lens = nullptr;        // [batch] tokens already in the cache (<= max_prefix_len)
  const long long* kv_pointers = nullptr;  // [batch, 2, max_blocks] absolute page addresses
  int batch = 0, num_tokens = 0, max_seqlen = 0, max_prefix_len = 0, max_blocks = 0;
  int num_heads = 0, num_kv_heads = 0, head_dim = 0, tokens_per_block = 64, size_per_token = 0;
  int int4_kv = 1;
  float softmax_scale = 0.f;
  void* stream = nullptr;
};
int prefix_attention(const PrefixAttnArgs& a);

}  // namespace qs
