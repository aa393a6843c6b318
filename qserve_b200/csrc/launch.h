// qserve_b200 -- internal host-side launch interfaces shared by the translation units.
#pragma once
#include <stddef.h>
#include <stdint.h>

struct qs_inflight_args;  // include/qserve_b200.h

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
// decode attention of rows that share the first pages of their group (qs_shared_prefix_decode_attention): d as for decode_attention (exactly
// one of d.out / d.q_out; d.lengths required; d.workspace >= shared_prefix_attention_workspace_bytes), plus the group layout
struct SharedPrefixAttnArgs {
  DecodeAttnArgs d;
  const int* group_offsets = nullptr;  // [num_groups + 1]
  const int* group_rows = nullptr;     // [group_offsets[num_groups]]
  const int* group_pages = nullptr;    // [num_groups] shared pages S_g
  const int* row_pages = nullptr;      // [batch] S of the row's group, 0 outside groups
  int num_groups = 0, max_group = 0, max_pages = 0;  // host bounds that plan the launches
};
int shared_prefix_decode_attention(const SharedPrefixAttnArgs& a);
size_t shared_prefix_attention_workspace_bytes(int batch, int num_heads, int num_kv_heads, int timestep, int num_groups, int max_group, int max_pages,
                                               int int4_kv);

struct PrefillAppendArgs {
  void* qkv = nullptr;  // fp16 [T, (Hq + 2 Hkv) * D], q and k rotated in place
  const int* seq_lens = nullptr;
  const int* padding_offset = nullptr;
  const long long* kv_pointers = nullptr;  // may be null: rotate only
  const int* start_pos = nullptr;          // optional [batch]: tokens of each sequence already cached; token pos sits at start_pos[b] + pos
  const int* tree_mask = nullptr;          // optional [num_tokens] draft-tree ancestor words (needs start_pos): node i is rotated at
                                           // start_pos[b] + depth(i) and stored in slot start_pos[b] + i
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

// multi_token_attention.cu: n <= 16 draft tokens per sequence over the paged INT4 / INT8 cache, each with the semantics of one decode step
// (speculative-decoding verification)
struct MultiTokenAttnArgs {
  const void* q = nullptr;    // fp16 [T, Hq, 128] draft rows (rotated), rows of q_stride halfs
  const void* k = nullptr;    // fp16 [T, Hkv, 128] (rotated)
  const void* v = nullptr;
  void* out = nullptr;        // fp16 [T, Hq, 128], rows of out_stride halfs
  long long q_stride = 0, k_stride = 0, v_stride = 0, out_stride = 0;
  const int* cu_seqlens = nullptr;         // [batch + 1] draft token offsets
  const int* prefix_lens = nullptr;        // [batch] tokens cached before the draft tokens (<= max_prefix_len)
  const long long* kv_pointers = nullptr;  // [batch, 2, max_blocks] absolute page addresses
  int batch = 0, num_tokens = 0, max_seqlen = 0, max_prefix_len = 0, max_blocks = 0;
  int num_heads = 0, num_kv_heads = 0, head_dim = 0, tokens_per_block = 64, size_per_token = 0;
  int int4_kv = 1;
  float softmax_scale = 0.f;  // <= 0: 1 / sqrt(128) exactly as the decode kernel computes it
  const int* tree_mask = nullptr;  // optional [num_tokens] ancestor words of tree-structured drafts (qs_tree_decode_attention)
  void* workspace = nullptr;  // zero-initialised once, then owned by the library (self-cleaning counters)
  size_t workspace_bytes = 0;
  void* stream = nullptr;
};
int multi_token_attention(const MultiTokenAttnArgs& a);
size_t multi_token_attention_workspace_bytes(int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads,
                                             int int4_kv);

// tree_verify.cu: greedy acceptance of a draft tree and compaction of the accepted path's K / V slots (speculative decoding with token trees)
int tree_accept_greedy(const long long* draft, const int* tree_mask, const long long* target, int* accept_len, int* path, long long* bonus,
                       int batch, int num_nodes, void* stream);
struct KvCompactArgs {
  const long long* kv_pointers = nullptr;  // [layers, batch, 2, max_blocks] absolute page addresses
  const int* start_pos = nullptr;          // [batch] tokens cached before the draft nodes
  const int* path = nullptr;               // [batch, num_nodes] accepted node indices
  const int* accept_len = nullptr;         // [batch]
  int layers = 1, batch = 0, num_nodes = 0, max_blocks = 0, num_kv_heads = 0, tokens_per_block = 64, size_per_token = 0, int4_kv = 1;
  void* stream = nullptr;
};
int kv_cache_compact(const KvCompactArgs& a);

// kv_fork.cu: copy-on-write fork of a cached prompt's partial tail page into other sequences (SamplingParams.n / best_of)
struct KvForkArgs {
  const long long* kv_pointers = nullptr;  // [layers, batch, 2, max_blocks] absolute page addresses
  const int* parents = nullptr;            // [num_pairs] parent rows
  const int* children = nullptr;           // [num_pairs] child rows
  const int* lens = nullptr;               // [batch] cached tokens of each row (read at the parent rows)
  int layers = 1, batch = 0, num_pairs = 0, max_blocks = 0, num_kv_heads = 0, tokens_per_block = 64, size_per_token = 0, int4_kv = 1;
  void* stream = nullptr;
};
int kv_cache_fork(const KvForkArgs& a);

// beam_search.cu: per-request beam selection and the in-place re-parenting of every beam's pages, tables and history
struct BeamSelectArgs {
  const long long* top_ids = nullptr;     // [batch, 2 W] candidates of every slot (logprobs_rows, n = 2 W)
  const float* top_logprobs = nullptr;    // [batch, 2 W]
  int* live = nullptr;                    // [batch], updated
  float* cum = nullptr;                   // [batch] cumulative log-probabilities, updated
  int* seq_lens = nullptr;                // [batch] tokens per beam (prompt + generated), read at the request's first slot, set
  int* context_lens = nullptr;            // [batch] set
  long long* tokens = nullptr;            // [batch] out: the token of every live slot
  int* parents = nullptr;                 // [batch] out: parent slot, -1 dead
  const int* prompt_lens = nullptr;       // [batch]
  const long long* history = nullptr;     // [batch, history_len]
  const float* length_penalty = nullptr;  // [num_requests]
  const int* early_stopping = nullptr;    // [num_requests] 0 False, 1 True, 2 "never"
  const long long* eos = nullptr;         // [num_requests], -1 none
  const long long* stop_ids = nullptr;    // [num_requests, num_stops], -1 pads
  const int* budget = nullptr;            // [num_requests] max_tokens
  int* done = nullptr;                    // [num_requests], set
  long long* pool_tokens = nullptr;       // [num_requests, W, max_tokens] finished hypotheses, best first
  int* pool_len = nullptr;                // [num_requests, W] generated tokens of each hypothesis
  float* pool_cum = nullptr;              // [num_requests, W]
  float* pool_score = nullptr;            // [num_requests, W]
  int* pool_count = nullptr;              // [num_requests]
  int num_requests = 0, beam_width = 1, num_stops = 0, max_tokens = 0, max_model_len = 0, history_len = 0;
  void* stream = nullptr;
};
int beam_select(const BeamSelectArgs& a);
struct BeamReorderArgs {
  long long* kv_pointers = nullptr;    // [layers, batch, 2, max_blocks] absolute page addresses, entries below P / 64 rewritten
  const int* parents = nullptr;        // [batch] parent slot inside the request, -1 dead
  const int* context_lens = nullptr;   // [batch] P + 1
  const int* prompt_lens = nullptr;    // [batch]
  const long long* tokens = nullptr;   // [batch] appended at history column P
  long long* history = nullptr;        // [batch, history_len]
  int layers = 1, batch = 0, beam_width = 1, max_blocks = 0, num_kv_heads = 0, tokens_per_block = 64, size_per_token = 0, int4_kv = 1, history_len = 0;
  void* stream = nullptr;
};
int beam_reorder(const BeamReorderArgs& a);

// sampling.cu: temperature / top-p / top-k sampling of fp16 logits and sampled (lossless) acceptance of draft trees; Philox4x32-10 draws
// keyed by `seed` and counted by the per-row `offsets`, which every call advances by one
struct SampleArgs {
  long long* out = nullptr;            // int64 [rows]
  const void* logits = nullptr;        // fp16 [rows, vocab]
  const float* temperature = nullptr;  // [rows]
  const int* top_k = nullptr;          // [rows], -1 disables
  const float* top_p = nullptr;        // [rows]
  long long* offsets = nullptr;        // [rows], read and advanced by one
  unsigned long long seed = 0;
  int rows = 0, vocab = 0;
  void* stream = nullptr;
};
int sample_rows(const SampleArgs& a);
struct TreeAcceptSamplingArgs {
  const long long* draft = nullptr;    // [batch, num_nodes]
  const int* tree_mask = nullptr;      // [batch, num_nodes] ancestor words
  const void* logits = nullptr;        // fp16 [batch, num_nodes, vocab]
  const float* draft_probs = nullptr;  // optional fp32 [batch, num_nodes, vocab]; null: one-hot at the draft token
  const float* temperature = nullptr;  // [batch]
  const int* top_k = nullptr;
  const float* top_p = nullptr;
  long long* offsets = nullptr;        // [batch], read and advanced by one
  unsigned long long seed = 0;
  int* accept_len = nullptr;           // [batch]
  int* path = nullptr;                 // [batch, num_nodes]
  long long* bonus = nullptr;          // [batch]
  int batch = 0, num_nodes = 0, vocab = 0;
  void* stream = nullptr;
};
int tree_accept_sampling(const TreeAcceptSamplingArgs& a);
// repetition / presence / frequency penalties applied in place to fp16 logits before sampling
struct PenaltyArgs {
  void* logits = nullptr;               // fp16 [rows, vocab], modified in place
  const long long* history = nullptr;   // [rows, history_len] token ids: prompt, then generated tokens; -1 / out of range ignored
  const int* prompt_lens = nullptr;     // [rows]
  const int* seq_lens = nullptr;        // [rows], clamped to 0 <= prompt_lens <= seq_lens <= history_len on the device
  const float* repetition = nullptr;    // [rows]
  const float* presence = nullptr;
  const float* frequency = nullptr;
  int rows = 0, vocab = 0, history_len = 0;
  void* stream = nullptr;
};
int apply_penalties(const PenaltyArgs& a);
// log-probability of a chosen token and the n <= 20 most likely tokens of each row's softmax (T = 1)
struct LogprobArgs {
  float* logprob = nullptr;         // [rows]
  long long* top_ids = nullptr;     // [rows, n]
  float* top_logprobs = nullptr;    // [rows, n]
  const void* logits = nullptr;     // fp16 [rows, vocab]
  const long long* tokens = nullptr;  // [rows]
  int rows = 0, vocab = 0, n = 0;
  void* stream = nullptr;
};
int logprobs_rows(const LogprobArgs& a);
// apply_penalties on every node row of a draft tree, each node's history extended by its ancestors' tokens and its own
struct PenaltyTreeArgs {
  void* logits = nullptr;               // fp16 [batch, num_nodes, vocab], modified in place
  const long long* draft = nullptr;     // [batch, num_nodes]: node 0 is the root (h[seq_lens - 1], not read), -1 / out of range ignored
  const int* tree_mask = nullptr;       // [batch, num_nodes] ancestor words
  const long long* history = nullptr;   // [batch, history_len]
  const int* prompt_lens = nullptr;     // [batch]
  const int* seq_lens = nullptr;        // [batch], clamped to [0, history_len] on the device
  const float* repetition = nullptr;    // [batch]
  const float* presence = nullptr;
  const float* frequency = nullptr;
  int batch = 0, num_nodes = 0, vocab = 0, history_len = 0;
  void* stream = nullptr;
};
int apply_penalties_tree(const PenaltyTreeArgs& a);
// logprobs_rows of the tokens a speculative step emits, scored by their node rows and written at their history columns
struct LogprobAcceptedArgs {
  float* logprob = nullptr;             // [batch, width]
  long long* top_ids = nullptr;         // [batch, width, n]
  float* top_logprobs = nullptr;        // [batch, width, n]
  const void* logits = nullptr;         // fp16 [batch, num_nodes, vocab]
  const long long* draft = nullptr;     // [batch, num_nodes]
  const int* path = nullptr;            // [batch, num_nodes]
  const int* accept_len = nullptr;      // [batch]
  const long long* bonus = nullptr;     // [batch]
  const int* seq_lens = nullptr;        // [batch], before the commit
  const int* finished = nullptr;        // [batch]
  int batch = 0, num_nodes = 0, vocab = 0, n = 0, width = 0;
  void* stream = nullptr;
};
int logprobs_accepted(const LogprobAcceptedArgs& a);

// speculative.cu: prompt-lookup draft trees from the token history, and the commit that advances every sequence by what it accepted
struct NgramProposeArgs {
  const long long* history = nullptr;  // [batch, history_len]
  const int* seq_lens = nullptr;       // [batch], clamped to [0, history_len] on the device
  long long* tokens = nullptr;         // [batch, num_nodes] out: root, drafted nodes, padding -1
  int* tree_mask = nullptr;            // [batch, num_nodes] out: ancestor words, padding 1
  int batch = 0, history_len = 0, num_nodes = 0, n_min = 1, n_max = 4, branches = 1;
  void* stream = nullptr;
};
int ngram_propose(const NgramProposeArgs& a);
struct SpecCommitArgs {
  const long long* draft = nullptr;    // [batch, num_nodes]
  const int* path = nullptr;           // [batch, num_nodes]
  const int* accept_len = nullptr;     // [batch]
  const long long* bonus = nullptr;    // [batch]
  long long* history = nullptr;        // [batch, history_len], appended in place
  int* seq_lens = nullptr;             // [batch], advanced in place
  const int* prompt_lens = nullptr;    // [batch]
  const int* budget = nullptr;         // [batch] tokens a row may generate
  const long long* eos = nullptr;      // [batch], -1: none
  int* finished = nullptr;             // [batch], set in place
  int* start_pos = nullptr;            // [batch] out: seq_lens - 1
  int* context_lens = nullptr;         // optional [batch] out: seq_lens
  long long* roots = nullptr;          // optional [batch] out: the last token of the row
  int batch = 0, num_nodes = 0, history_len = 0;
  void* stream = nullptr;
};
int spec_commit(const SpecCommitArgs& a);
// spec_commit with a stop-token set per row: stop_ids [batch, num_stops <= 8], -1 pads
int spec_commit_stops(const SpecCommitArgs& a, const long long* stop_ids, int num_stops);

// the in-flight step's schedule (inflight.cu): the arguments of qs_inflight_schedule
int inflight_schedule(const qs_inflight_args& a, void* stream);

}  // namespace qs
