// qserve_b200 -- extern "C" entry points (include/qserve_b200.h) and error plumbing.
#include <cstdarg>
#include <cstdio>
#include <map>
#include <mutex>
#include <utility>

#include "../../include/qserve_b200.h"
#include "common.cuh"
#include "launch.cuh"

namespace qs {

static thread_local char g_err[1024] = "";
static int g_pdl = 1;
static int g_force_split = 0;
static int g_force_nt = 0;
static void* g_gemm_prof = nullptr;

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return QS_OK;
  cudaGetLastError();  // clear the sticky launch error
  return set_error(QS_ERR_CUDA, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
}

bool pdl_enabled() { return g_pdl != 0; }

int device_ordinal() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}
int num_sms() {
  static int sms[kMaxDevices] = {};
  const int dev = device_ordinal();
  if (!sms[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    sms[dev] = n > 0 ? n : 132;
  }
  return sms[dev];
}

int check_page_geometry(const char* op, int head_dim, int num_heads, int num_kv_heads, int tokens_per_block, int size_per_token, int int4_kv) {
  QS_REQUIRE(head_dim == 128, "%s: head_dim=%d, only 128 is supported", op, head_dim);
  QS_REQUIRE(num_kv_heads > 0 && num_heads % num_kv_heads == 0, "%s: heads %d / kv heads %d", op, num_heads, num_kv_heads);
  QS_REQUIRE(tokens_per_block == 64, "%s: tokens_per_block=%d, only 64 is supported", op, tokens_per_block);
  const int bits = int4_kv ? 4 : 8;
  QS_REQUIRE(size_per_token == num_kv_heads * 128 * bits / 8, "%s: size_per_token=%d does not match %d kv heads x %d bits", op, size_per_token,
             num_kv_heads, bits);
  return QS_OK;
}

int raise_smem_limit(const void* kern, size_t bytes, const char* what) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> limits;
  const std::pair<const void*, int> key(kern, device_ordinal());
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = limits[key];
  if (bytes <= have) return QS_OK;
  const int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)), what);
  if (rc == QS_OK) have = bytes;
  return rc;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The GemmArgs fields the three GEMM entries share, and the process-wide tuning controls.
static GemmArgs gemm_args(const int8_t* in_feats, const int8_t* kernel, const void* wscales, const void* ascales, void* out_feats, int32_t* acc_out, int M,
                          int N, int K, void* workspace, size_t workspace_bytes, void* stream) {
  GemmArgs a;
  a.act = in_feats; a.weight = kernel; a.wscales = wscales; a.ascales = ascales; a.out = out_feats; a.acc_out = acc_out; a.M = M; a.N = N; a.K = K;
  a.workspace = workspace; a.workspace_bytes = workspace_bytes; a.force_split = g_force_split; a.force_nt = g_force_nt; a.prof = g_gemm_prof; a.stream = stream;
  return a;
}

// The three qs_apply_bias_rope_update_kv_cache* entries; start_pos and tree_mask are null where an entry has none.
static int rope_append(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int32_t* start_pos, const int32_t* tree_mask,
                       const int64_t* kv_pointers, int batch, int num_tokens, int max_blocks, int head_num, int kv_head_num, int head_dim, int seq_len,
                       int tokens_per_block, int size_per_token, int rotary_dim, float rotary_base, int max_positions, int int4_kv, int kv_zeros,
                       void* stream) {
  PrefillAppendArgs a;
  a.qkv = qkv; a.seq_lens = seq_lens; a.padding_offset = padding_offset; a.start_pos = start_pos; a.tree_mask = tree_mask;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.batch = batch; a.num_tokens = num_tokens; a.max_blocks = max_blocks;
  a.num_heads = head_num; a.num_kv_heads = kv_head_num; a.head_dim = head_dim; a.seq_len = seq_len; a.tokens_per_block = tokens_per_block;
  a.size_per_token = size_per_token; a.rotary_dim = rotary_dim; a.rotary_base = rotary_base; a.max_positions = max_positions; a.int4_kv = int4_kv;
  a.kv_zeros = kv_zeros; a.stream = stream;
  return prefill_rope_append(a);
}

// qs_multi_token_decode_attention (tree_mask null) and qs_tree_decode_attention.
static int multi_token(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out, int64_t out_stride,
                       const int32_t* cu_seqlens, const int32_t* prefix_lens, const int32_t* tree_mask, const int64_t* kv_pointers, int batch, int num_tokens,
                       int max_seqlen, int max_prefix_len, int max_blocks, int num_heads, int num_kv_heads, int head_dim, int tokens_per_block,
                       int size_per_token, int int4_kv, float softmax_scale, void* workspace, size_t workspace_bytes, void* stream) {
  MultiTokenAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.out = out; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride; a.out_stride = out_stride;
  a.cu_seqlens = cu_seqlens; a.prefix_lens = prefix_lens; a.tree_mask = tree_mask; a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers);
  a.batch = batch; a.num_tokens = num_tokens; a.max_seqlen = max_seqlen; a.max_prefix_len = max_prefix_len; a.max_blocks = max_blocks; a.num_heads = num_heads;
  a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.int4_kv = int4_kv;
  a.softmax_scale = softmax_scale; a.workspace = workspace; a.workspace_bytes = workspace_bytes; a.stream = stream;
  return multi_token_attention(a);
}

}  // namespace qs

using namespace qs;

extern "C" {

int qs_abi_version(void) { return QS_ABI_VERSION; }
const char* qs_last_error(void) { return g_err; }
int qs_set_pdl(int enabled) {
  const int old = g_pdl;
  g_pdl = enabled ? 1 : 0;
  return old;
}
int qs_gemm_force_tile_tokens(int nt) {
  const int old = g_force_nt;
  g_force_nt = nt;
  return old;
}

int qs_gemm_force_split(int split) {
  const int old = g_force_split;
  g_force_split = split;
  return old;
}
size_t qs_gemm_workspace_bytes(void) { return gemm_workspace_bytes(); }
int qs_set_trace_buffer(void* dev_buffer, unsigned capacity_records) {
  if (gemm_trace_install(dev_buffer, capacity_records) || attention_trace_install(dev_buffer, capacity_records) ||
      elementwise_trace_install(dev_buffer, capacity_records))
    return set_error(qs::QS_ERR_CUDA, "qs_set_trace_buffer: cudaMemcpyToSymbol failed");
  return 0;
}
int qs_gemm_set_profile_buffer(void* dev_buffer) {
  g_gemm_prof = dev_buffer;
  return 0;
}

int qs_w4a8_gemm_per_chn(const int8_t* in_feats, const int8_t* kernel, const void* wscales, const void* ascales, const void* w_szs,
                         const void* a_ssums, void* out_feats, int32_t* acc_out, int M, int N, int K, void* workspace, size_t workspace_bytes,
                         void* stream) {
  QS_REQUIRE(in_feats && kernel && wscales && ascales && w_szs && a_ssums && out_feats, "qgemm_w4a8_per_chn: null tensor");
  GemmArgs a = gemm_args(in_feats, kernel, wscales, ascales, out_feats, acc_out, M, N, K, workspace, workspace_bytes, stream);
  a.w_szs = w_szs; a.a_ssums = a_ssums;
  return gemm_w4a8_per_chn(a);
}

int qs_w4a8_gemm_per_group(const int8_t* in_feats, const int8_t* kernel, const int8_t* zeros, const int8_t* scales_i8, const void* wscales,
                           const void* ascales, void* out_feats, int32_t* acc_out, int M, int N, int K, void* workspace,
                           size_t workspace_bytes, void* stream) {
  QS_REQUIRE(in_feats && kernel && zeros && scales_i8 && wscales && ascales && out_feats, "qgemm_w4a8_per_group: null tensor");
  QS_REQUIRE(aligned16(zeros) && aligned16(scales_i8), "qgemm_w4a8_per_group: level-2 scale/zero tensors must be 16-byte aligned");
  GemmArgs a = gemm_args(in_feats, kernel, wscales, ascales, out_feats, acc_out, M, N, K, workspace, workspace_bytes, stream);
  a.s2_zeros = zeros; a.s2_scales = scales_i8;
  return gemm_w4a8_per_group(a);
}

int qs_w8a8_gemm(const int8_t* in_feats, const int8_t* kernel, const void* wscales, const void* ascales, void* out_feats, int32_t* acc_out,
                 int M, int N, int K, void* workspace, size_t workspace_bytes, void* stream) {
  QS_REQUIRE(in_feats && kernel && wscales && ascales && out_feats, "qgemm_w8a8: null tensor");
  return gemm_w8a8(gemm_args(in_feats, kernel, wscales, ascales, out_feats, acc_out, M, N, K, workspace, workspace_bytes, stream));
}

size_t qs_attention_workspace_bytes(int batch, int num_heads, int head_dim) { return attention_workspace_bytes(batch, num_heads, head_dim, 32); }

int qs_single_query_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                              const int64_t* kv_pointers, const int32_t* length_per_sample, void* out, int batch, int num_heads,
                              int num_kv_heads, int head_dim, int max_blocks_per_seq, int memory_max_seqlen, int tokens_per_block,
                              int size_per_token, int timestep, int rotary_embedding_dim, float rotary_base, int neox_rotary_style,
                              int int4_kv_cache, int kv_cache_with_zeros, void* workspace, size_t workspace_bytes, void* stream) {
  (void)neox_rotary_style;  // accepted and ignored: NeoX is hard-wired in the reference as well (fused_attention.cpp:109)
  QS_REQUIRE(q && k && v && kv_pointers && out, "single_query_attention: null tensor");
  DecodeAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.lengths = length_per_sample; a.out = out;
  a.batch = batch; a.num_heads = num_heads; a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.max_blocks = max_blocks_per_seq;
  a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.timestep = timestep; a.memory_max_len = memory_max_seqlen;
  a.rotary_dim = rotary_embedding_dim; a.rotary_base = rotary_base; a.int4_kv = int4_kv_cache; a.kv_zeros = kv_cache_with_zeros;
  a.workspace = workspace; a.workspace_bytes = workspace_bytes; a.prof = g_gemm_prof; a.stream = stream;
  return decode_attention(a);
}

int qs_single_query_attention_quant(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                                    const int64_t* kv_pointers, const int32_t* length_per_sample, int8_t* out_q, void* out_scale, void* out_sum, int batch,
                                    int num_heads, int num_kv_heads, int head_dim, int max_blocks_per_seq, int memory_max_seqlen, int tokens_per_block,
                                    int size_per_token, int timestep, int rotary_embedding_dim, float rotary_base, int int4_kv_cache,
                                    int kv_cache_with_zeros, void* workspace, size_t workspace_bytes, void* stream) {
  QS_REQUIRE(q && k && v && kv_pointers && out_q && out_scale, "single_query_attention_quant: null tensor");
  DecodeAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.lengths = length_per_sample; a.out = nullptr;
  a.q_out = out_q; a.q_scale = out_scale; a.q_sum = out_sum; a.workspace = workspace; a.workspace_bytes = workspace_bytes; a.prof = g_gemm_prof;
  a.batch = batch; a.num_heads = num_heads; a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.max_blocks = max_blocks_per_seq;
  a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.timestep = timestep; a.memory_max_len = memory_max_seqlen;
  a.rotary_dim = rotary_embedding_dim; a.rotary_base = rotary_base; a.int4_kv = int4_kv_cache; a.kv_zeros = kv_cache_with_zeros;
  a.stream = stream;
  return decode_attention(a);
}

int qs_apply_bias_rope_update_kv_cache(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int64_t* kv_pointers, int batch,
                                       int num_tokens, int max_blocks_per_seq, int head_num, int kv_head_num, int head_dim, int seq_len,
                                       int tokens_per_block, int size_per_token, int rotary_embedding_dim, float rotary_embedding_base,
                                       int rotary_embedding_max_positions, int neox_rotary_style, int int4_kv_cache, int kv_cache_with_zeros,
                                       void* stream) {
  (void)neox_rotary_style;
  QS_REQUIRE(qkv && seq_lens, "apply_bias_rope_update_kv_cache: null tensor");
  return rope_append(qkv, seq_lens, padding_offset, nullptr, nullptr, kv_pointers, batch, num_tokens, max_blocks_per_seq, head_num, kv_head_num, head_dim,
                     seq_len, tokens_per_block, size_per_token, rotary_embedding_dim, rotary_embedding_base, rotary_embedding_max_positions, int4_kv_cache,
                     kv_cache_with_zeros, stream);
}

int qs_apply_bias_rope_update_kv_cache_at(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int32_t* start_pos,
                                          const int64_t* kv_pointers, int batch, int num_tokens, int max_blocks_per_seq, int head_num, int kv_head_num,
                                          int head_dim, int seq_len, int tokens_per_block, int size_per_token, int rotary_embedding_dim,
                                          float rotary_embedding_base, int rotary_embedding_max_positions, int neox_rotary_style, int int4_kv_cache,
                                          int kv_cache_with_zeros, void* stream) {
  (void)neox_rotary_style;
  QS_REQUIRE(qkv && seq_lens && start_pos, "apply_bias_rope_update_kv_cache_at: null tensor");
  return rope_append(qkv, seq_lens, padding_offset, start_pos, nullptr, kv_pointers, batch, num_tokens, max_blocks_per_seq, head_num, kv_head_num, head_dim,
                     seq_len, tokens_per_block, size_per_token, rotary_embedding_dim, rotary_embedding_base, rotary_embedding_max_positions, int4_kv_cache,
                     kv_cache_with_zeros, stream);
}

int qs_apply_bias_rope_update_kv_cache_tree(void* qkv, const int32_t* seq_lens, const int32_t* padding_offset, const int32_t* start_pos,
                                            const int32_t* tree_mask, const int64_t* kv_pointers, int batch, int num_tokens, int max_blocks_per_seq,
                                            int head_num, int kv_head_num, int head_dim, int seq_len, int tokens_per_block, int size_per_token,
                                            int rotary_embedding_dim, float rotary_embedding_base, int rotary_embedding_max_positions,
                                            int neox_rotary_style, int int4_kv_cache, int kv_cache_with_zeros, void* stream) {
  (void)neox_rotary_style;
  QS_REQUIRE(qkv && seq_lens && start_pos && tree_mask, "apply_bias_rope_update_kv_cache_tree: null tensor");
  return rope_append(qkv, seq_lens, padding_offset, start_pos, tree_mask, kv_pointers, batch, num_tokens, max_blocks_per_seq, head_num, kv_head_num, head_dim,
                     seq_len, tokens_per_block, size_per_token, rotary_embedding_dim, rotary_embedding_base, rotary_embedding_max_positions, int4_kv_cache,
                     kv_cache_with_zeros, stream);
}

int qs_prefix_prefill_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                                int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens, const int64_t* kv_pointers, int batch,
                                int num_tokens, int max_seqlen, int max_prefix_len, int max_blocks_per_seq, int num_heads, int num_kv_heads, int head_dim,
                                int tokens_per_block, int size_per_token, int int4_kv_cache, float softmax_scale, void* stream) {
  PrefixAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.out = out; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride; a.out_stride = out_stride;
  a.cu_seqlens = cu_seqlens; a.prefix_lens = prefix_lens; a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers);
  a.batch = batch; a.num_tokens = num_tokens; a.max_seqlen = max_seqlen; a.max_prefix_len = max_prefix_len; a.max_blocks = max_blocks_per_seq;
  a.num_heads = num_heads; a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.tokens_per_block = tokens_per_block;
  a.size_per_token = size_per_token; a.int4_kv = int4_kv_cache; a.softmax_scale = softmax_scale; a.stream = stream;
  return prefix_attention(a);
}

int qs_multi_token_decode_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                                    int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens, const int64_t* kv_pointers, int batch,
                                    int num_tokens, int max_seqlen, int max_prefix_len, int max_blocks_per_seq, int num_heads, int num_kv_heads,
                                    int head_dim, int tokens_per_block, int size_per_token, int int4_kv_cache, float softmax_scale, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  return multi_token(q, k, v, q_stride, k_stride, v_stride, out, out_stride, cu_seqlens, prefix_lens, nullptr, kv_pointers, batch, num_tokens, max_seqlen,
                     max_prefix_len, max_blocks_per_seq, num_heads, num_kv_heads, head_dim, tokens_per_block, size_per_token, int4_kv_cache, softmax_scale,
                     workspace, workspace_bytes, stream);
}
size_t qs_multi_token_attention_workspace_bytes(int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads,
                                                int int4_kv_cache) {
  return multi_token_attention_workspace_bytes(batch, num_tokens, max_seqlen, max_prefix_len, num_heads, num_kv_heads, int4_kv_cache);
}

int qs_tree_decode_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                             int64_t out_stride, const int32_t* cu_seqlens, const int32_t* prefix_lens, const int32_t* tree_mask,
                             const int64_t* kv_pointers, int batch, int num_tokens, int max_seqlen, int max_prefix_len, int max_blocks_per_seq,
                             int num_heads, int num_kv_heads, int head_dim, int tokens_per_block, int size_per_token, int int4_kv_cache,
                             float softmax_scale, void* workspace, size_t workspace_bytes, void* stream) {
  QS_REQUIRE(tree_mask, "tree_decode_attention: null tree_mask");
  return multi_token(q, k, v, q_stride, k_stride, v_stride, out, out_stride, cu_seqlens, prefix_lens, tree_mask, kv_pointers, batch, num_tokens, max_seqlen,
                     max_prefix_len, max_blocks_per_seq, num_heads, num_kv_heads, head_dim, tokens_per_block, size_per_token, int4_kv_cache, softmax_scale,
                     workspace, workspace_bytes, stream);
}

int qs_tree_accept_greedy(const int64_t* draft_tokens, const int32_t* tree_mask, const int64_t* target_tokens, int32_t* accept_len, int32_t* path,
                          int64_t* bonus, int batch, int num_nodes, void* stream) {
  return tree_accept_greedy(reinterpret_cast<const long long*>(draft_tokens), tree_mask, reinterpret_cast<const long long*>(target_tokens), accept_len,
                            path, reinterpret_cast<long long*>(bonus), batch, num_nodes, stream);
}

int qs_kv_cache_compact(const int64_t* kv_pointers, const int32_t* start_pos, const int32_t* path, const int32_t* accept_len, int num_layers, int batch,
                        int num_nodes, int max_blocks_per_seq, int num_kv_heads, int tokens_per_block, int size_per_token, int int4_kv_cache,
                        void* stream) {
  KvCompactArgs a;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.start_pos = start_pos; a.path = path; a.accept_len = accept_len;
  a.layers = num_layers; a.batch = batch; a.num_nodes = num_nodes; a.max_blocks = max_blocks_per_seq; a.num_kv_heads = num_kv_heads;
  a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.int4_kv = int4_kv_cache; a.stream = stream;
  return kv_cache_compact(a);
}

int qs_shared_prefix_decode_attention(const void* q, const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride,
                                      const int64_t* kv_pointers, const int32_t* length_per_sample, const int32_t* group_offsets,
                                      const int32_t* group_rows, const int32_t* group_pages, const int32_t* row_pages, void* out, int8_t* out_q,
                                      void* out_scale, void* out_sum, int batch, int num_heads, int num_kv_heads, int head_dim, int max_blocks_per_seq,
                                      int tokens_per_block, int size_per_token, int timestep, int rotary_embedding_dim, float rotary_base,
                                      int int4_kv_cache, int num_groups, int max_group, int max_pages, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  SharedPrefixAttnArgs s;
  DecodeAttnArgs& a = s.d;
  a.q = q; a.k = k; a.v = v; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.lengths = length_per_sample; a.out = out;
  a.q_out = out_q; a.q_scale = out_scale; a.q_sum = out_sum; a.workspace = workspace; a.workspace_bytes = workspace_bytes;
  a.batch = batch; a.num_heads = num_heads; a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.max_blocks = max_blocks_per_seq;
  a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.timestep = timestep;
  a.rotary_dim = rotary_embedding_dim; a.rotary_base = rotary_base; a.int4_kv = int4_kv_cache; a.kv_zeros = 1; a.stream = stream;
  s.group_offsets = group_offsets; s.group_rows = group_rows; s.group_pages = group_pages; s.row_pages = row_pages;
  s.num_groups = num_groups; s.max_group = max_group; s.max_pages = max_pages;
  return shared_prefix_decode_attention(s);
}
size_t qs_shared_prefix_attention_workspace_bytes(int batch, int num_heads, int num_kv_heads, int timestep, int num_groups, int max_group, int max_pages,
                                                  int int4_kv_cache) {
  return shared_prefix_attention_workspace_bytes(batch, num_heads, num_kv_heads, timestep, num_groups, max_group, max_pages, int4_kv_cache);
}

int qs_kv_cache_fork(const int64_t* kv_pointers, const int32_t* parents, const int32_t* children, const int32_t* lens, int num_layers, int batch,
                     int num_pairs, int max_blocks_per_seq, int num_kv_heads, int tokens_per_block, int size_per_token, int int4_kv_cache, void* stream) {
  KvForkArgs a;
  a.kv_pointers = reinterpret_cast<const long long*>(kv_pointers); a.parents = parents; a.children = children; a.lens = lens;
  a.layers = num_layers; a.batch = batch; a.num_pairs = num_pairs; a.max_blocks = max_blocks_per_seq; a.num_kv_heads = num_kv_heads;
  a.tokens_per_block = tokens_per_block; a.size_per_token = size_per_token; a.int4_kv = int4_kv_cache; a.stream = stream;
  return kv_cache_fork(a);
}

int qs_beam_select(const int64_t* top_ids, const float* top_logprobs, int32_t* live, float* cum, int32_t* seq_lens, int32_t* context_lens,
                   int64_t* tokens, int32_t* parents, const int32_t* prompt_lens, const int64_t* history, const float* length_penalty,
                   const int32_t* early_stopping, const int64_t* eos, const int64_t* stop_ids, int num_stops, const int32_t* budget, int32_t* done,
                   int64_t* pool_tokens, int32_t* pool_len, float* pool_cum, float* pool_score, int32_t* pool_count, int num_requests, int beam_width,
                   int max_tokens, int max_model_len, int history_len, void* stream) {
  BeamSelectArgs a;
  a.top_ids = reinterpret_cast<const long long*>(top_ids); a.top_logprobs = top_logprobs; a.live = live; a.cum = cum; a.seq_lens = seq_lens;
  a.context_lens = context_lens; a.tokens = reinterpret_cast<long long*>(tokens); a.parents = parents; a.prompt_lens = prompt_lens;
  a.history = reinterpret_cast<const long long*>(history); a.length_penalty = length_penalty; a.early_stopping = early_stopping;
  a.eos = reinterpret_cast<const long long*>(eos); a.stop_ids = reinterpret_cast<const long long*>(stop_ids); a.num_stops = num_stops;
  a.budget = budget; a.done = done; a.pool_tokens = reinterpret_cast<long long*>(pool_tokens); a.pool_len = pool_len; a.pool_cum = pool_cum;
  a.pool_score = pool_score; a.pool_count = pool_count; a.num_requests = num_requests; a.beam_width = beam_width; a.max_tokens = max_tokens;
  a.max_model_len = max_model_len; a.history_len = history_len; a.stream = stream;
  return beam_select(a);
}

int qs_beam_reorder(int64_t* kv_pointers, const int32_t* parents, const int32_t* context_lens, const int32_t* prompt_lens, const int64_t* tokens,
                    int64_t* history, int num_layers, int batch, int beam_width, int max_blocks_per_seq, int num_kv_heads, int tokens_per_block,
                    int size_per_token, int int4_kv_cache, int history_len, void* stream) {
  BeamReorderArgs a;
  a.kv_pointers = reinterpret_cast<long long*>(kv_pointers); a.parents = parents; a.context_lens = context_lens; a.prompt_lens = prompt_lens;
  a.tokens = reinterpret_cast<const long long*>(tokens); a.history = reinterpret_cast<long long*>(history); a.layers = num_layers; a.batch = batch;
  a.beam_width = beam_width; a.max_blocks = max_blocks_per_seq; a.num_kv_heads = num_kv_heads; a.tokens_per_block = tokens_per_block;
  a.size_per_token = size_per_token; a.int4_kv = int4_kv_cache; a.history_len = history_len; a.stream = stream;
  return beam_reorder(a);
}

int qs_sample_rows(int64_t* out, const void* logits, const float* temperature, const int32_t* top_k, const float* top_p, uint64_t seed,
                   int64_t* offsets, int rows, int vocab, void* stream) {
  QS_REQUIRE(logits == nullptr || aligned16(logits), "sample_rows: logits must be 16-byte aligned");
  SampleArgs a;
  a.out = reinterpret_cast<long long*>(out); a.logits = logits; a.temperature = temperature; a.top_k = top_k; a.top_p = top_p;
  a.offsets = reinterpret_cast<long long*>(offsets); a.seed = seed; a.rows = rows; a.vocab = vocab; a.stream = stream;
  return sample_rows(a);
}

int qs_tree_accept_sampling(const int64_t* draft_tokens, const int32_t* tree_mask, const void* logits, const float* draft_probs,
                            const float* temperature, const int32_t* top_k, const float* top_p, uint64_t seed, int64_t* offsets, int32_t* accept_len,
                            int32_t* path, int64_t* bonus, int batch, int num_nodes, int vocab, void* stream) {
  QS_REQUIRE(logits == nullptr || aligned16(logits), "tree_accept_sampling: logits must be 16-byte aligned");
  TreeAcceptSamplingArgs a;
  a.draft = reinterpret_cast<const long long*>(draft_tokens); a.tree_mask = tree_mask; a.logits = logits; a.draft_probs = draft_probs;
  a.temperature = temperature; a.top_k = top_k; a.top_p = top_p; a.offsets = reinterpret_cast<long long*>(offsets); a.seed = seed;
  a.accept_len = accept_len; a.path = path; a.bonus = reinterpret_cast<long long*>(bonus);
  a.batch = batch; a.num_nodes = num_nodes; a.vocab = vocab; a.stream = stream;
  return tree_accept_sampling(a);
}

int qs_apply_penalties(void* logits, const int64_t* history, const int32_t* prompt_lens, const int32_t* seq_lens, const float* repetition,
                       const float* presence, const float* frequency, int rows, int vocab, int history_len, void* stream) {
  PenaltyArgs a;
  a.logits = logits; a.history = reinterpret_cast<const long long*>(history); a.prompt_lens = prompt_lens; a.seq_lens = seq_lens;
  a.repetition = repetition; a.presence = presence; a.frequency = frequency; a.rows = rows; a.vocab = vocab; a.history_len = history_len;
  a.stream = stream;
  return apply_penalties(a);
}

int qs_logprobs_rows(float* logprob, int64_t* top_ids, float* top_logprobs, const void* logits, const int64_t* tokens, int rows, int vocab, int n,
                     void* stream) {
  QS_REQUIRE(logits == nullptr || aligned16(logits), "logprobs_rows: logits must be 16-byte aligned");
  LogprobArgs a;
  a.logprob = logprob; a.top_ids = reinterpret_cast<long long*>(top_ids); a.top_logprobs = top_logprobs; a.logits = logits;
  a.tokens = reinterpret_cast<const long long*>(tokens); a.rows = rows; a.vocab = vocab; a.n = n; a.stream = stream;
  return logprobs_rows(a);
}

int qs_ngram_propose(const int64_t* history, const int32_t* seq_lens, int64_t* tokens, int32_t* tree_mask, int batch, int history_len, int num_nodes,
                     int n_min, int n_max, int branches, void* stream) {
  NgramProposeArgs a;
  a.history = reinterpret_cast<const long long*>(history); a.seq_lens = seq_lens; a.tokens = reinterpret_cast<long long*>(tokens);
  a.tree_mask = tree_mask; a.batch = batch; a.history_len = history_len; a.num_nodes = num_nodes; a.n_min = n_min; a.n_max = n_max;
  a.branches = branches; a.stream = stream;
  return ngram_propose(a);
}

int qs_spec_commit(const int64_t* draft_tokens, const int32_t* path, const int32_t* accept_len, const int64_t* bonus, int64_t* history, int32_t* seq_lens,
                   const int32_t* prompt_lens, const int32_t* budget, const int64_t* eos, int32_t* finished, int32_t* start_pos, int32_t* context_lens,
                   int64_t* roots, int batch, int num_nodes, int history_len, void* stream) {
  SpecCommitArgs a;
  a.draft = reinterpret_cast<const long long*>(draft_tokens); a.path = path; a.accept_len = accept_len; a.bonus = reinterpret_cast<const long long*>(bonus);
  a.history = reinterpret_cast<long long*>(history); a.seq_lens = seq_lens; a.prompt_lens = prompt_lens; a.budget = budget;
  a.eos = reinterpret_cast<const long long*>(eos); a.finished = finished; a.start_pos = start_pos; a.context_lens = context_lens;
  a.roots = reinterpret_cast<long long*>(roots); a.batch = batch; a.num_nodes = num_nodes; a.history_len = history_len; a.stream = stream;
  return spec_commit(a);
}

int qs_spec_commit_stops(const int64_t* draft_tokens, const int32_t* path, const int32_t* accept_len, const int64_t* bonus, int64_t* history,
                         int32_t* seq_lens, const int32_t* prompt_lens, const int32_t* budget, const int64_t* eos, const int64_t* stop_ids,
                         int num_stops, int32_t* finished, int32_t* start_pos, int32_t* context_lens, int64_t* roots, int batch, int num_nodes,
                         int history_len, void* stream) {
  SpecCommitArgs a;
  a.draft = reinterpret_cast<const long long*>(draft_tokens); a.path = path; a.accept_len = accept_len; a.bonus = reinterpret_cast<const long long*>(bonus);
  a.history = reinterpret_cast<long long*>(history); a.seq_lens = seq_lens; a.prompt_lens = prompt_lens; a.budget = budget;
  a.eos = reinterpret_cast<const long long*>(eos); a.finished = finished; a.start_pos = start_pos; a.context_lens = context_lens;
  a.roots = reinterpret_cast<long long*>(roots); a.batch = batch; a.num_nodes = num_nodes; a.history_len = history_len; a.stream = stream;
  return spec_commit_stops(a, reinterpret_cast<const long long*>(stop_ids), num_stops);
}

int qs_apply_penalties_tree(void* logits, const int64_t* draft_tokens, const int32_t* tree_mask, const int64_t* history, const int32_t* prompt_lens,
                            const int32_t* seq_lens, const float* repetition, const float* presence, const float* frequency, int batch, int num_nodes,
                            int vocab, int history_len, void* stream) {
  PenaltyTreeArgs a;
  a.logits = logits; a.draft = reinterpret_cast<const long long*>(draft_tokens); a.tree_mask = tree_mask;
  a.history = reinterpret_cast<const long long*>(history); a.prompt_lens = prompt_lens; a.seq_lens = seq_lens; a.repetition = repetition;
  a.presence = presence; a.frequency = frequency; a.batch = batch; a.num_nodes = num_nodes; a.vocab = vocab; a.history_len = history_len;
  a.stream = stream;
  return apply_penalties_tree(a);
}

int qs_logprobs_accepted(float* logprob, int64_t* top_ids, float* top_logprobs, const void* logits, const int64_t* draft_tokens, const int32_t* path,
                         const int32_t* accept_len, const int64_t* bonus, const int32_t* seq_lens, const int32_t* finished, int batch, int num_nodes,
                         int vocab, int n, int width, void* stream) {
  QS_REQUIRE(logits == nullptr || aligned16(logits), "logprobs_accepted: logits must be 16-byte aligned");
  LogprobAcceptedArgs a;
  a.logprob = logprob; a.top_ids = reinterpret_cast<long long*>(top_ids); a.top_logprobs = top_logprobs; a.logits = logits;
  a.draft = reinterpret_cast<const long long*>(draft_tokens); a.path = path; a.accept_len = accept_len;
  a.bonus = reinterpret_cast<const long long*>(bonus); a.seq_lens = seq_lens; a.finished = finished; a.batch = batch; a.num_nodes = num_nodes;
  a.vocab = vocab; a.n = n; a.width = width; a.stream = stream;
  return logprobs_accepted(a);
}

int qs_prefill_attention(const void* q,const void* k, const void* v, int64_t q_stride, int64_t k_stride, int64_t v_stride, void* out,
                         int64_t out_stride, const int32_t* cu_seqlens, int batch, int num_tokens, int max_seqlen, int num_heads, int num_kv_heads,
                         int head_dim, float softmax_scale, void* stream) {
  PrefillAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.out = out; a.q_stride = q_stride; a.k_stride = k_stride; a.v_stride = v_stride; a.out_stride = out_stride;
  a.cu_seqlens = cu_seqlens; a.batch = batch; a.num_tokens = num_tokens; a.max_seqlen = max_seqlen; a.num_heads = num_heads;
  a.num_kv_heads = num_kv_heads; a.head_dim = head_dim; a.softmax_scale = softmax_scale; a.stream = stream;
  return prefill_attention(a);
}

int qs_compute_padding_offsets(int32_t* out, const int32_t* cu_seqlens, int batch, int max_seqlen, void* stream) {
  QS_REQUIRE(out && cu_seqlens, "compute_padding_offsets: null tensor");
  return padding_offsets(out, cu_seqlens, batch, max_seqlen, stream);
}

int qs_rms_norm(void* out, const void* input, const void* weight, float epsilon, int use_quant, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && weight, "rms_norm: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input) && aligned16(weight), "rms_norm: tensors must be 16-byte aligned");
  return rms_norm(out, input, weight, epsilon, use_quant, tokens, hidden, stream);
}

int qs_rms_norm_general(int8_t* out, const void* input, const void* weight, void* scaling, float epsilon, int use_per_token_quant, int tokens,
                        int hidden, void* stream) {
  QS_REQUIRE(out && input && weight && scaling, "rms_norm_general: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input) && aligned16(weight), "rms_norm_general: tensors must be 16-byte aligned");
  return layernorm_general_quant(out, input, weight, nullptr, scaling, epsilon, tokens, hidden, use_per_token_quant, stream);
}

int qs_rms_norm_general_fuse_sum(int8_t* out, const void* input, const void* weight, void* input_sum, void* scaling, float epsilon,
                                 int use_per_token_quant, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && weight && scaling && input_sum, "rms_norm_general_fuse_sum: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input) && aligned16(weight), "rms_norm_general_fuse_sum: tensors must be 16-byte aligned");
  return layernorm_general_quant(out, input, weight, input_sum, scaling, epsilon, tokens, hidden, use_per_token_quant, stream);
}

int qs_dequant_add_residual_rms_norm_quant(int8_t* out, const int32_t* input, void* residual, const void* gamma, const void* scale_vec,
                                           float scale, float epsilon, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && residual && gamma, "invoke_dequant_add_residual_rms_norm_quant: null tensor");
  return dequant_add_residual_rms_norm_quant(out, input, residual, gamma, scale_vec, scale, epsilon, tokens, hidden, stream);
}

int qs_invoke_quant(int8_t* out, const void* input, void* scale, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && scale, "invoke_quant: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input), "invoke_quant: tensors must be 16-byte aligned");
  return quant_per_token(out, input, nullptr, scale, tokens, hidden, stream);
}
int qs_invoke_quant_scalar(int8_t* out, const void* input, float scale, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input, "invoke_quant: null tensor");
  return quant_scalar(out, input, scale, tokens, hidden, stream);
}
int qs_invoke_quant_fuse_sum(int8_t* out, const void* input, void* input_sum, void* scale, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && scale && input_sum, "invoke_quant_fuse_sum: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input), "invoke_quant_fuse_sum: tensors must be 16-byte aligned");
  return quant_per_token(out, input, input_sum, scale, tokens, hidden, stream);
}
int qs_add_rms_norm_general_peer(int8_t* out, void* hidden_out, const void* x, const void* const* delta_ptrs, void* const* flag_ptrs, void* state, int world,
                                 int rank, int phase, const void* gamma, void* input_sum, void* scaling, float epsilon, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && hidden_out && x && delta_ptrs && flag_ptrs && state && gamma && scaling, "add_rms_norm_general_peer: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(hidden_out) && aligned16(x) && aligned16(gamma), "add_rms_norm_general_peer: tensors must be 16-byte aligned");
  return add_layernorm_quant_peer(out, hidden_out, x, delta_ptrs, flag_ptrs, state, world, rank, phase, gamma, input_sum, scaling, epsilon, tokens, hidden, stream);
}
int qs_row_absmax(float* amax_out, const void* input, int tokens, int hidden, void* stream) {
  QS_REQUIRE(amax_out && input, "row_absmax: null tensor");
  QS_REQUIRE(aligned16(input), "row_absmax: input must be 16-byte aligned");
  return row_absmax(amax_out, input, tokens, hidden, stream);
}
int qs_invoke_quant_given_amax(int8_t* out, const void* input, const float* amax, void* input_sum, void* scale, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && input && amax && scale, "invoke_quant_given_amax: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input), "invoke_quant_given_amax: tensors must be 16-byte aligned");
  return quant_given_amax(out, input, amax, input_sum, scale, tokens, hidden, stream);
}
int qs_invoke_dequant_add_residual(void* out, const int32_t* input, const void* residual, const void* scale_vec, float scale, int tokens,
                                   int hidden, void* stream) {
  QS_REQUIRE(out && input && residual, "invoke_dequant_add_residual: null tensor");
  return dequant_add_residual(out, input, residual, scale_vec, scale, tokens, hidden, stream);
}
int qs_invoke_dequant(void* out, const int32_t* input, float scale, int tokens, int hidden, int input_stride, int out_stride, void* stream) {
  QS_REQUIRE(out && input, "invoke_dequant: null tensor");
  return dequant(out, input, scale, tokens, hidden, input_stride, out_stride, stream);
}

int qs_argmax_rows(int64_t* out, const void* logits, int rows, int vocab, void* stream) {
  QS_REQUIRE(out && logits, "argmax_rows: null tensor");
  QS_REQUIRE(aligned16(logits) && (static_cast<size_t>(vocab) * 2) % 16 == 0, "argmax_rows: rows must be 16-byte aligned");
  return argmax_rows(out, logits, rows, vocab, stream);
}

int qs_silu_and_mul_quant(int8_t* out, const void* input, void* input_sum, void* scale, int tokens, int d, void* stream) {
  QS_REQUIRE(out && input && scale, "silu_and_mul_quant: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input), "silu_and_mul_quant: tensors must be 16-byte aligned");
  return silu_and_mul_quant(out, input, input_sum, scale, tokens, d, stream);
}
int qs_add_rms_norm_general(int8_t* out, void* hidden_out, const void* x, const void* delta, const void* weight, void* input_sum, void* scaling,
                            float epsilon, int tokens, int hidden, void* stream) {
  QS_REQUIRE(out && hidden_out && x && delta && weight && scaling, "add_rms_norm_general: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(hidden_out) && aligned16(x) && aligned16(delta) && aligned16(weight), "add_rms_norm_general: tensors must be 16-byte aligned");
  return add_layernorm_quant(out, hidden_out, x, delta, weight, input_sum, scaling, epsilon, tokens, hidden, stream);
}
int qs_silu_and_mul(void* out, const void* input, int tokens, int d, void* stream) {
  QS_REQUIRE(out && input, "silu_and_mul: null tensor");
  QS_REQUIRE(aligned16(out) && aligned16(input), "silu_and_mul: tensors must be 16-byte aligned");
  return silu_and_mul(out, input, tokens, d, stream);
}
int qs_gelu_new(void* out, const void* input, int tokens, int d, void* stream) {
  QS_REQUIRE(out && input, "gelu_new: null tensor");
  return gelu(out, input, tokens, d, 0, stream);
}
int qs_gelu_fast(void* out, const void* input, int tokens, int d, void* stream) {
  QS_REQUIRE(out && input, "gelu_fast: null tensor");
  return gelu(out, input, tokens, d, 1, stream);
}
int qs_dequant_silu_and_mul_quant(int8_t* out, const int32_t* input, float scale_gate, float scale_up, float scale_out, float* scale_out_vec,
                                  float* tmp, int tokens, int d, void* stream) {
  QS_REQUIRE(out && input, "invoke_dequant_silu_and_mul_quant: null tensor");
  QS_REQUIRE((scale_out_vec == nullptr) == (tmp == nullptr), "invoke_dequant_silu_and_mul_quant: scale_out and tmp must be given together");
  return dequant_silu_and_mul_quant(out, input, scale_gate, scale_up, scale_out, scale_out_vec, tmp, tokens, d, stream);
}

int qs_inflight_schedule(const qs_inflight_args* args, void* stream) {
  QS_REQUIRE(args != nullptr, "inflight_schedule: null arguments");
  return inflight_schedule(*args, stream);
}

int qs_inflight_schedule_pool(const qs_inflight_args* args, const qs_kv_pool_args* pool, void* stream) {
  QS_REQUIRE(args != nullptr && pool != nullptr, "inflight_schedule_pool: null arguments");
  return inflight_schedule_pool(*args, *pool, stream);
}

int qs_inflight_schedule_pool_cache(const qs_inflight_args* args, const qs_kv_pool_args* pool, const qs_prefix_cache_args* cache, void* stream) {
  QS_REQUIRE(args != nullptr && pool != nullptr && cache != nullptr, "inflight_schedule_pool_cache: null arguments");
  return inflight_schedule_pool_cache(*args, *pool, *cache, stream);
}

}  // extern "C"
