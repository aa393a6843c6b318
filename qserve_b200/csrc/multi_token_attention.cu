// qserve_b200 -- multi-token decode attention over the INT4 / INT8 paged KV cache (speculative-decoding verification), sm_90a.
//
// A batch of n_b <= 16 draft tokens per sequence, already rotated and appended at positions P_b .. P_b + n_b - 1 by
// apply_bias_rope_update_kv_cache_at.  Query token i of sequence b gets exactly what single_query_attention computes for it as a decode step:
// it attends to the cache positions 0 .. P_b + i - 1 dequantised from the pages (the earlier draft tokens of the step included, read back
// quantised) and to its own key / value as the un-quantised fp16 rows; its own cache slot P_b + i is not read.
//
// Design (DESIGN.md 3.6): the decode kernel of attention.cu (DESIGN.md 3.2) with the n8 column side of its mma.m16n8k16 carrying
// (draft token x query head of the GQA group) instead of query heads only.  One CTA (4 warps) owns a (KV head, column part, sequence,
// context split); column c of part cp is (token i, head h) with cp * C + c = i * G + h.  Every INT4 / INT8 code a warp unpacks feeds C = 8 * NT
// columns (NT n8 tiles), so a verify of n tokens costs about one decode launch instead of n.  Page streaming (per-warp cp.async.bulk rings),
// biased-code operands, scale folding, the online softmax in log2 units and the self-cleaning split merge are the decode kernel's
// (paged_attention.cuh); the page stream is column_tile_stream, shared with shared_prefix_attention_kernel.  The per-column causal limit
// P_b + i is applied only to the slices that hold draft tokens.  There is no RoPE and no page append here.
//
// Tree-structured drafts (TREE = true, qs_tree_decode_attention): tree_mask[tok0 + i] bit j says that node j is an ancestor of node i (bits
// >= i are ignored).  Node i attends to the prefix 0 .. P_b - 1, to the slots P_b + j of its ancestors j and to its own un-quantised key /
// value; the per-column limit becomes the column's ancestor word, tested in the same causal-tail branch.  A chain mask ((1 << i) - 1) masks
// exactly the positions >= P_b + i, so it gives the chain kernel's result bit for bit.
#include <math_constants.h>

#include "common.cuh"
#include "launch.cuh"
#include "paged_attention.cuh"

namespace qs {
namespace {

struct MultiTokenParams {
  const __half* q;                // [T, Hq * 128] rows of q_stride halfs (rotated)
  const __half* k;                // [T, Hkv * 128] (rotated)
  const __half* v;
  __half* out;                    // [T, Hq * 128] rows of out_stride halfs
  long long q_stride, k_stride, v_stride, out_stride;
  const int* cu_seqlens;          // [B + 1] draft token offsets
  const int* prefix_lens;         // [B] tokens cached before the draft tokens
  const long long* kv_pointers;   // [B, 2, max_blocks] absolute page addresses
  int num_heads, num_kv_heads, max_blocks;
  int cparts;                     // column parts per KV head
  int nsplit;                     // context splits
  PageGeom pg;
  float scale_log2;               // softmax scale * log2(e); 0: the decode kernel's rsqrt(128) * log2(e)
  float* ws_part;                 // [T, Hq, nsplit, 130] split partials (O, max, sum)
  uint32_t* ws_cnt;               // [B, gridDim.x] arrival counters (zero between launches), in the fixed counter region
  const int* tree_mask;           // TREE: [T] ancestor words of the draft nodes (read after the dependency wait)
};

template <int BITS, int NT, bool TREE>
__global__ void __launch_bounds__(kAttnConsumers, kColumnMinBlocks<NT>) multi_token_attention_kernel(const MultiTokenParams p) {
  constexpr int C = 8 * NT;  // columns per CTA
  const int G = p.num_heads / p.num_kv_heads;
  const int hk = blockIdx.x / p.cparts;
  const int col0 = (blockIdx.x - hk * p.cparts) * C;
  const int b = blockIdx.y;
  const int split = blockIdx.z;
  const int nsplit = p.nsplit;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q4 = lane & 3;

  // The draft lengths, the prefix lengths and the page table are prepared by the host before the step: read before the dependency wait
  // (INTEGRATION.md 1c).  q / k / v and the page contents are only touched after it.
  const int tok0 = p.cu_seqlens[b];
  const int n_b = p.cu_seqlens[b + 1] - tok0;
  const int P = p.prefix_lens[b];
  const int ncol = min(C, G * n_b - col0);  // columns of this CTA that carry data
  if (ncol <= 0) return;                    // uniform over the CTA and over the context splits of this (sequence, column part)

  extern __shared__ __align__(128) uint8_t smem_attn[];
  uint8_t* s_ring = smem_attn;                   // kWarps private rings
  __shared__ ColumnShared<BITS, NT> sh;
  __shared__ __align__(16) __half s_k[C * kD];   // own key and value of the token of each column
  __shared__ __align__(16) __half s_v[C * kD];
  __shared__ uint32_t s_last;

  // causal limit of this thread's S^T columns 8t + 2q4, 8t + 2q4 + 1: cache positions >= P + i are masked (columns without data: the last token's).
  // TREE: the column's ancestor word instead (bits < i of tree_mask[tok0 + i]; the same registers)
  int lim[NT][2];
  auto stage = [&] {
    // q, k, v of every column (zeros for the columns without data)
    for (int idx = threadIdx.x; idx < C * (kD / 8); idx += kAttnConsumers) {
      const int c = idx / (kD / 8), e = (idx % (kD / 8)) * 8;
      uint4 qv = make_uint4(0u, 0u, 0u, 0u), kv = qv, vv = qv;
      if (c < ncol) {
        const int i = (col0 + c) / G, h = col0 + c - i * G;
        const size_t row = static_cast<size_t>(tok0 + i);
        qv = *reinterpret_cast<const uint4*>(p.q + row * p.q_stride + static_cast<size_t>(hk * G + h) * kD + e);
        kv = *reinterpret_cast<const uint4*>(p.k + row * p.k_stride + static_cast<size_t>(hk) * kD + e);
        vv = *reinterpret_cast<const uint4*>(p.v + row * p.v_stride + static_cast<size_t>(hk) * kD + e);
      }
      *reinterpret_cast<uint4*>(sh.q + c * kD + e) = qv;
      *reinterpret_cast<uint4*>(s_k + c * kD + e) = kv;
      *reinterpret_cast<uint4*>(s_v + c * kD + e) = vv;
    }
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = min((col0 + 8 * t + 2 * q4 + u) / G, n_b - 1);
        if constexpr (TREE) {
          lim[t][u] = p.tree_mask[tok0 + i] & static_cast<int>((1u << i) - 1u);
        } else {
          lim[t][u] = P + i;
        }
      }
  };
  auto tail = [&](int t0, int tokA, float (&tl)[2][NT][4]) {
    if (t0 + 2 * kChunk > P) {  // causal tail: only the slices that hold draft tokens (or unread slots)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int tA = t0 + c * kChunk + tokA, tB = tA + 8;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          if constexpr (TREE) {
            // position P + r with r >= 0 is allowed iff bit r of the ancestor word is set (the word has no bits >= 16)
            auto blocked = [&](int r, int word) { return r >= 0 && !((static_cast<uint32_t>(word) >> min(r, 31)) & 1u); };
            if (blocked(tA - P, lim[t][0])) tl[c][t][0] = -CUDART_INF_F;
            if (blocked(tA - P, lim[t][1])) tl[c][t][1] = -CUDART_INF_F;
            if (blocked(tB - P, lim[t][0])) tl[c][t][2] = -CUDART_INF_F;
            if (blocked(tB - P, lim[t][1])) tl[c][t][3] = -CUDART_INF_F;
          } else {
            if (tA >= lim[t][0]) tl[c][t][0] = -CUDART_INF_F;
            if (tA >= lim[t][1]) tl[c][t][1] = -CUDART_INF_F;
            if (tB >= lim[t][0]) tl[c][t][2] = -CUDART_INF_F;
            if (tB >= lim[t][1]) tl[c][t][3] = -CUDART_INF_F;
          }
        }
      }
    }
  };
  const float sm_scale = p.scale_log2 > 0.f ? p.scale_log2 : rsqrtf(static_cast<float>(kD)) * 1.4426950408889634f;
  // cache tokens read by any column: the prefix and every draft token but the last (column i reads the positions < P + i)
  const int tlen = P + n_b - 1;
  auto unread = [&](int t) { return t >= tlen; };
  column_tile_stream<BITS, NT, true>(sh, s_ring, p.kv_pointers, b, p.max_blocks, p.pg, hk, (tlen + kPageTokens - 1) / kPageTokens, nsplit, sm_scale,
                                     stage, unread, tail);

  // own-token logit: fp32 dot of the rotated, un-quantised q and k of the column's token (as decode_attention_kernel's new token)
  if (split == 0) {
    for (int r = warp; r < ncol; r += kWarps) {
      const float acc = own_logit(sh.q + r * kD, s_k + r * kD, lane);
      if (lane == 0) {
        sh.m[kWarps][r] = acc * sm_scale;
        sh.l[kWarps][r] = 1.f;
      }
    }
  }
  __syncthreads();

  // ---------------- merge the warps (and the un-quantised own token) ----------------
  const int nparts = kWarps + (split == 0 ? 1 : 0);
  if (threadIdx.x < C) merge_weights<C>(threadIdx.x, nparts, nsplit, sh.m, sh.l, sh.f);
  __syncthreads();
  auto out_row = [&](int r) {  // (token row, query head) of column r
    const int i = (col0 + r) / G;
    return make_int2(tok0 + i, hk * G + col0 + r - i * G);
  };
  if (threadIdx.x < kD) {
    const int d = 16 * (threadIdx.x & 7) + (threadIdx.x >> 3);
#pragma unroll
    for (int r = 0; r < C; ++r) {
      if (r < ncol) {
        const float acc = merge_warps<BITS, C>(s_ring, r, __half2float(s_v[r * kD + d]), sh.f);
        const int2 rh = out_row(r);
        if (nsplit == 1) {
          p.out[static_cast<size_t>(rh.x) * p.out_stride + static_cast<size_t>(rh.y) * kD + d] = __float2half_rn(acc);
        } else {
          float* pr = p.ws_part + ((static_cast<size_t>(rh.x) * p.num_heads + rh.y) * nsplit + split) * (kD + 2);
          pr[d] = acc;
          if (threadIdx.x == 0) {
            pr[kD] = sh.m[0][r];
            pr[kD + 1] = sh.l[0][r];
          }
        }
      }
    }
  }
  // the last split CTA of this (sequence, KV head, column part) to arrive merges the partials in split order (deterministic)
  if (nsplit > 1 && arrive_last(p.ws_cnt + static_cast<size_t>(b) * gridDim.x + blockIdx.x, nsplit, s_last) && threadIdx.x < kD) {
    const int d = threadIdx.x;
    __threadfence();
    for (int r = 0; r < ncol; ++r) {
      const int2 rh = out_row(r);
      const float* pr = p.ws_part + (static_cast<size_t>(rh.x) * p.num_heads + rh.y) * nsplit * (kD + 2);
      p.out[static_cast<size_t>(rh.x) * p.out_stride + static_cast<size_t>(rh.y) * kD + d] = __float2half_rn(merge_splits(pr, nsplit, d));
    }
  }
}

// The split counters sit in a fixed region at the start of the workspace, so that the partials of one launch shape never overlap the
// counters of another (the workspace is reused across shapes and the counters must read zero at every launch).
constexpr size_t kCounterBytes = 16384;

// multi_token_attention_kernel<bits, ntile, tree>: the one place the plan's occupancy lookup and the launch pick it
ColumnKernel<void (*)(MultiTokenParams)> multi_token_kernel(int bits, int ntile, bool tree) {
  if (tree) {
    if (bits == 4) return ntile == 1 ? column_kernel<multi_token_attention_kernel<4, 1, true>>() : column_kernel<multi_token_attention_kernel<4, 2, true>>();
    return ntile == 1 ? column_kernel<multi_token_attention_kernel<8, 1, true>>() : column_kernel<multi_token_attention_kernel<8, 2, true>>();
  }
  if (bits == 4) return ntile == 1 ? column_kernel<multi_token_attention_kernel<4, 1, false>>() : column_kernel<multi_token_attention_kernel<4, 2, false>>();
  return ntile == 1 ? column_kernel<multi_token_attention_kernel<8, 1, false>>() : column_kernel<multi_token_attention_kernel<8, 2, false>>();
}

struct MultiTokenPlan : ColumnPlan {
  size_t part_bytes;  // split partials, after the counter region
};

// plan_columns over the (query heads of a group) x (draft tokens) columns, with context splits only while the split counters fit their region.
// Chain and tree share the plan (and the workspace size): it asks the occupancy of the chain instantiation
MultiTokenPlan plan_multi_token(int bits, int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads) {
  auto per_sm = [&](int ntile) { return multi_token_kernel(bits, ntile, false).resident(ring_bytes(bits), "multi_token_decode_attention smem attribute"); };
  MultiTokenPlan pl{plan_columns(num_heads / num_kv_heads * max_seqlen, static_cast<long long>(num_kv_heads) * batch, max_prefix_len + max_seqlen - 1, per_sm), 0};
  if (pl.ctas > static_cast<long long>(kCounterBytes / sizeof(uint32_t))) pl.nsplit = 1;
  pl.part_bytes = pl.nsplit > 1 ? static_cast<size_t>(num_tokens) * num_heads * pl.nsplit * (kD + 2) * sizeof(float) : 0;
  return pl;
}

}  // namespace

size_t multi_token_attention_workspace_bytes(int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads,
                                             int int4_kv) {
  if (batch <= 0 || num_tokens <= 0 || max_seqlen <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0) return 0;
  return kCounterBytes + plan_multi_token(int4_kv ? 4 : 8, batch, num_tokens, max_seqlen, max_prefix_len, num_heads, num_kv_heads).part_bytes;
}

int multi_token_attention(const MultiTokenAttnArgs& a) {
  const int rc = check_page_geometry("multi_token_decode_attention", a.head_dim, a.num_heads, a.num_kv_heads, a.tokens_per_block, a.size_per_token,
                                     a.int4_kv);
  if (rc) return rc;
  QS_REQUIRE(a.num_heads > 0 && a.batch >= 0 && a.num_tokens >= 0 && a.max_prefix_len >= 0, "multi_token_decode_attention: heads=%d, or negative size",
             a.num_heads);
  QS_REQUIRE(a.max_seqlen >= 1 && a.max_seqlen <= 16, "multi_token_decode_attention: max_seqlen=%d, must be 1 .. 16", a.max_seqlen);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(static_cast<long long>(a.max_prefix_len) + a.max_seqlen <= static_cast<long long>(a.max_blocks) * kPageTokens,
             "multi_token_decode_attention: max_prefix_len %d + max_seqlen %d exceed the page table (%d blocks of %d tokens)", a.max_prefix_len,
             a.max_seqlen, a.max_blocks, kPageTokens);
  if (a.batch == 0 || a.num_tokens == 0) return QS_OK;
  QS_REQUIRE(a.batch <= 65535, "multi_token_decode_attention: batch=%d exceeds the grid limit", a.batch);
  QS_REQUIRE(a.q && a.k && a.v && a.out && a.cu_seqlens && a.prefix_lens && a.kv_pointers, "multi_token_decode_attention: null pointer");
  QS_REQUIRE(a.q_stride % 8 == 0 && a.k_stride % 8 == 0 && a.v_stride % 8 == 0 && a.out_stride >= a.num_heads * kD,
             "multi_token_decode_attention: q / k / v row strides must be multiples of 8 halfs, out rows must hold Hq * 128 halfs");
  QS_REQUIRE(a.q_stride >= a.num_heads * kD && a.k_stride >= a.num_kv_heads * kD && a.v_stride >= a.num_kv_heads * kD,
             "multi_token_decode_attention: row stride smaller than the row");
  QS_REQUIRE(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v)) & 15) == 0,
             "multi_token_decode_attention: q, k, v must be 16-byte aligned");
  const MultiTokenPlan pl = plan_multi_token(bits, a.batch, a.num_tokens, a.max_seqlen, a.max_prefix_len, a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= kCounterBytes + pl.part_bytes,
             "multi_token_decode_attention: workspace of %zu bytes, need %zu (qs_multi_token_attention_workspace_bytes)", a.workspace_bytes,
             kCounterBytes + pl.part_bytes);
  const long long gx = static_cast<long long>(a.num_kv_heads) * pl.cparts;
  QS_REQUIRE(gx <= 0x7fffffffLL, "multi_token_decode_attention: grid too large");
  MultiTokenParams p{};
  p.q = static_cast<const __half*>(a.q);
  p.k = static_cast<const __half*>(a.k);
  p.v = static_cast<const __half*>(a.v);
  p.out = static_cast<__half*>(a.out);
  p.q_stride = a.q_stride; p.k_stride = a.k_stride; p.v_stride = a.v_stride; p.out_stride = a.out_stride;
  p.cu_seqlens = a.cu_seqlens;
  p.prefix_lens = a.prefix_lens;
  p.kv_pointers = a.kv_pointers;
  p.num_heads = a.num_heads;
  p.num_kv_heads = a.num_kv_heads;
  p.max_blocks = a.max_blocks;
  p.cparts = pl.cparts;
  p.nsplit = pl.nsplit;
  p.pg = PageGeom{kPageTokens, kPageTokens * a.size_per_token, a.num_kv_heads};
  p.scale_log2 = a.softmax_scale > 0.f ? a.softmax_scale * 1.4426950408889634f : 0.f;
  p.ws_cnt = static_cast<uint32_t*>(a.workspace);
  p.ws_part = pl.nsplit > 1 ? reinterpret_cast<float*>(static_cast<uint8_t*>(a.workspace) + kCounterBytes) : nullptr;
  p.tree_mask = a.tree_mask;
  const dim3 grid(static_cast<unsigned>(gx), a.batch, pl.nsplit);
  const size_t smem = ring_bytes(bits);
  const auto kern = multi_token_kernel(bits, pl.ntile, a.tree_mask != nullptr).fn;
  if (const int err = raise_smem_limit(kern, smem, "multi_token_decode_attention smem attribute")) return err;
  return launch(kern, grid, dim3(kAttnConsumers), smem, 0, a.stream, "multi_token_decode_attention", p);
}

}  // namespace qs
