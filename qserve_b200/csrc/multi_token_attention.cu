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
// (paged_attention.cuh); the per-column causal limit P_b + i is applied only to the slices that hold draft tokens.  There is no RoPE and no
// page append here.
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

// Resident CTAs per SM the register budget is sized for: ptxas needs 134 / 146 (KV4 / KV8) registers for one n8 tile and 211 / 241 for two
// without spilling (the O^T accumulators alone are 32 fp32 registers per tile), so 3 and 2 CTAs of 128 threads.  Shared memory can lower it
// further (KV8, one tile: 2); the host asks the occupancy calculator.
template <int NT>
constexpr int kMinBlocks = NT == 1 ? 3 : 2;

template <int BITS, int NT, bool TREE>
__global__ void __launch_bounds__(kAttnConsumers, kMinBlocks<NT>) multi_token_attention_kernel(const MultiTokenParams p) {
  using SL = StageLayout<BITS>;
  constexpr int R = SL::kStages;
  constexpr int C = 8 * NT;  // columns per CTA
  static_assert(SL::kWarpBytes >= C * kOStride * 4, "the per-warp ring must hold the warp's partial output");
  const int G = p.num_heads / p.num_kv_heads;
  const int hk = blockIdx.x / p.cparts;
  const int col0 = (blockIdx.x - hk * p.cparts) * C;
  const int b = blockIdx.y;
  const int split = blockIdx.z;
  const int nsplit = p.nsplit;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, q4 = lane & 3;

  // The draft lengths, the prefix lengths and the page table are prepared by the host before the step: read before the dependency wait
  // (INTEGRATION.md 1c).  q / k / v and the page contents are only touched after it.
  const int tok0 = p.cu_seqlens[b];
  const int n_b = p.cu_seqlens[b + 1] - tok0;
  const int P = p.prefix_lens[b];
  const int ncol = min(C, G * n_b - col0);  // columns of this CTA that carry data
  if (ncol <= 0) return;                    // uniform over the CTA and over the context splits of this (sequence, column part)

  extern __shared__ __align__(128) uint8_t smem_attn[];
  uint8_t* s_ring = smem_attn;                                           // kWarps private rings of R slices
  __shared__ __align__(16) __half s_q[C * kD];
  __shared__ __align__(16) __half s_k[C * kD];                           // own key and value of the token of each column
  __shared__ __align__(16) __half s_v[C * kD];
  __shared__ uint4 s_qb[NT][4][32];                                      // Q B fragments, see below
  __shared__ float s_m[kWarps + 1][C], s_l[kWarps + 1][C];
  __shared__ float s_f[kWarps + 1][C];                                   // merge weights exp2(m_w - M) [* 1 / L]
  __shared__ float2 s_meta[kWarps][2][kSliceTokens];                     // per token (scale, c) of the slice in flight
  __shared__ __align__(8) uint64_t s_full[kWarps][R];
  __shared__ uint32_t s_last;

  if (lane == 0) {
    for (int i = 0; i < R; ++i) mbar_init(&s_full[warp][i], 1);
    fence_barrier_init();
  }
  __syncwarp();
  if (threadIdx.x == 0) pdl_launch_dependents();

  // cache tokens read by any column: the prefix and every draft token but the last (column i reads the positions < P + i)
  const int tlen = P + n_b - 1;
  const long long* kptrs = p.kv_pointers + (static_cast<size_t>(b) * 2 + 0) * p.max_blocks;
  const long long* vptrs = p.kv_pointers + (static_cast<size_t>(b) * 2 + 1) * p.max_blocks;
  const int n_pages = (tlen + kPageTokens - 1) / kPageTokens;
  const int pps = (n_pages + nsplit - 1) / nsplit;
  const int p_begin = split * pps, p_end = min(n_pages, p_begin + pps);

  // ---- this warp's stream: token slice [32 (warp & 1), +32) of the pages p_begin + (warp >> 1), +2, ... (as in decode_attention_kernel) ----
  const int hslice = warp & 1;
  const int my_first = p_begin + (warp >> 1);
  const int n_my = (p_end > my_first) ? (p_end - my_first + 1) / 2 : 0;
  uint8_t* my_ring = s_ring + warp * SL::kWarpBytes;
  uint64_t* my_full = &s_full[warp][0];
  const int zoff = p.pg.num_kv_heads * p.pg.tokens_per_block * 2;
  long long kp_l = 0, vp_l = 0;  // lane l: page pointers of this warp's slice (batch * 32 + l)
  auto load_ptr_batch = [&](int j0) { slice_ptrs(kptrs, vptrs, my_first + 2 * (j0 + lane), p_end, kp_l, vp_l); };
  auto issue = [&](int j, int slot) {
    issue_slice<BITS>(lane, kp_l, vp_l, j, my_ring + slot * SL::kBytes, &my_full[slot], hk, hslice, p.pg.code_bytes, zoff);
  };
  load_ptr_batch(0);
  pdl_wait();
  for (int j = 0; j < R && j < n_my; ++j) issue(j, j);  // the cache stream starts before the staging below

  // ---- stage q, k, v of every column (zeros for the columns without data) ----
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
    *reinterpret_cast<uint4*>(s_q + c * kD + e) = qv;
    *reinterpret_cast<uint4*>(s_k + c * kD + e) = kv;
    *reinterpret_cast<uint4*>(s_v + c * kD + e) = vv;
  }
  __syncthreads();

  // causal limit of this thread's S^T columns 8t + 2q4, 8t + 2q4 + 1: cache positions >= P + i are masked (columns without data: the last token's).
  // TREE: the column's ancestor word instead (bits < i of tree_mask[tok0 + i]; the same registers)
  int lim[NT][2];
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

  // ---- Q as the MMA "B" operand per n8 tile (q_operand).  The B fragments live in shared memory (s_qb[t][w][lane] = the two k-steps of
  //      word w), not in registers: with NT = 2 the O^T accumulators alone take 64 registers, and 32 more for Q would spill ----
  float sumq[NT][2], biasq[NT][2];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    uint32_t qb0[8], qb1[8];
    q_operand<BITS>(s_q + (8 * t + g) * kD + 32 * q4, q4, qb0, qb1, sumq[t], biasq[t]);
    if (warp == 0) {
#pragma unroll
      for (int w = 0; w < 4; ++w) s_qb[t][w][lane] = make_uint4(qb0[2 * w], qb1[2 * w], qb0[2 * w + 1], qb1[2 * w + 1]);
    }
  }
  __syncthreads();
  auto qb = [&](int t, int ks, uint32_t& b0, uint32_t& b1) {
    const uint4 qq = s_qb[t][ks >> 1][lane];
    b0 = (ks & 1) ? qq.z : qq.x;
    b1 = (ks & 1) ? qq.w : qq.y;
  };

  const float sm_scale = p.scale_log2 > 0.f ? p.scale_log2 : rsqrtf(static_cast<float>(kD)) * 1.4426950408889634f;
  float o[NT][8][4];
  float m[NT][2], l[NT][2], cr[NT][2], spa[NT][4];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
#pragma unroll
    for (int i = 0; i < 8; ++i) o[t][i][0] = o[t][i][1] = o[t][i][2] = o[t][i][3] = 0.f;
    m[t][0] = m[t][1] = -CUDART_INF_F;
    l[t][0] = l[t][1] = cr[t][0] = cr[t][1] = 0.f;
    spa[t][0] = spa[t][1] = spa[t][2] = spa[t][3] = 0.f;
  }

  const int tokA = (g & 1) * 4 + (g >> 1);
  constexpr int kRow = kD * BITS / 8;
  const int hbase = hslice * kSliceTokens;
  int s = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_my; ++j) {
    const int pidx = my_first + 2 * j;
    mbar_wait(&my_full[s], ph);
    const uint8_t* st = my_ring + s * SL::kBytes;
    const int t0 = pidx * kPageTokens + hbase;
    if (t0 < tlen) {
      slice_meta<BITS>(st, lane, t0 + lane >= tlen, sm_scale, s_meta[warp][0], s_meta[warp][1]);
      __syncwarp();
      // ---- S^T (2 x 16 tokens x C columns) ----
      float sc[2][NT][4];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
#pragma unroll
        for (int t = 0; t < NT; ++t) sc[c][t][0] = sc[c][t][1] = sc[c][t][2] = sc[c][t][3] = 0.f;
        qk_chunk<BITS, NT>(st + SL::kOffK + (c * kChunk + tokA) * kRow, q4, sc[c], qb);
      }
      float tl[2][NT][4], vs[2][2], vc[2][2];
#pragma unroll
      for (int c = 0; c < 2; ++c) chunk_logits<NT>(s_meta[warp][0], s_meta[warp][1], c, tokA, sc[c], biasq, sumq, tl[c], vs[c], vc[c]);
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
      uint32_t bp[2][NT][2];
#pragma unroll
      for (int t = 0; t < NT; ++t) softmax_tile<NT, true>(t, tl, vs, vc, m[t], l[t], cr[t], spa[t], o[t], bp);
      // ---- O^T += V^T P'^T ----
#pragma unroll
      for (int c = 0; c < 2; ++c) pv_chunk<BITS, NT>(st + SL::kOffV + (c * kChunk + q4) * kRow, g, o, bp[c]);
    }
    __syncwarp();
    if (j + R < n_my) {
      if (((j + R) & 31) == 0) load_ptr_batch(j + R);
      issue(j + R, s);
    }
    if (++s == R) { s = 0; ph ^= 1; }
  }

  // ---- per-warp partials -> the warp's own (drained) ring ----
#pragma unroll
  for (int t = 0; t < NT; ++t) reduce_tile_sums(l[t], cr[t]);
  if (g == 0) {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      s_m[warp][8 * t + 2 * q4] = m[t][0]; s_m[warp][8 * t + 2 * q4 + 1] = m[t][1];
      s_l[warp][8 * t + 2 * q4] = l[t][0]; s_l[warp][8 * t + 2 * q4 + 1] = l[t][1];
    }
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < NT; ++t) store_partial<BITS>(reinterpret_cast<float*>(my_ring) + (8 * t + 2 * q4) * kOStride + g, o[t], spa[t], cr[t]);
  // own-token logit: fp32 dot of the rotated, un-quantised q and k of the column's token (as decode_attention_kernel's new token)
  if (split == 0) {
    for (int r = warp; r < ncol; r += kWarps) {
      const float acc = own_logit(s_q + r * kD, s_k + r * kD, lane);
      if (lane == 0) {
        s_m[kWarps][r] = acc * sm_scale;
        s_l[kWarps][r] = 1.f;
      }
    }
  }
  __syncthreads();

  // ---------------- merge the warps (and the un-quantised own token) ----------------
  const int nparts = kWarps + (split == 0 ? 1 : 0);
  if (threadIdx.x < C) merge_weights<C>(threadIdx.x, nparts, nsplit, s_m, s_l, s_f);
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
        const float acc = merge_warps<BITS, C>(s_ring, r, __half2float(s_v[r * kD + d]), s_f);
        const int2 rh = out_row(r);
        if (nsplit == 1) {
          p.out[static_cast<size_t>(rh.x) * p.out_stride + static_cast<size_t>(rh.y) * kD + d] = __float2half_rn(acc);
        } else {
          float* pr = p.ws_part + ((static_cast<size_t>(rh.x) * p.num_heads + rh.y) * nsplit + split) * (kD + 2);
          pr[d] = acc;
          if (threadIdx.x == 0) {
            pr[kD] = s_m[0][r];
            pr[kD + 1] = s_l[0][r];
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

constexpr int kMaxSplits = 32;
// The split counters sit in a fixed region at the start of the workspace, so that the partials of one launch shape never overlap the
// counters of another (the workspace is reused across shapes and the counters must read zero at every launch).
constexpr size_t kCounterBytes = 16384;

struct MultiTokenPlan {
  int ntile;    // n8 tiles per CTA (C = 8 * ntile columns)
  int cparts;   // column parts per KV head
  int nsplit;   // context splits
  size_t cnt_bytes, part_bytes;
};

// Launch shape: C = 8 columns when the (query heads of a group) x (draft tokens) fit one n8 tile, else 16; context splits as
// decode_attention() chooses them (enough CTAs to fill the resident slots, at most one split per 256 cached tokens, at most 32).
template <int BITS, int NT>
int resident_ctas() {
  // kernel attribute (the KV8 ring exceeds the default 48 KB of dynamic shared memory) and occupancy, once per device
  static int cached[kMaxDevices] = {};
  int& r = cached[device_ordinal()];
  if (r == 0) {
    const int smem = kWarps * StageLayout<BITS>::kWarpBytes;
    int n = 0;
    if (raise_smem_limit(multi_token_attention_kernel<BITS, NT, false>, smem, "multi_token_decode_attention smem attribute") != QS_OK ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, multi_token_attention_kernel<BITS, NT, false>, kAttnConsumers, smem) != cudaSuccess || n < 1) {
      cudaGetLastError();
      n = 1;
    }
    r = n;
  }
  return r;
}

MultiTokenPlan plan_multi_token(int bits, int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads) {
  MultiTokenPlan pl{};
  const int G = num_heads / num_kv_heads;
  const int cols = G * max_seqlen;
  pl.ntile = cols <= 8 ? 1 : 2;
  pl.cparts = (cols + 8 * pl.ntile - 1) / (8 * pl.ntile);
  const int ctx = max_prefix_len + max_seqlen - 1;
  const long long ctas = static_cast<long long>(num_kv_heads) * pl.cparts * batch;
  const int per_sm = bits == 4 ? (pl.ntile == 1 ? resident_ctas<4, 1>() : resident_ctas<4, 2>())
                                : (pl.ntile == 1 ? resident_ctas<8, 1>() : resident_ctas<8, 2>());
  const long long slots = static_cast<long long>(num_sms()) * per_sm;
  pl.nsplit = 1;
  if (2 * ctas <= slots && ctx > 512 && ctas <= static_cast<long long>(kCounterBytes / sizeof(uint32_t))) {
    pl.nsplit = static_cast<int>((slots + ctas - 1) / ctas);
    pl.nsplit = min(pl.nsplit, (ctx + 255) / 256);
    pl.nsplit = min(pl.nsplit, kMaxSplits);
  }
  pl.cnt_bytes = kCounterBytes;
  pl.part_bytes = pl.nsplit > 1 ? static_cast<size_t>(num_tokens) * num_heads * pl.nsplit * (kD + 2) * sizeof(float) : 0;
  return pl;
}

}  // namespace

size_t multi_token_attention_workspace_bytes(int batch, int num_tokens, int max_seqlen, int max_prefix_len, int num_heads, int num_kv_heads,
                                             int int4_kv) {
  if (batch <= 0 || num_tokens <= 0 || max_seqlen <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0) return 0;
  const MultiTokenPlan pl = plan_multi_token(int4_kv ? 4 : 8, batch, num_tokens, max_seqlen, max_prefix_len, num_heads, num_kv_heads);
  return pl.cnt_bytes + pl.part_bytes;
}

int multi_token_attention(const MultiTokenAttnArgs& a) {
  QS_REQUIRE(a.head_dim == kD, "multi_token_decode_attention: head_dim=%d (only 128 is built)", a.head_dim);
  QS_REQUIRE(a.num_heads > 0 && a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "multi_token_decode_attention: heads=%d kv_heads=%d",
             a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.batch >= 0 && a.num_tokens >= 0 && a.max_prefix_len >= 0, "multi_token_decode_attention: negative size");
  QS_REQUIRE(a.max_seqlen >= 1 && a.max_seqlen <= 16, "multi_token_decode_attention: max_seqlen=%d, must be 1 .. 16", a.max_seqlen);
  QS_REQUIRE(a.tokens_per_block == kPageTokens, "multi_token_decode_attention: tokens_per_block=%d, only 64 is supported", a.tokens_per_block);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * kD * bits / 8, "multi_token_decode_attention: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
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
  QS_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= pl.cnt_bytes + pl.part_bytes,
             "multi_token_decode_attention: workspace of %zu bytes, need %zu (qs_multi_token_attention_workspace_bytes)", a.workspace_bytes,
             pl.cnt_bytes + pl.part_bytes);
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
  p.ws_part = pl.nsplit > 1 ? reinterpret_cast<float*>(static_cast<uint8_t*>(a.workspace) + pl.cnt_bytes) : nullptr;
  p.tree_mask = a.tree_mask;
  const dim3 grid(static_cast<unsigned>(gx), a.batch, pl.nsplit);
  auto run = [&](auto kern, size_t smem) {
    const int rc = raise_smem_limit(kern, smem, "multi_token_decode_attention smem attribute");
    if (rc) return rc;
    return launch(kern, grid, dim3(kAttnConsumers), smem, 0, a.stream, "multi_token_decode_attention", p);
  };
  const size_t smem4 = static_cast<size_t>(kWarps) * StageLayout<4>::kWarpBytes, smem8 = static_cast<size_t>(kWarps) * StageLayout<8>::kWarpBytes;
  if (a.tree_mask) {
    if (a.int4_kv) return pl.ntile == 1 ? run(multi_token_attention_kernel<4, 1, true>, smem4) : run(multi_token_attention_kernel<4, 2, true>, smem4);
    return pl.ntile == 1 ? run(multi_token_attention_kernel<8, 1, true>, smem8) : run(multi_token_attention_kernel<8, 2, true>, smem8);
  }
  if (a.int4_kv) return pl.ntile == 1 ? run(multi_token_attention_kernel<4, 1, false>, smem4) : run(multi_token_attention_kernel<4, 2, false>, smem4);
  return pl.ntile == 1 ? run(multi_token_attention_kernel<8, 1, false>, smem8) : run(multi_token_attention_kernel<8, 2, false>, smem8);
}

}  // namespace qs
