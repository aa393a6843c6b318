// qserve_b200 -- what the two causal prompt-attention kernels share: prefill_attention_kernel (prefill_attention.cu, DESIGN.md 3.4) and
// prefix_attention_kernel (prefix_attention.cu, DESIGN.md 3.5).  Both run one CTA per (sequence, query head, block of 128 query rows) with a
// Q tile and a two-deep K / V ring in shared memory, and the same two consumer warpgroups; they differ in the producer that fills the ring and
// in the per-block key mask they hand to the consumer.  Everything here is internal to the translation unit that includes it.
#pragma once

#include <math_constants.h>

#include "common.cuh"

namespace qs {
namespace {

constexpr int kD = 128;         // head dim
constexpr int kBQ = 128;        // query rows per CTA (two consumer warpgroups x m64)
constexpr int kBKV = 128;       // keys per block (N of S, K extent of PV)
constexpr int kStages = 2;      // K / V ring depth
constexpr int kTileBytes = kBQ * kD * 2;      // 32 KB: two swizzled [128 rows x 64 halfs] sub-tiles
constexpr int kSubBytes = kTileBytes / 2;     // 16 KB
constexpr int kOffQ = 0, kOffK = kTileBytes, kOffV = kOffK + kStages * kTileBytes, kOffBar = kOffV + kStages * kTileBytes;
constexpr int kSmemBytes = kOffBar + 128;

// The mbarriers at kOffBar
struct RingBarriers {
  uint64_t* q;      // Q tile landed
  uint64_t* kfull;  // [kStages] K block ready
  uint64_t* kfree;  // [kStages] S = Q K^T retired in all eight consumer warps
  uint64_t* vfull;  // [kStages] V block ready
  uint64_t* vfree;  // [kStages] O += P V retired in all eight consumer warps
};
__device__ __forceinline__ RingBarriers ring_barriers(uint8_t* smem) {
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  return RingBarriers{bar, bar + 1, bar + 1 + kStages, bar + 1 + 2 * kStages, bar + 1 + 3 * kStages};
}
// Thread 0: prefetch the three tensor maps and initialise the barriers; a K / V block is ready after `fill_arrivals` arrivals (and the bytes
// the producer announces with mbar_expect_tx).
__device__ __forceinline__ void init_ring(const RingBarriers& bar, uint32_t fill_arrivals, const CUtensorMap* tmap_q, const CUtensorMap* tmap_k,
                                          const CUtensorMap* tmap_v) {
  tma_prefetch_desc(tmap_q);
  tma_prefetch_desc(tmap_k);
  tma_prefetch_desc(tmap_v);
  mbar_init(bar.q, 1);
  for (int i = 0; i < kStages; ++i) {
    mbar_init(&bar.kfull[i], fill_arrivals);
    mbar_init(&bar.kfree[i], 8);
    mbar_init(&bar.vfull[i], fill_arrivals);
    mbar_init(&bar.vfree[i], 8);
  }
  fence_barrier_init();
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b, float& sum) {
  const __half2 h2 = __floats2half2_rn(a, b);
  // the row sum is taken over the ROUNDED probabilities: numerator (the MMA sees fp16 P) and denominator then agree
  const float2 f = __half22float2(h2);
  sum += f.x + f.y;
  return *reinterpret_cast<const uint32_t*>(&h2);
}

// Key block j as the consumer masks it: key k (kbase <= k < kbase + 128) is visible to row a iff !masked || k <= lim_a, likewise row b.
struct BlockMask {
  bool masked;
  int kbase, lim_a, lim_b;
};

// One of the two consumer warpgroups; consumer warp cw (0 .. 7) of the CTA.  Warpgroup cw / 4 owns query rows [64 g, 64 g + 64) of query
// block qb.  Per key block j = 0 .. n_kb - 1 of the ring:
//     S = Q K^T      8 x wgmma m64n128k16, both operands K-major in shared memory (128-byte swizzle), fp32 accumulators in registers
//     mask           block_mask(j, q_pos_a, q_pos_b) -> BlockMask; masked keys are set to -inf
//     softmax        online, in the accumulator fragment (a row lives in the four threads of a quad): running max / sum in the log2 domain,
//                    P = exp2(..) rounded to fp16 and re-packed in registers as the A operand of the next MMA
//     O += P V       8 x wgmma m64n128k16, A = P from registers, B = the V tile as [key][dim] rows (an MN-major operand, transposed B)
// Then O / l is written as fp16 to rows seq_start + q_pos of `out` (rows of out_stride halfs), head h; rows q_pos >= seq_len are skipped.
// The first key of every block must be visible to every row, so that the running maxima are finite from block 0 on.
template <typename Mask>
__device__ __forceinline__ void consume(uint8_t* smem, int cw, int lane, int qb, int n_kb, float scale_log2, __half* out, long long out_stride,
                                        int seq_start, int seq_len, int h, Mask block_mask) {
  const uint8_t* s_q = smem + kOffQ;
  const uint8_t* s_k = smem + kOffK;
  const uint8_t* s_v = smem + kOffV;
  const RingBarriers bar = ring_barriers(smem);
  const int g = cw >> 2;
  const int row_a = g * 64 + (cw & 3) * 16 + (lane >> 2);  // this thread's two rows: row_a and row_a + 8
  const int q_pos_a = qb * kBQ + row_a, q_pos_b = q_pos_a + 8;
  const int col0 = (lane & 3) * 2;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_a = -CUDART_INF_F, m_b = -CUDART_INF_F;  // running maxima (log2 domain, scaled)
  float l_a = 0.f, l_b = 0.f;                      // this thread's share of the row sums
  mbar_wait(bar.q, 0);
  for (int j = 0; j < n_kb; ++j) {
    const int st = j % kStages;
    const uint32_t ph = static_cast<uint32_t>(j / kStages) & 1u;
    const uint8_t* sk = s_k + st * kTileBytes;
    const uint8_t* sv = s_v + st * kTileBytes;
    mbar_wait(&bar.kfull[st], ph);
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kD / 16; ++ks) {
      const uint32_t off = (ks >> 2) * kSubBytes;
      const uint64_t adesc = gmma_desc_sw128(smem_u32(s_q + off + g * 64 * 128)) + (ks & 3) * 2;
      const uint64_t bdesc = gmma_desc_sw128(smem_u32(sk + off)) + (ks & 3) * 2;
      wgmma_f16_ss_n128(s, adesc, bdesc, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar.kfree[st]);

    // ---- mask and row maxima ----
    const BlockMask bm = block_mask(j, q_pos_a, q_pos_b);
    float mx_a = -CUDART_INF_F, mx_b = -CUDART_INF_F;
#pragma unroll
    for (int c = 0; c < kBKV / 8; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = bm.kbase + c * 8 + col0 + (e & 1);
        float& v = s[c * 4 + e];
        if (e < 2) {
          if (bm.masked && key > bm.lim_a) v = -CUDART_INF_F;  // -inf: exp2 turns it into an exact 0
          mx_a = fmaxf(mx_a, v);
        } else {
          if (bm.masked && key > bm.lim_b) v = -CUDART_INF_F;
          mx_b = fmaxf(mx_b, v);
        }
      }
#pragma unroll
    for (int sh = 1; sh <= 2; sh <<= 1) {
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, sh));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, sh));
    }
    const float mn_a = fmaxf(m_a, mx_a * scale_log2), mn_b = fmaxf(m_b, mx_b * scale_log2);
    const float alpha_a = ex2_approx(m_a - mn_a), alpha_b = ex2_approx(m_b - mn_b);  // 0 on the first block (m = -inf)
    m_a = mn_a;
    m_b = mn_b;
    l_a *= alpha_a;
    l_b *= alpha_b;
#pragma unroll
    for (int c = 0; c < kD / 8; ++c) {
      o[c * 4 + 0] *= alpha_a; o[c * 4 + 1] *= alpha_a;
      o[c * 4 + 2] *= alpha_b; o[c * 4 + 3] *= alpha_b;
    }
    // ---- P = exp2(s * scale - m), fp16, as wgmma A fragments: 16 keys (two accumulator column groups) per fragment ----
    uint32_t pa[kBKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float* sc = s + (2 * kk + hf) * 4;
        pa[kk][2 * hf + 0] = pack_half2(ex2_approx(fmaf(sc[0], scale_log2, -m_a)), ex2_approx(fmaf(sc[1], scale_log2, -m_a)), l_a);
        pa[kk][2 * hf + 1] = pack_half2(ex2_approx(fmaf(sc[2], scale_log2, -m_b)), ex2_approx(fmaf(sc[3], scale_log2, -m_b)), l_b);
      }
    mbar_wait(&bar.vfull[st], ph);
    wgmma_fence();
    // O += P V: B = V rows [key][dim] = MN-major, 16 keys (2 KB of each 64-dim sub-tile) per instruction, the second sub-tile 16 KB on
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk) wgmma_f16_rs_n128_tb(o, pa[kk], gmma_desc_sw128(smem_u32(sv + kk * 2048), kSubBytes));
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar.vfree[st]);
  }
  // ---- epilogue: O / l -> fp16 ----
#pragma unroll
  for (int sh = 1; sh <= 2; sh <<= 1) {
    l_a += __shfl_xor_sync(0xffffffffu, l_a, sh);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, sh);
  }
  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
  __half* dst_a = out + static_cast<long long>(seq_start + q_pos_a) * out_stride + h * kD + col0;
  __half* dst_b = dst_a + 8 * out_stride;
  const bool valid_a = q_pos_a < seq_len, valid_b = q_pos_b < seq_len;
#pragma unroll
  for (int c = 0; c < kD / 8; ++c) {
    if (valid_a) *reinterpret_cast<__half2*>(dst_a + c * 8) = __floats2half2_rn(o[c * 4 + 0] * inv_a, o[c * 4 + 1] * inv_a);
    if (valid_b) *reinterpret_cast<__half2*>(dst_b + c * 8) = __floats2half2_rn(o[c * 4 + 2] * inv_b, o[c * 4 + 3] * inv_b);
  }
}

// Host: the checks prefill_attention and prefix_prefill_attention share (error messages start with `op`), and the q / k / v tensor maps.
// *empty = true: nothing to launch.
template <typename Args>
int prompt_attention_prepare(const Args& a, const char* op, bool* empty, CUtensorMap* tq, CUtensorMap* tk, CUtensorMap* tv) {
  QS_REQUIRE(a.head_dim == kD, "%s: head_dim=%d (only 128 is built, as in the reference)", op, a.head_dim);
  QS_REQUIRE(a.num_heads > 0 && a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "%s: heads=%d kv_heads=%d", op, a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.batch >= 0 && a.num_tokens >= 0 && a.max_seqlen >= 0, "%s: negative size", op);
  *empty = a.batch == 0 || a.num_tokens == 0 || a.max_seqlen == 0;
  if (*empty) return QS_OK;
  QS_REQUIRE(a.batch <= 65535 && a.num_heads <= 65535, "%s: batch=%d / heads=%d exceed the grid limits", op, a.batch, a.num_heads);
  QS_REQUIRE(a.q && a.k && a.v && a.out && a.cu_seqlens, "%s: null pointer", op);
  QS_REQUIRE(a.q_stride % 8 == 0 && a.k_stride % 8 == 0 && a.v_stride % 8 == 0 && a.out_stride % 8 == 0, "%s: row strides must be multiples of 8 halfs",
             op);
  QS_REQUIRE(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) | reinterpret_cast<uintptr_t>(a.out)) & 15) == 0,
             "%s: q, k, v, out must be 16-byte aligned", op);
  QS_REQUIRE(a.q_stride >= a.num_heads * kD && a.k_stride >= a.num_kv_heads * kD && a.v_stride >= a.num_kv_heads * kD && a.out_stride >= a.num_heads * kD,
             "%s: row stride smaller than the row", op);
  int rc = make_tmap_f16(tq, a.q, a.num_tokens, static_cast<uint64_t>(a.num_heads) * kD, a.q_stride);
  if (rc) return rc;
  rc = make_tmap_f16(tk, a.k, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.k_stride);
  if (rc) return rc;
  return make_tmap_f16(tv, a.v, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.v_stride);
}

}  // namespace
}  // namespace qs
