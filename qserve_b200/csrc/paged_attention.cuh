// qserve_b200 -- device helpers shared by the attention kernels that stream the INT4 / INT8 paged KV cache through per-warp bulk-copy rings
// and multiply "biased" code operands with mma.sync m16n8k16: decode_attention_kernel (attention.cu, DESIGN.md 3.2) and
// multi_token_attention_kernel (multi_token_attention.cu, DESIGN.md 3.6).  Everything here is internal to the translation unit that
// includes it.
#pragma once

#include <math_constants.h>

#include "common.cuh"

namespace qs {
namespace {

constexpr int kD = 128;          // head dim (the reference only instantiates Dh = 128, decoderMaskedMultiheadAttention.cu:352-354)
constexpr int kWarps = 4;
constexpr int kChunk = 16;       // tokens per warp iteration
constexpr int kMaxG = 8;         // query heads per CTA (rows of the m16 tile that carry data)

struct PageGeom {
  int tokens_per_block;   // 64
  int code_bytes;         // tokens_per_block * size_per_token = bytes of codes per page (mBytesPerSeq)
  int num_kv_heads;
};

// ---- fp16 helpers ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t x, uint32_t mask, uint32_t orv) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(x), "r"(mask), "r"(orv));  // (x & mask) | orv
  return d;
}
__device__ __forceinline__ uint32_t pack_f2h2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
constexpr uint32_t kMagic = 0x64006400u;      // half2(1024, 1024)
constexpr uint32_t kOnesH2 = 0x3c003c00u;     // half2(1, 1)

constexpr int kAttnConsumers = 128;
constexpr int kPageTokens = 64;
constexpr int kOStride = kD + 4;  // floats per (warp, head) row of the merge buffer

// One stage = the 32-token slice of one 64-token page of one kv head that a warp consumes in one iteration:
// K codes | V codes | K scales | K zeros | V scales | V zeros.  Each warp owns a private ring of kStages such slices, filled by
// its lane 0 with six cp.async.bulk copies and guarded by one "full" mbarrier per slot (the refill of a slot is issued by the
// same warp right after it has consumed it, so no "empty" barrier and no producer warp are needed).
constexpr int kSliceTokens = 32;
template <int BITS>
struct StageLayout {
  static constexpr int kCodes = kPageTokens * kD * BITS / 8;       // bytes of K (or V) codes of one head-page
  static constexpr int kSliceCodes = kSliceTokens * kD * BITS / 8;  // ... of one 32-token slice
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kSliceCodes;
  static constexpr int kOffKs = 2 * kSliceCodes;   // fp16 [32]
  static constexpr int kOffKz = kOffKs + 64;
  static constexpr int kOffVs = kOffKz + 64;
  static constexpr int kOffVz = kOffVs + 64;
  static constexpr int kBytes = kOffVz + 64;
  static constexpr int kStages = 2;
  static constexpr int kWarpBytes = kStages * kBytes;  // private ring of one warp (also holds its partial O^T at the end)
  static_assert(kWarpBytes >= kMaxG * kOStride * 4, "the per-warp ring must hold the warp's partial output");
};

// full m16n8k16: all four A registers and all four accumulators carry data
__device__ __forceinline__ void mma_full(float& c0, float& c1, float& c2, float& c3, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// 8x8 b16 transpose across the warp: thread t holds (row t/4, cols 2(t%4), 2(t%4)+1) before and after
__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t x) {
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(x));
  return d;
}

// =========================================================================================================================================
// Pieces of the paged-attention main loop shared by decode_attention_kernel and multi_token_attention_kernel.  Both kernels are 4 warps; the
// S^T / O^T tiles have the cache tokens on the m16 side and NT n8 tiles of "columns" (query heads, or draft token x query head) on the n side:
// thread (g = lane / 4, q4 = lane % 4) holds columns 8t + 2q4, 8t + 2q4 + 1 of tile t.  See DESIGN.md 3.2 for the arithmetic.
// =========================================================================================================================================

// ---- page streaming: warp w consumes the 32-token slice (w & 1) of every second page of its range, through a private ring ----
// lane l of the warp holds the page pointers of the warp's slice j0 + l
__device__ __forceinline__ void slice_ptrs(const long long* kptrs, const long long* vptrs, int pidx, int p_end, long long& kp_l, long long& vp_l) {
  kp_l = (pidx < p_end) ? kptrs[pidx] : 0;
  vp_l = (pidx < p_end) ? vptrs[pidx] : 0;
}
// all lanes call; lane 0 issues the six bulk copies of slice j (K codes | V codes | K scales | K zeros | V scales | V zeros) into `dst`
template <int BITS>
__device__ __forceinline__ void issue_slice(int lane, long long kp_l, long long vp_l, int j, uint8_t* dst, uint64_t* bar, int hk, int hslice, int code_bytes,
                                            int zoff) {
  using SL = StageLayout<BITS>;
  const long long kp_j = __shfl_sync(0xffffffffu, kp_l, j & 31), vp_j = __shfl_sync(0xffffffffu, vp_l, j & 31);
  if (lane == 0) {
    const uint8_t* kpage = reinterpret_cast<const uint8_t*>(kp_j);
    const uint8_t* vpage = reinterpret_cast<const uint8_t*>(vp_j);
    fence_proxy_async();  // the slot was last read through the generic proxy
    mbar_expect_tx(bar, SL::kBytes);
    bulk_copy_g2s(dst + SL::kOffK, kpage + static_cast<size_t>(hk) * SL::kCodes + hslice * SL::kSliceCodes, SL::kSliceCodes, bar);
    bulk_copy_g2s(dst + SL::kOffV, vpage + static_cast<size_t>(hk) * SL::kCodes + hslice * SL::kSliceCodes, SL::kSliceCodes, bar);
    const uint8_t* kmeta = kpage + code_bytes + hk * 128 + hslice * 64;
    const uint8_t* vmeta = vpage + code_bytes + hk * 128 + hslice * 64;
    bulk_copy_g2s(dst + SL::kOffKs, kmeta, 64, bar);
    bulk_copy_g2s(dst + SL::kOffKz, kmeta + zoff, 64, bar);
    bulk_copy_g2s(dst + SL::kOffVs, vmeta, 64, bar);
    bulk_copy_g2s(dst + SL::kOffVz, vmeta + zoff, 64, bar);
  }
}

// ---- Q as the MMA "B" operand of one n8 tile (n = column g), permuted to the in-register order of the unpacked codes; sum(q) and the operand
//      bias of this thread's columns 2q4, 2q4 + 1.  The tensor-core operands are the codes with the fp16 magic exponent still attached: 1024 + u
//      (low nibble / byte) or 1024 + 16 u (high nibble, the matching Q entries are pre-scaled by 1/16).  The constant part is removed after the
//      MMA:  sum_d (1024 + w_d u_d) q'_d = B(q) + sum_d u_d q_d ,   B(q) = 1024 sum_{low} q_d + 64 sum_{high} q_d.
//      qrow = the 32 q values of column g, dims 32 q4 .. (shared memory) ----
template <int BITS>
__device__ __forceinline__ void q_operand(const __half* qrow, int q4, uint32_t (&qb0)[8], uint32_t (&qb1)[8], float (&sumq)[2], float (&biasq)[2]) {
  // word k holds dims (2k, 2k+1)
  uint32_t qw[16];
  const uint4* qv = reinterpret_cast<const uint4*>(qrow);
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    const uint4 t = qv[k4];
    qw[4 * k4] = t.x; qw[4 * k4 + 1] = t.y; qw[4 * k4 + 2] = t.z; qw[4 * k4 + 3] = t.w;
  }
  float ae[2] = {0.f, 0.f}, ao[2] = {0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&qw[k]));
    ae[k & 1] += f.x;
    ao[k & 1] += f.y;
  }
  float acc_e = ae[0] + ae[1], acc_o = ao[0] + ao[1];
  acc_e += __shfl_xor_sync(0xffffffffu, acc_e, 1);
  acc_o += __shfl_xor_sync(0xffffffffu, acc_o, 1);
  acc_e += __shfl_xor_sync(0xffffffffu, acc_e, 2);
  acc_o += __shfl_xor_sync(0xffffffffu, acc_o, 2);
  const float acc = acc_e + acc_o;
  const float bias = (BITS == 4) ? fmaf(1024.f, acc_e, 64.f * acc_o) : 1024.f * acc;  // KV4: odd dims sit in the high nibbles
  sumq[0] = __shfl_sync(0xffffffffu, acc, (2 * q4) * 4);
  sumq[1] = __shfl_sync(0xffffffffu, acc, (2 * q4 + 1) * 4);
  biasq[0] = __shfl_sync(0xffffffffu, bias, (2 * q4) * 4);
  biasq[1] = __shfl_sync(0xffffffffu, bias, (2 * q4 + 1) * 4);
#pragma unroll
  for (int s = 0; s < 8; ++s) {
    if constexpr (BITS == 4) {
      // k-step 2w: nibbles (0,4 | 1,5); 2w+1: (2,6 | 3,7) of word w  ->  dims d0, d0+4 | d0+1, d0+5 with d0 = 8 (s>>1) + 2 (s&1)
      const int k0 = 4 * (s >> 1) + (s & 1);
      qb0[s] = __byte_perm(qw[k0], qw[k0 + 2], 0x5410);
      const uint32_t hi = __byte_perm(qw[k0], qw[k0 + 2], 0x7632);
      const __half2 sc16 = __hmul2(*reinterpret_cast<const __half2*>(&hi), __float2half2_rn(0.0625f));  // exact: a power of two
      qb1[s] = *reinterpret_cast<const uint32_t*>(&sc16);
    } else {
      qb0[s] = qw[2 * s];
      qb1[s] = qw[2 * s + 1];
    }
  }
}

// ---- NeoX RoPE of one query / key row at position pos: the pair (i, i + half_rot) of x0 = row[i], x1 = row[i + half_rot] goes to dst, rounded to
//      fp16.  decode_attention_kernel and shared_prefix_attention_kernel both rotate through these two functions, so a member's q has the
//      same bits in both passes ----
__device__ __forceinline__ void rope_sincos(int pos, int i, float rotary_base, int rotary_dim, float& sn, float& cs) {
  const float inv_freq = __fdiv_rn(static_cast<float>(pos), powf(rotary_base, __fdiv_rn(static_cast<float>(2 * i), static_cast<float>(rotary_dim))));
  sincosf(inv_freq, &sn, &cs);
}
__device__ __forceinline__ void rope_store(__half* dst, int i, int half_rot, __half x0, __half x1, float sn, float cs) {
  const float f0 = __half2float(x0), f1 = __half2float(x1);
  dst[i] = __float2half_rn(__fsub_rn(__fmul_rn(cs, f0), __fmul_rn(sn, f1)));
  dst[i + half_rot] = __float2half_rn(__fadd_rn(__fmul_rn(cs, f1), __fmul_rn(sn, f0)));
}

// ---- per-token (scale, c = -scale * zero) pairs of the 32 K and 32 V tokens of a slice, converted to fp32 ONCE per token (fp16 -> fp32
//      conversions run on the slow XU pipe: the logit code must not repeat them per thread); K pre-multiplied by the softmax scale.
//      `unread`: a slot no column reads (its scale may be anything, NaN included): forced to finite zeros, its logits are masked ----
template <int BITS>
__device__ __forceinline__ void slice_meta(const uint8_t* st, int lane, bool unread, float sm_scale, float2* meta_k, float2* meta_v) {
  using SL = StageLayout<BITS>;
  const __half* kp = reinterpret_cast<const __half*>(st + SL::kOffKs) + lane;
  const __half* vp = reinterpret_cast<const __half*>(st + SL::kOffVs) + lane;
  const __half ksc = kp[0], kzp = kp[32], vsc = vp[0], vzp = vp[32];
  float2 fk, fv;
  if constexpr (BITS == 4) {
    // c = half(-s * z): the fp16 product of two fp16 values, rounded once
    fk = __half22float2(__halves2half2(ksc, __hmul(__hneg(ksc), kzp)));
    fv = __half22float2(__halves2half2(vsc, __hmul(__hneg(vsc), vzp)));
  } else {
    fk = __half22float2(__halves2half2(ksc, kzp));
    fv = __half22float2(__halves2half2(vsc, vzp));
    fk.y = -fk.x * fk.y;  // aux holds the zero point: c = -s * z in fp32
    fv.y = -fv.x * fv.y;
  }
  fk.x *= sm_scale;
  fk.y *= sm_scale;
  if (unread) fk = fv = make_float2(0.f, 0.f);
  meta_k[lane] = fk;
  meta_v[lane] = fv;
}

// ---- S^T of one 16-token chunk (A rows g / g+8 <-> chunk tokens tokA / 8+tokA) x NT n8 tiles on biased codes.  Every unpacked code operand
//      feeds the NT tiles; qb(t, s, b0, b1) yields the B fragment of tile t, k-step s ----
template <int BITS, int NT, class QB>
__device__ __forceinline__ void qk_chunk(const uint8_t* krow, int q4, float (&sc)[NT][4], const QB& qb) {
  constexpr int kRow = kD * BITS / 8;  // bytes per token row
  if constexpr (BITS == 4) {
    const uint4 ka = *reinterpret_cast<const uint4*>(krow + q4 * 16);
    const uint4 kb = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 16);
    const uint32_t wa[4] = {ka.x, ka.y, ka.z, ka.w}, wb[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const uint32_t xa = wa[w], xb = wb[w], ta = xa >> 8, tb = xb >> 8;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        uint32_t b0, b1;
        qb(t, 2 * w, b0, b1);
        mma_full(sc[t][0], sc[t][1], sc[t][2], sc[t][3], lop3_and_or(xa, 0x000f000fu, kMagic), lop3_and_or(xb, 0x000f000fu, kMagic),
                 lop3_and_or(xa, 0x00f000f0u, kMagic), lop3_and_or(xb, 0x00f000f0u, kMagic), b0, b1);
      }
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        uint32_t b0, b1;
        qb(t, 2 * w + 1, b0, b1);
        mma_full(sc[t][0], sc[t][1], sc[t][2], sc[t][3], lop3_and_or(ta, 0x000f000fu, kMagic), lop3_and_or(tb, 0x000f000fu, kMagic),
                 lop3_and_or(ta, 0x00f000f0u, kMagic), lop3_and_or(tb, 0x00f000f0u, kMagic), b0, b1);
      }
    }
  } else {
    const uint4 ka0 = *reinterpret_cast<const uint4*>(krow + q4 * 32), ka1 = *reinterpret_cast<const uint4*>(krow + q4 * 32 + 16);
    const uint4 kb0 = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 32), kb1 = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 32 + 16);
    const uint32_t wa[8] = {ka0.x, ka0.y, ka0.z, ka0.w, ka1.x, ka1.y, ka1.z, ka1.w};
    const uint32_t wb[8] = {kb0.x, kb0.y, kb0.z, kb0.w, kb1.x, kb1.y, kb1.z, kb1.w};
#pragma unroll
    for (int w = 0; w < 8; ++w) {
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        uint32_t b0, b1;
        qb(t, w, b0, b1);
        // bytes -> fp16: 0x6400 | u = 1024 + u
        mma_full(sc[t][0], sc[t][1], sc[t][2], sc[t][3], __byte_perm(wa[w], kMagic, 0x7150), __byte_perm(wb[w], kMagic, 0x7150),
                 __byte_perm(wa[w], kMagic, 0x7352), __byte_perm(wb[w], kMagic, 0x7352), b0, b1);
      }
    }
  }
}

// ---- logits (log2 units) of tokens A = tokA, B = 8 + tokA of chunk c for this thread's columns, and the chunk tokens' V (scale, c) ----
template <int NT>
__device__ __forceinline__ void chunk_logits(const float2* meta_k, const float2* meta_v, int c, int tokA, const float (&sc)[NT][4], const float (&biasq)[NT][2],
                                             const float (&sumq)[NT][2], float (&tl)[NT][4], float (&vs)[2], float (&vc)[2]) {
  const float2 fkA = meta_k[c * kChunk + tokA], fkB = meta_k[c * kChunk + 8 + tokA];
  const float2 fvA = meta_v[c * kChunk + tokA], fvB = meta_v[c * kChunk + 8 + tokA];
  vs[0] = fvA.x; vs[1] = fvB.x; vc[0] = fvA.y; vc[1] = fvB.y;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    tl[t][0] = fmaf(fkA.x, sc[t][0] - biasq[t][0], fkA.y * sumq[t][0]);
    tl[t][1] = fmaf(fkA.x, sc[t][1] - biasq[t][1], fkA.y * sumq[t][1]);
    tl[t][2] = fmaf(fkB.x, sc[t][2] - biasq[t][0], fkB.y * sumq[t][0]);
    tl[t][3] = fmaf(fkB.x, sc[t][3] - biasq[t][1], fkB.y * sumq[t][1]);
  }
}

// ---- online softmax of n8 tile t over the two chunks of a slice, with lazy rescaling (only when a running max moves by more than 2^8);
//      produces the P'^T fragments bp[c][t] of the V MMAs.  Running state per column: max m, sum p l, sum p*c (zero-point correction) cr, and
//      spa = sum p' (bias correction of the V operand), accumulated by one MMA against an all-ones tile from the very operand the V MMAs consume.
//      EMPTY: a column may have every key of a slice masked while its running max is still -inf; it then exponentiates against 0 (p = 0,
//      not NaN) ----
template <int NT, bool EMPTY>
__device__ __forceinline__ void softmax_tile(int t, const float (&tl)[2][NT][4], const float (&vs)[2][2], const float (&vc)[2][2], float (&m)[2], float (&l)[2],
                                             float (&cr)[2], float (&spa)[4], float (&o)[8][4], uint32_t (&bp)[2][NT][2]) {
  float mh0 = fmaxf(fmaxf(tl[0][t][0], tl[0][t][2]), fmaxf(tl[1][t][0], tl[1][t][2]));
  float mh1 = fmaxf(fmaxf(tl[0][t][1], tl[0][t][3]), fmaxf(tl[1][t][1], tl[1][t][3]));
#pragma unroll
  for (int sh = 4; sh <= 16; sh <<= 1) {
    mh0 = fmaxf(mh0, __shfl_xor_sync(0xffffffffu, mh0, sh));
    mh1 = fmaxf(mh1, __shfl_xor_sync(0xffffffffu, mh1, sh));
  }
  const bool n0 = mh0 > m[0] + 8.f, n1 = mh1 > m[1] + 8.f;
  if (__any_sync(0xffffffffu, n0 || n1)) {
    const float a0 = n0 ? exp2f(m[0] - mh0) : 1.f, a1 = n1 ? exp2f(m[1] - mh1) : 1.f;
    if (n0) m[0] = mh0;
    if (n1) m[1] = mh1;
    l[0] *= a0; cr[0] *= a0; l[1] *= a1; cr[1] *= a1;
    spa[0] *= a0; spa[2] *= a0; spa[1] *= a1; spa[3] *= a1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i][0] *= a0; o[i][2] *= a0;
      o[i][1] *= a1; o[i][3] *= a1;
    }
  }
  float mb0 = m[0], mb1 = m[1];
  if constexpr (EMPTY) {
    mb0 = mb0 == -CUDART_INF_F ? 0.f : mb0;
    mb1 = mb1 == -CUDART_INF_F ? 0.f : mb1;
  }
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const float pA0 = ex2_approx(tl[c][t][0] - mb0), pA1 = ex2_approx(tl[c][t][1] - mb1);
    const float pB0 = ex2_approx(tl[c][t][2] - mb0), pB1 = ex2_approx(tl[c][t][3] - mb1);
    l[0] += pA0 + pB0; l[1] += pA1 + pB1;
    cr[0] = fmaf(pA0, vc[c][0], fmaf(pB0, vc[c][1], cr[0]));
    cr[1] = fmaf(pA1, vc[c][0], fmaf(pB1, vc[c][1], cr[1]));
    // P' = p * s_v rounded to fp16 (the MMA operand); its exact sum removes the 1024 bias of the V operand afterwards
    const uint32_t hA = pack_f2h2(pA0 * vs[c][0], pA1 * vs[c][0]), hB = pack_f2h2(pB0 * vs[c][1], pB1 * vs[c][1]);
    // P'^T fragments: transpose the (token, column) tiles so that tokens become the MMA k index
    bp[c][t][0] = movmatrix_trans(hA);  // k = 2q4, 2q4+1  <-> chunk tokens q4, 4+q4
    bp[c][t][1] = movmatrix_trans(hB);  // k = 2q4+8, +9   <-> chunk tokens 8+q4, 12+q4
    mma_full(spa[0], spa[1], spa[2], spa[3], kOnesH2, kOnesH2, kOnesH2, kOnesH2, bp[c][t][0], bp[c][t][1]);
  }
}

// ---- O^T += V^T P'^T of one 16-token chunk on biased codes (m-tile i = 16 dims): every unpacked V operand feeds the NT tiles ----
template <int BITS, int NT>
__device__ __forceinline__ void pv_chunk(const uint8_t* vbase, int g, float (&o)[NT][8][4], const uint32_t (&bp)[NT][2]) {
  constexpr int kRow = kD * BITS / 8;
  if constexpr (BITS == 4) {
    const uint2 va = *reinterpret_cast<const uint2*>(vbase + g * 8);
    const uint2 vb = *reinterpret_cast<const uint2*>(vbase + 4 * kRow + g * 8);
    const uint2 vcw = *reinterpret_cast<const uint2*>(vbase + 8 * kRow + g * 8);
    const uint2 vd = *reinterpret_cast<const uint2*>(vbase + 12 * kRow + g * 8);
#pragma unroll
    for (int ww = 0; ww < 2; ++ww) {
      const uint32_t a = ww ? va.y : va.x, bb = ww ? vb.y : vb.x, cc = ww ? vcw.y : vcw.x, dd = ww ? vd.y : vd.x;
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        const uint32_t sel = static_cast<uint32_t>(kb) | (static_cast<uint32_t>(kb) << 4) | (static_cast<uint32_t>(4 + kb) << 8) |
                             (static_cast<uint32_t>(4 + kb) << 12);  // bytes [a_kb, a_kb, b_kb, b_kb]
        const uint32_t m01 = __byte_perm(a, bb, sel), m89 = __byte_perm(cc, dd, sel);
        const int i = 4 * ww + kb;
#pragma unroll
        for (int t = 0; t < NT; ++t)
          mma_full(o[t][i][0], o[t][i][1], o[t][i][2], o[t][i][3], lop3_and_or(m01, 0x000f000fu, kMagic), lop3_and_or(m01, 0x00f000f0u, kMagic),
                   lop3_and_or(m89, 0x000f000fu, kMagic), lop3_and_or(m89, 0x00f000f0u, kMagic), bp[t][0], bp[t][1]);
      }
    }
  } else {
    const uint4 va = *reinterpret_cast<const uint4*>(vbase + g * 16);
    const uint4 vb = *reinterpret_cast<const uint4*>(vbase + 4 * kRow + g * 16);
    const uint4 vcw = *reinterpret_cast<const uint4*>(vbase + 8 * kRow + g * 16);
    const uint4 vd = *reinterpret_cast<const uint4*>(vbase + 12 * kRow + g * 16);
    const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
    const uint32_t wc[4] = {vcw.x, vcw.y, vcw.z, vcw.w}, wd[4] = {vd.x, vd.y, vd.z, vd.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      // dims 16g + 2i (row g) and 16g + 2i + 1 (row g+8): bytes 2i, 2i+1 of the 16-byte row chunk
      const int w = i >> 1, b0 = 2 * (i & 1), b1 = b0 + 1;
      const uint32_t sel0 = static_cast<uint32_t>(b0) | (static_cast<uint32_t>(b0) << 4) | (static_cast<uint32_t>(4 + b0) << 8) | (static_cast<uint32_t>(4 + b0) << 12);
      const uint32_t sel1 = static_cast<uint32_t>(b1) | (static_cast<uint32_t>(b1) << 4) | (static_cast<uint32_t>(4 + b1) << 8) | (static_cast<uint32_t>(4 + b1) << 12);
#pragma unroll
      for (int t = 0; t < NT; ++t)
        mma_full(o[t][i][0], o[t][i][1], o[t][i][2], o[t][i][3], lop3_and_or(__byte_perm(wa[w], wb[w], sel0), 0x00ff00ffu, kMagic),
                 lop3_and_or(__byte_perm(wa[w], wb[w], sel1), 0x00ff00ffu, kMagic), lop3_and_or(__byte_perm(wc[w], wd[w], sel0), 0x00ff00ffu, kMagic),
                 lop3_and_or(__byte_perm(wc[w], wd[w], sel1), 0x00ff00ffu, kMagic), bp[t][0], bp[t][1]);
    }
  }
}

// ---- end of the stream: warp-reduce the per-column sums of tile t ----
__device__ __forceinline__ void reduce_tile_sums(float (&l)[2], float (&cr)[2]) {
#pragma unroll
  for (int sh = 4; sh <= 16; sh <<= 1) {
    l[0] += __shfl_xor_sync(0xffffffffu, l[0], sh);
    l[1] += __shfl_xor_sync(0xffffffffu, l[1], sh);
    cr[0] += __shfl_xor_sync(0xffffffffu, cr[0], sh);
    cr[1] += __shfl_xor_sync(0xffffffffu, cr[1], sh);
  }
}
// ---- a warp's partial O^T of one tile -> its own (drained) ring.  Layout [column][(d % 16) * 8 + d / 16], column stride kOStride floats:
//      conflict-free for these stores and for the merge reads (thread t owns dim 16 (t % 8) + t / 8).  so0 = ring + (8t + 2q4) * kOStride + g ----
template <int BITS>
__device__ __forceinline__ void store_partial(float* so0, const float (&o)[8][4], const float (&spa)[4], const float (&cr)[2]) {
  float* so1 = so0 + kOStride;  // column 2q4 + 1
  constexpr float hs = (BITS == 4) ? 0.0625f : 1.f;
  const float b0 = 1024.f * spa[0], b1 = 1024.f * spa[1];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    // remove the operand bias (1024 sum p'); KV4: the odd dims came from the high nibbles, i.e. 16 x the code
    so0[8 * (2 * i)] = (o[i][0] - b0) + cr[0]; so0[8 * (2 * i + 1)] = (o[i][2] - b0) * hs + cr[0];
    so1[8 * (2 * i)] = (o[i][1] - b1) + cr[1]; so1[8 * (2 * i + 1)] = (o[i][3] - b1) * hs + cr[1];
  }
}

// ---- the un-quantised own / new token: fp32 dot of the rotated q and k (Template.hpp:1410-1441), complete in every lane ----
__device__ __forceinline__ float own_logit(const __half* q, const __half* k, int lane) {
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) acc = fmaf(__half2float(q[lane * 4 + j]), __half2float(k[lane * 4 + j]), acc);
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  return acc;
}

// ---- merge of the warps (and, for the owner of split 0, the own token as part kWarps) of column r: weights exp2(m_w - M), normalised by
//      1 / (sum + 1e-6) (Template.hpp:1818) when this CTA produces the final output; M and the sum go to s_m[0][r], s_l[0][r] ----
template <int COLS>
__device__ __forceinline__ void merge_weights(int r, int nparts, int nsplit, float (&s_m)[kWarps + 1][COLS], float (&s_l)[kWarps + 1][COLS],
                                              float (&s_f)[kWarps + 1][COLS]) {
  float M = -CUDART_INF_F;
  for (int w = 0; w < nparts; ++w) M = fmaxf(M, s_m[w][r]);
  float e[kWarps + 1], L = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps + 1; ++w) {
    e[w] = (w < nparts && s_m[w][r] != -CUDART_INF_F) ? exp2f(s_m[w][r] - M) : 0.f;
    if (w < nparts) L += s_l[w][r] * e[w];
  }
  const float inv = (nsplit == 1) ? __fdividef(1.f, L + 1.e-6f) : 1.f;
#pragma unroll
  for (int w = 0; w < kWarps + 1; ++w) s_f[w][r] = e[w] * inv;
  s_m[0][r] = M;   // only read back by the split path
  s_l[0][r] = L;
}
// output dim of thread threadIdx.x (< kD) for column r: the own token's value plus the warps' partials (in the rings), weighted
template <int BITS, int COLS>
__device__ __forceinline__ float merge_warps(const uint8_t* s_ring, int r, float own_v, const float (&s_f)[kWarps + 1][COLS]) {
  float acc = s_f[kWarps][r] * own_v;
#pragma unroll
  for (int w = 0; w < kWarps; ++w)
    acc = fmaf(reinterpret_cast<const float*>(s_ring + w * StageLayout<BITS>::kWarpBytes)[r * kOStride + threadIdx.x], s_f[w][r], acc);
  return acc;
}

// ---- context splits: every CTA arrives on the counter of its group; the last to arrive resets it (self-cleaning) and merges ----
__device__ __forceinline__ bool arrive_last(uint32_t* cnt, int nsplit, uint32_t& s_last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t old = atomicAdd(cnt, 1u);
    const bool last = (old == static_cast<uint32_t>(nsplit - 1));
    if (last) *cnt = 0;
    s_last = last ? 1u : 0u;
  }
  __syncthreads();
  return s_last != 0;
}
// the split partials of one column, in split order (deterministic): [nsplit][kD values, max, sum] -> normalised output of dim d
__device__ __forceinline__ float merge_splits(const float* pr, int nsplit, int d) {
  float M = -CUDART_INF_F;
  for (int sp = 0; sp < nsplit; ++sp) M = fmaxf(M, __ldcg(pr + sp * (kD + 2) + kD));
  float L = 0.f, acc = 0.f;
  for (int sp = 0; sp < nsplit; ++sp) {
    const float ms = __ldcg(pr + sp * (kD + 2) + kD);
    const float e = (ms == -CUDART_INF_F) ? 0.f : exp2f(ms - M);
    L += __ldcg(pr + sp * (kD + 2) + kD + 1) * e;
    acc += __ldcg(pr + sp * (kD + 2) + d) * e;
  }
  return acc * __fdividef(1.f, L + 1.e-6f);
}

}  // namespace
}  // namespace qs
