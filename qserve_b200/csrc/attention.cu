// qserve_b200 -- single-query (decode) attention over the INT4 / INT8 paged KV cache, the prefill
// RoPE + KV-quantise + page-append kernel, and the padding-offset helper.
//
// Replaces  kernels/csrc/fused_attention/decoderMaskedMultiheadAttentionTemplate.hpp:717-2222 (decode),
//           kernels/csrc/fused_attention/applyBiasRopeUpdateKVCache.h:94-455 (prefill append),
//           kernels/csrc/fused_attention/input_metadata_helper.cu:11-45.
//
// Design (DESIGN.md 3.2): the reference launches one CTA per *query* head and therefore streams every KV head
// Hq/Hkv times; here one CTA (4 warps) owns a (sequence, KV head, context split) and serves all query heads of the GQA
// group from a single pass over the pages, so HBM traffic is the algorithmic minimum.  Every warp streams its own 32-token
// slices of the pages with cp.async.bulk into a private shared-memory ring; the (<= 8 heads) x 32-token QK^T and PV
// products run as mma.sync m16n8k16 on "biased" operands (0x6400 | code = 1024 + code in fp16: one LOP3 per two codes, the
// constant parts are removed after the MMA), per-token scale / zero are folded into the logits and probabilities, the
// softmax is an online (flash-decoding) softmax with lazy rescaling, and context splits are merged by the last-arriving
// CTA.  RoPE of q/k, KV quantisation and the page append of the new token are fused in; optionally also the per-token
// INT8 quantisation of the output row (single_query_attention_quant).
#include <math_constants.h>

#include "common.cuh"
#include "launch.h"

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

__device__ __forceinline__ unsigned long long attn_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
  return t;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr uint32_t kMagic = 0x64006400u;      // half2(1024, 1024)
constexpr uint32_t kOnesH2 = 0x3c003c00u;     // half2(1, 1)

// A4 quantisation parameters (Template.hpp:1243,1067): scale = half((max-min)/L), zero = half(-L*min/(max-min))
__device__ __forceinline__ void kv_quant_params(float mx, float mn, float L, __half& s, __half& z) {
  const float d = __fsub_rn(mx, mn);
  s = __float2half_rn(__fdiv_rn(d, L));
  z = __float2half_rn(__fdiv_rn(__fmul_rn(-L, mn), d));
}
__device__ __forceinline__ uint32_t kv_quant_code(float x, float inv_s, float z) {
  uint32_t r;
  const float t = __fadd_rn(__fmul_rn(x, inv_s), z);
  asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(r) : "f"(t));
  return r;
}

// ------------------------------------------------------------------------------------------------
// K1: decode attention
//   Warp w consumes the 32-token slice (w & 1) of the pages of parity (w >> 1) of its CTA's context range.
//   Scale folding (exact in real arithmetic; skips the reference's per-element fp16 rounding of the dequantised values):
//     q.k_t   = s_t * (q . u_t) + c_t * sum(q)          u = integer codes,   c_t = half(-s_t * z_t)
//     sum_t p_t v_t = sum_t (p_t s_t) u_t + sum_t p_t c_t
//   so the per-token scale touches 4 logits / 4 probabilities per thread instead of 2 x 128 elements
//   (KV8: k_t = s_t * (u_t - z_t), same folding with c_t = -s_t * z_t in fp32).
//   Biased operands: the MMA sees 1024 + u (low nibble / byte) or 1024 + 16 u (high nibble; Q pre-scaled by 1/16 on the K
//   side, output rows rescaled at the end on the V side); sum_d (1024 + w_d u_d) q'_d = B(q) + sum_d u_d q_d with B(q) computed
//   once per head, and sum_t p'_t (1024 + u_t) = 1024 sum_t p'_t + ... with sum_t p'_t from one MMA against an all-ones tile.
// ------------------------------------------------------------------------------------------------
constexpr int kAttnConsumers = 128;
constexpr int kAttnThreadsV2 = kAttnConsumers;  // no dedicated producer warp: every warp streams its own half pages
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

template <int BITS>
__global__ void __launch_bounds__(kAttnThreadsV2, 4)
decode_attention_kernel(const __half* __restrict__ q_in, const __half* __restrict__ k_in, const __half* __restrict__ v_in, long long q_stride,
                        long long k_stride, long long v_stride, const long long* __restrict__ kv_pointers, const int* __restrict__ lengths,
                        __half* __restrict__ out, int num_heads, int num_kv_heads, int max_blocks, PageGeom pg, float rotary_base, int rotary_dim,
                        int timestep, int nsplit, float* __restrict__ ws_part, uint32_t* __restrict__ ws_cnt, uint32_t* __restrict__ tok_cnt, int8_t* __restrict__ q_out,
                        __half* __restrict__ q_scale, __half* __restrict__ q_sum, unsigned long long* __restrict__ prof) {
  using SL = StageLayout<BITS>;
  constexpr int R = SL::kStages;
  const int G = num_heads / num_kv_heads;
  const int gparts = (G + kMaxG - 1) / kMaxG;
  const int hk = blockIdx.x / gparts;
  const int gpart = blockIdx.x - hk * gparts;
  const int h0 = hk * G + gpart * kMaxG;
  const int Gc = min(kMaxG, G - gpart * kMaxG);
  const int b = blockIdx.y;
  const int split = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, q4 = lane & 3;

  extern __shared__ __align__(128) uint8_t smem_attn[];
  uint8_t* s_ring = smem_attn;                                           // kWarps private rings of R slices
  __shared__ __align__(16) __half s_q[kMaxG * kD];
  __shared__ __align__(16) __half s_k[kD];
  __shared__ __align__(16) __half s_v[kD];
  __shared__ float s_m[kWarps + 1][kMaxG], s_l[kWarps + 1][kMaxG];
  __shared__ float s_f[kWarps + 1][kMaxG];                                // merge weights exp2(m_w - M) [* 1 / L]
  __shared__ float2 s_meta[kWarps][2][kSliceTokens];                     // per token (scale, c) of the slice in flight: K pre-multiplied by sm_scale
  __shared__ __align__(8) uint64_t s_full[kWarps][R];
  __shared__ uint32_t s_last;

  // Every warp initialises the barriers of ITS OWN ring (lane 0, the lane that later arms them and issues the copies), so no block-wide
  // barrier is needed between initialisation and first use.  Round 1 let thread 0 initialise all rings without a barrier: harmless while every
  // CTA of a single-wave launch sat in griddepcontrol.wait long enough, but a late CTA of a multi-wave launch (64 kv heads x 64 sequences =
  // 4096 CTAs at Qwen1.5-72B) could arm a ring before thread 0 had initialised it -- the initialisation then wiped the pending transaction
  // count and that warp waited forever (about one hung warp per 10^8 slices).
  if (lane == 0) {
    for (int i = 0; i < R; ++i) mbar_init(&s_full[warp][i], 1);
    fence_barrier_init();
  }
  __syncwarp();
#define ATTN_PROF(slot) do { if (prof) prof[((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 16 + (slot)] = attn_gtime(); } while (0)
  if (threadIdx.x == 0) ATTN_PROF(0);
  qs_trace(QS_K_ATTN, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away

  // The sequence lengths and the page-pointer table are prepared by the host side before the step (model_runner.py:506-530):
  // they are read BEFORE the dependency wait, so that the chain length -> page pointers -> first bulk copy (two dependent
  // global round trips) overlaps the tail of the preceding qkv GEMM.  Page CONTENTS and q/k/v are only touched after the wait.
  const int tlen = lengths ? lengths[b] - 1 : timestep;  // tokens already in the cache (Template.hpp:901: length_per_sample ? len - 1 : timestep)
  const long long* kptrs = kv_pointers + (static_cast<size_t>(b) * 2 + 0) * max_blocks;
  const long long* vptrs = kv_pointers + (static_cast<size_t>(b) * 2 + 1) * max_blocks;
  const int n_pages = (tlen + kPageTokens - 1) / kPageTokens;
  const int pps = (n_pages + nsplit - 1) / nsplit;
  const int p_begin = split * pps, p_end = min(n_pages, p_begin + pps);
  const int last_blk = tlen / pg.tokens_per_block;  // page receiving the new token

  // ---- this warp's stream: token slice [32 (warp & 1), +32) of the pages p_begin + (warp >> 1), +2, ...  ----
  const int hslice = warp & 1;
  const int my_first = p_begin + (warp >> 1);
  const int n_my = (p_end > my_first) ? (p_end - my_first + 1) / 2 : 0;
  uint8_t* my_ring = s_ring + warp * SL::kWarpBytes;
  uint64_t* my_full = &s_full[warp][0];
  const int zoff = pg.num_kv_heads * pg.tokens_per_block * 2;  // bytes from a scale row to the zero row
  long long kp_l = 0, vp_l = 0;  // lane l: page pointers of this warp's page (batch * 32 + l)
  auto load_ptr_batch = [&](int j0) {
    const int pidx = my_first + 2 * (j0 + lane);
    kp_l = (pidx < p_end) ? kptrs[pidx] : 0;
    vp_l = (pidx < p_end) ? vptrs[pidx] : 0;
  };
  auto issue = [&](int j, int slot) {  // all lanes call; lane 0 issues the six copies of this warp's j-th slice into `slot`
    const long long kp_j = __shfl_sync(0xffffffffu, kp_l, j & 31), vp_j = __shfl_sync(0xffffffffu, vp_l, j & 31);
    if (lane == 0) {
      const uint8_t* kpage = reinterpret_cast<const uint8_t*>(kp_j);
      const uint8_t* vpage = reinterpret_cast<const uint8_t*>(vp_j);
      uint8_t* dst = my_ring + slot * SL::kBytes;
      fence_proxy_async();  // the slot was last read through the generic proxy
      mbar_expect_tx(&my_full[slot], SL::kBytes);
      bulk_copy_g2s(dst + SL::kOffK, kpage + static_cast<size_t>(hk) * SL::kCodes + hslice * SL::kSliceCodes, SL::kSliceCodes, &my_full[slot]);
      bulk_copy_g2s(dst + SL::kOffV, vpage + static_cast<size_t>(hk) * SL::kCodes + hslice * SL::kSliceCodes, SL::kSliceCodes, &my_full[slot]);
      const uint8_t* kmeta = kpage + pg.code_bytes + hk * 128 + hslice * 64;
      const uint8_t* vmeta = vpage + pg.code_bytes + hk * 128 + hslice * 64;
      bulk_copy_g2s(dst + SL::kOffKs, kmeta, 64, &my_full[slot]);
      bulk_copy_g2s(dst + SL::kOffKz, kmeta + zoff, 64, &my_full[slot]);
      bulk_copy_g2s(dst + SL::kOffVs, vmeta, 64, &my_full[slot]);
      bulk_copy_g2s(dst + SL::kOffVz, vmeta + zoff, 64, &my_full[slot]);
    }
  };
  load_ptr_batch(0);
  pdl_wait();
  qs_trace(QS_K_ATTN, 1);
  if (threadIdx.x == 0) ATTN_PROF(1);
  for (int j = 0; j < R && j < n_my; ++j) issue(j, j);  // the cache stream starts before the new-token work below
  if (threadIdx.x == 0) ATTN_PROF(3);
  {
    // ================================ consumer warps ================================
    // ---- new token: RoPE (NeoX, position tlen) of q and k; stage q, k, v in shared memory.
    //      Thread t rotates the pair (i, i + 64), i = t % 64, of rows t / 64, t / 64 + 2, ... (row Gc is k): the global loads
    //      go out first, the cos / sin of its own pair is computed while they are in flight (no table, no extra barrier) ----
    const int half_rot = rotary_dim / 2;  // == 64 (checked on the host)
    const int ri = threadIdx.x & 63, r0 = threadIdx.x >> 6;
    const __half* kg = k_in + static_cast<size_t>(b) * k_stride + static_cast<size_t>(hk) * kD;
    const __half* vg = v_in + static_cast<size_t>(b) * v_stride + static_cast<size_t>(hk) * kD;
    constexpr int kRowsPerThread = (kMaxG + 2) / 2;
    __half x0[kRowsPerThread], x1[kRowsPerThread];
#pragma unroll
    for (int e = 0; e < kRowsPerThread; ++e) {
      const int r = r0 + 2 * e;
      if (r <= Gc) {
        const __half* src = (r < Gc) ? (q_in + static_cast<size_t>(b) * q_stride + static_cast<size_t>(h0 + r) * kD) : kg;
        x0[e] = src[ri];
        x1[e] = src[ri + half_rot];
      }
    }
    const __half vnew = vg[threadIdx.x];
    float sn, cs;
    {
      const float inv_freq = __fdiv_rn(static_cast<float>(tlen), powf(rotary_base, __fdiv_rn(static_cast<float>(2 * ri), static_cast<float>(rotary_dim))));
      sincosf(inv_freq, &sn, &cs);
    }
#pragma unroll
    for (int e = 0; e < kRowsPerThread; ++e) {
      const int r = r0 + 2 * e;
      if (r <= Gc) {
        __half* dst = (r < Gc) ? (s_q + r * kD) : s_k;
        const float f0 = __half2float(x0[e]), f1 = __half2float(x1[e]);
        dst[ri] = __float2half_rn(__fsub_rn(__fmul_rn(cs, f0), __fmul_rn(sn, f1)));
        dst[ri + half_rot] = __float2half_rn(__fadd_rn(__fmul_rn(cs, f1), __fmul_rn(sn, f0)));
      }
    }
    s_v[threadIdx.x] = vnew;
    for (int i = threadIdx.x + Gc * kD; i < kMaxG * kD; i += kAttnConsumers) s_q[i] = __float2half_rn(0.f);
    asm volatile("bar.sync 1, 128;" ::: "memory");

    // ---- quantise + append the new K / V (one CTA per kv head) ----
    const bool owner_w = (split == 0) && (gpart == 0);
    if (owner_w && warp >= 2) {  // warps 2, 3: the first two warps start the main loop one page earlier
      const bool is_k = (warp == 2);
      const __half* src = is_k ? s_k : s_v;
      const float L = (BITS == 4) ? 15.f : 255.f;
      float x[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = __half2float(src[lane * 4 + j]);
      float mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3]));
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, m));
      }
      __half sc, zp;
      kv_quant_params(mx, mn, L, sc, zp);
      const float inv_s = __fdiv_rn(1.0f, __half2float(sc)), zf = __half2float(zp);
      const int slot = tlen - last_blk * pg.tokens_per_block;
      uint8_t* page = reinterpret_cast<uint8_t*>(is_k ? kptrs[last_blk] : vptrs[last_blk]);
      uint32_t c[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) c[j] = kv_quant_code(x[j], inv_s, zf);
      if constexpr (BITS == 4) {
        const uint16_t packed = static_cast<uint16_t>((c[0] & 0xF) | ((c[1] & 0xF) << 4) | ((c[2] & 0xF) << 8) | ((c[3] & 0xF) << 12));
        reinterpret_cast<uint16_t*>(page + static_cast<size_t>(hk * pg.tokens_per_block + slot) * (kD / 2))[lane] = packed;
      } else {
        reinterpret_cast<uint32_t*>(page + static_cast<size_t>(hk * pg.tokens_per_block + slot) * kD)[lane] = c[0] | (c[1] << 8) | (c[2] << 16) | (c[3] << 24);
      }
      if (lane == 0) {
        __half* meta = reinterpret_cast<__half*>(page + pg.code_bytes);
        meta[hk * pg.tokens_per_block + slot] = sc;
        meta[pg.num_kv_heads * pg.tokens_per_block + hk * pg.tokens_per_block + slot] = zp;
      }
    }

    // ---- Q as the MMA "B" operand (n = head g), permuted to the in-register order of the unpacked codes; sum(q) per head ----
    uint32_t qb0[8], qb1[8];
    float sumq0, sumq1;  // heads 2*q4 and 2*q4+1 (this thread's S^T columns)
    // The tensor-core operands are the codes with the fp16 magic exponent still attached: 1024 + u (low nibble / byte) or
    // 1024 + 16 u (high nibble, the matching Q entries are pre-scaled by 1/16).  The constant part is removed after the MMA:
    //   sum_d (1024 + w_d u_d) q'_d = B(q) + sum_d u_d q_d ,   B(q) = 1024 sum_{low} q_d + 64 sum_{high} q_d
    float biasq0, biasq1;
    {
      // this thread's 32 q values (head g, dims 32 q4 ..): word k holds dims (2k, 2k+1)
      uint32_t qw[16];
      const uint4* qv = reinterpret_cast<const uint4*>(s_q + g * kD + 32 * q4);
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
      sumq0 = __shfl_sync(0xffffffffu, acc, (2 * q4) * 4);
      sumq1 = __shfl_sync(0xffffffffu, acc, (2 * q4 + 1) * 4);
      biasq0 = __shfl_sync(0xffffffffu, bias, (2 * q4) * 4);
      biasq1 = __shfl_sync(0xffffffffu, bias, (2 * q4 + 1) * 4);
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

    const float sm_scale = rsqrtf(static_cast<float>(kD)) * 1.4426950408889634f;  // 1/sqrt(D) * log2(e)
    // O^T accumulators: m-tile i (dims 16g + 2i, 16g + 2i + 1) x heads (2q4, 2q4+1)
    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    // running max, sum p, sum p*c (zero-point correction), sum p' (bias correction of the V operand) per head
    float m0 = -CUDART_INF_F, m1 = -CUDART_INF_F, l0 = 0.f, l1 = 0.f, cr0 = 0.f, cr1 = 0.f;
    float spa[4] = {0.f, 0.f, 0.f, 0.f};  // [0], [1]: sum p' of heads 2q4, 2q4+1 over ALL tokens this warp has seen

    // S^T = K Q^T: A rows g / g+8 <-> chunk tokens tokA / 8+tokA (the permutation keeps the V row reads at a 2-way conflict)
    const int tokA = (g & 1) * 4 + (g >> 1);
    constexpr int kRow = kD * BITS / 8;  // bytes per token row
    // warp w consumes tokens [32 (w & 1), +32) of the pages whose index has parity (w >> 1): two 16-token MMA chunks per
    // iteration share one barrier wait, one max reduction and one set of address computations
    const int hbase = hslice * kSliceTokens;
    int s = 0;
    uint32_t ph = 0;
    if (threadIdx.x == 0) ATTN_PROF(4);
    for (int j = 0; j < n_my; ++j) {
      const int pidx = my_first + 2 * j;
      mbar_wait(&my_full[s], ph);
      if (threadIdx.x == 0 && j == 0) ATTN_PROF(5);
      const uint8_t* st = my_ring + s * SL::kBytes;
      const int t0 = pidx * kPageTokens + hbase;  // first token of this warp's 32-token slice
      if (t0 < tlen) {
        // per-token (scale, c = -scale * zero) pairs of the 32 K and 32 V tokens, converted to fp32 ONCE per token here
        // (fp16 -> fp32 conversions run on the slow XU pipe: the logit code below must not repeat them per thread)
        {
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
          if (t0 + lane >= tlen) fk = fv = make_float2(0.f, 0.f);  // unwritten slots: force finite zeros (their logits are masked below)
          s_meta[warp][0][lane] = fk;
          s_meta[warp][1][lane] = fv;
        }
        __syncwarp();
        // ---- S^T (2 x 16 tokens x 8 heads) on biased codes: 16 MMAs ----
        float sc[2][4];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          sc[c][0] = sc[c][1] = sc[c][2] = sc[c][3] = 0.f;
          const uint8_t* krow = st + SL::kOffK + (c * kChunk + tokA) * kRow;
          if constexpr (BITS == 4) {
            const uint4 ka = *reinterpret_cast<const uint4*>(krow + q4 * 16);
            const uint4 kb = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 16);
            const uint32_t wa[4] = {ka.x, ka.y, ka.z, ka.w}, wb[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              const uint32_t xa = wa[w], xb = wb[w], ta = xa >> 8, tb = xb >> 8;
              mma_full(sc[c][0], sc[c][1], sc[c][2], sc[c][3], lop3_and_or(xa, 0x000f000fu, kMagic), lop3_and_or(xb, 0x000f000fu, kMagic),
                       lop3_and_or(xa, 0x00f000f0u, kMagic), lop3_and_or(xb, 0x00f000f0u, kMagic), qb0[2 * w], qb1[2 * w]);
              mma_full(sc[c][0], sc[c][1], sc[c][2], sc[c][3], lop3_and_or(ta, 0x000f000fu, kMagic), lop3_and_or(tb, 0x000f000fu, kMagic),
                       lop3_and_or(ta, 0x00f000f0u, kMagic), lop3_and_or(tb, 0x00f000f0u, kMagic), qb0[2 * w + 1], qb1[2 * w + 1]);
            }
          } else {
            const uint4 ka0 = *reinterpret_cast<const uint4*>(krow + q4 * 32), ka1 = *reinterpret_cast<const uint4*>(krow + q4 * 32 + 16);
            const uint4 kb0 = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 32), kb1 = *reinterpret_cast<const uint4*>(krow + 8 * kRow + q4 * 32 + 16);
            const uint32_t wa[8] = {ka0.x, ka0.y, ka0.z, ka0.w, ka1.x, ka1.y, ka1.z, ka1.w};
            const uint32_t wb[8] = {kb0.x, kb0.y, kb0.z, kb0.w, kb1.x, kb1.y, kb1.z, kb1.w};
#pragma unroll
            for (int w = 0; w < 8; ++w) {
              // bytes -> fp16: 0x6400 | u = 1024 + u
              mma_full(sc[c][0], sc[c][1], sc[c][2], sc[c][3], __byte_perm(wa[w], kMagic, 0x7150), __byte_perm(wb[w], kMagic, 0x7150),
                       __byte_perm(wa[w], kMagic, 0x7352), __byte_perm(wb[w], kMagic, 0x7352), qb0[w], qb1[w]);
            }
          }
        }
        // ---- logits (log2 units) of tokens A = tokA, B = 8 + tokA of both chunks for heads 2q4, 2q4+1 ----
        float tl[2][4], vs[2][2], vc[2][2];
        const bool partial = (t0 + 2 * kChunk > tlen);  // only the last page of a sequence
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float2 fkA = s_meta[warp][0][c * kChunk + tokA], fkB = s_meta[warp][0][c * kChunk + 8 + tokA];
          const float2 fvA = s_meta[warp][1][c * kChunk + tokA], fvB = s_meta[warp][1][c * kChunk + 8 + tokA];
          vs[c][0] = fvA.x; vs[c][1] = fvB.x; vc[c][0] = fvA.y; vc[c][1] = fvB.y;
          tl[c][0] = fmaf(fkA.x, sc[c][0] - biasq0, fkA.y * sumq0);
          tl[c][1] = fmaf(fkA.x, sc[c][1] - biasq1, fkA.y * sumq1);
          tl[c][2] = fmaf(fkB.x, sc[c][2] - biasq0, fkB.y * sumq0);
          tl[c][3] = fmaf(fkB.x, sc[c][3] - biasq1, fkB.y * sumq1);
        }
        if (partial) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (t0 + c * kChunk + tokA >= tlen) tl[c][0] = tl[c][1] = -CUDART_INF_F;
            if (t0 + c * kChunk + 8 + tokA >= tlen) tl[c][2] = tl[c][3] = -CUDART_INF_F;
          }
        }
        // online softmax with lazy rescale
        float mh0 = fmaxf(fmaxf(tl[0][0], tl[0][2]), fmaxf(tl[1][0], tl[1][2]));
        float mh1 = fmaxf(fmaxf(tl[0][1], tl[0][3]), fmaxf(tl[1][1], tl[1][3]));
#pragma unroll
        for (int m = 4; m <= 16; m <<= 1) {
          mh0 = fmaxf(mh0, __shfl_xor_sync(0xffffffffu, mh0, m));
          mh1 = fmaxf(mh1, __shfl_xor_sync(0xffffffffu, mh1, m));
        }
        const bool n0 = mh0 > m0 + 8.f, n1 = mh1 > m1 + 8.f;  // rescale only when a running max moves by more than 2^8
        if (__any_sync(0xffffffffu, n0 || n1)) {
          const float a0 = n0 ? exp2f(m0 - mh0) : 1.f, a1 = n1 ? exp2f(m1 - mh1) : 1.f;
          if (n0) m0 = mh0;
          if (n1) m1 = mh1;
          l0 *= a0; cr0 *= a0; l1 *= a1; cr1 *= a1;
          spa[0] *= a0; spa[2] *= a0; spa[1] *= a1; spa[3] *= a1;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            o[i][0] *= a0; o[i][2] *= a0;
            o[i][1] *= a1; o[i][3] *= a1;
          }
        }
        uint32_t bp[2][2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float pA0 = ex2_approx(tl[c][0] - m0), pA1 = ex2_approx(tl[c][1] - m1);
          const float pB0 = ex2_approx(tl[c][2] - m0), pB1 = ex2_approx(tl[c][3] - m1);
          l0 += pA0 + pB0; l1 += pA1 + pB1;
          cr0 = fmaf(pA0, vc[c][0], fmaf(pB0, vc[c][1], cr0));
          cr1 = fmaf(pA1, vc[c][0], fmaf(pB1, vc[c][1], cr1));
          // P' = p * s_v rounded to fp16 (the MMA operand); its exact sum removes the 1024 bias of the V operand afterwards
          const uint32_t hA = pack_f2h2(pA0 * vs[c][0], pA1 * vs[c][0]), hB = pack_f2h2(pB0 * vs[c][1], pB1 * vs[c][1]);
          // P'^T fragments: transpose the (token, head) tiles so that tokens become the MMA k index
          bp[c][0] = movmatrix_trans(hA);  // k = 2q4, 2q4+1  <-> chunk tokens q4, 4+q4
          bp[c][1] = movmatrix_trans(hB);  // k = 2q4+8, +9   <-> chunk tokens 8+q4, 12+q4
          // sum_t p'_t per head, from the very operand the V MMAs consume: an all-ones A tile (every output row is the sum)
          mma_full(spa[0], spa[1], spa[2], spa[3], kOnesH2, kOnesH2, kOnesH2, kOnesH2, bp[c][0], bp[c][1]);
        }
        // ---- O^T += V^T P'^T on biased codes: 2 x 8 MMAs (m-tile = 16 dims) ----
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const uint8_t* vbase = st + SL::kOffV + (c * kChunk + q4) * kRow;
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
                mma_full(o[i][0], o[i][1], o[i][2], o[i][3], lop3_and_or(m01, 0x000f000fu, kMagic), lop3_and_or(m01, 0x00f000f0u, kMagic),
                         lop3_and_or(m89, 0x000f000fu, kMagic), lop3_and_or(m89, 0x00f000f0u, kMagic), bp[c][0], bp[c][1]);
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
              mma_full(o[i][0], o[i][1], o[i][2], o[i][3], lop3_and_or(__byte_perm(wa[w], wb[w], sel0), 0x00ff00ffu, kMagic),
                       lop3_and_or(__byte_perm(wa[w], wb[w], sel1), 0x00ff00ffu, kMagic), lop3_and_or(__byte_perm(wc[w], wd[w], sel0), 0x00ff00ffu, kMagic),
                       lop3_and_or(__byte_perm(wc[w], wd[w], sel1), 0x00ff00ffu, kMagic), bp[c][0], bp[c][1]);
            }
          }
        }
      }
      __syncwarp();
      // refill the slot just consumed with the slice R iterations ahead
      if (j + R < n_my) {
        if (((j + R) & 31) == 0) load_ptr_batch(j + R);
        issue(j + R, s);
      }
      if (++s == R) { s = 0; ph ^= 1; }
    }

    if (threadIdx.x == 0) ATTN_PROF(6);
    // ---- per-warp partials -> the warp's own (drained) ring: no need to wait for the other warps ----
#pragma unroll
    for (int m = 4; m <= 16; m <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, m);
      l1 += __shfl_xor_sync(0xffffffffu, l1, m);
      cr0 += __shfl_xor_sync(0xffffffffu, cr0, m);
      cr1 += __shfl_xor_sync(0xffffffffu, cr1, m);
    }
    if (g == 0) {
      s_m[warp][2 * q4] = m0; s_m[warp][2 * q4 + 1] = m1;
      s_l[warp][2 * q4] = l0; s_l[warp][2 * q4 + 1] = l1;
    }
    {
      // layout [warp][head][(d % 16) * 8 + d / 16] with a head stride of 132 floats: conflict-free for these stores and for the
      // merge reads below (thread t owns dim 16 (t % 8) + t / 8)
      __syncwarp();  // every lane is done with the ring slots this overwrites
      float* so0 = reinterpret_cast<float*>(my_ring) + (2 * q4) * kOStride + g;  // head 2q4, dims 16g + j at offset 8 j
      float* so1 = so0 + kOStride;                                // head 2q4+1
      constexpr float hs = (BITS == 4) ? 0.0625f : 1.f;
      const float b0 = 1024.f * spa[0], b1 = 1024.f * spa[1];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        // remove the operand bias (1024 sum p'); KV4: the odd dims came from the high nibbles, i.e. 16 x the code
        so0[8 * (2 * i)] = (o[i][0] - b0) + cr0; so0[8 * (2 * i + 1)] = (o[i][2] - b0) * hs + cr0;
        so1[8 * (2 * i)] = (o[i][1] - b1) + cr1; so1[8 * (2 * i + 1)] = (o[i][3] - b1) * hs + cr1;
      }
    }
    // new token logit: fp32 dot of the rotated, un-quantised q and k  (Template.hpp:1410-1441)
    if (split == 0) {
      for (int r = warp; r < Gc; r += kWarps) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc = fmaf(__half2float(s_q[r * kD + lane * 4 + j]), __half2float(s_k[lane * 4 + j]), acc);
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
        if (lane == 0) {
          s_m[kWarps][r] = acc * sm_scale;
          s_l[kWarps][r] = 1.f;
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) ATTN_PROF(7);

  // ---------------- merge the warps (and the un-quantised new token) ----------------
  const bool owner = (split == 0);
  const int nparts = kWarps + (owner ? 1 : 0);
  if (threadIdx.x < kMaxG) {
    // one thread per head: weights exp2(m_w - M), normalised by 1 / (sum + 1e-6) when this CTA produces the final output
    const int r = threadIdx.x;
    float M = -CUDART_INF_F;
    for (int w = 0; w < nparts; ++w) M = fmaxf(M, s_m[w][r]);
    float e[kWarps + 1], L = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps + 1; ++w) {
      e[w] = (w < nparts && s_m[w][r] != -CUDART_INF_F) ? exp2f(s_m[w][r] - M) : 0.f;
      if (w < nparts) L += s_l[w][r] * e[w];
    }
    // reference normalisation: 1 / (sum + 1e-6)   (Template.hpp:1818)
    const float inv = (nsplit == 1) ? __fdividef(1.f, L + 1.e-6f) : 1.f;
#pragma unroll
    for (int w = 0; w < kWarps + 1; ++w) s_f[w][r] = e[w] * inv;
    s_m[0][r] = M;   // only read back by the split path below
    s_l[0][r] = L;
  }
  __syncthreads();
  if (threadIdx.x < kD) {
    const int d = 16 * (threadIdx.x & 7) + (threadIdx.x >> 3);  // the dim whose partials sit at offset threadIdx.x
    float* part = nullptr;
    if (nsplit > 1) part = ws_part + ((static_cast<size_t>(b) * num_heads + h0) * nsplit + split) * (kD + 2);
    const float vd = __half2float(s_v[d]);
#pragma unroll
    for (int r = 0; r < kMaxG; ++r) {
      if (r < Gc) {
        float acc = s_f[kWarps][r] * vd;
#pragma unroll
        for (int w = 0; w < kWarps; ++w)
          acc = fmaf(reinterpret_cast<const float*>(s_ring + w * SL::kWarpBytes)[r * kOStride + threadIdx.x], s_f[w][r], acc);
        if (nsplit == 1) {
          out[(static_cast<size_t>(b) * num_heads + h0 + r) * kD + d] = __float2half_rn(acc);
        } else {
          float* pr = part + static_cast<size_t>(r) * nsplit * (kD + 2);
          pr[d] = acc;
          if (threadIdx.x == 0) {
            pr[kD] = s_m[0][r];
            pr[kD + 1] = s_l[0][r];
          }
        }
      }
    }
  }
  qs_trace(QS_K_ATTN, 2);
  if (threadIdx.x == 0) ATTN_PROF(8);
  bool final_written = (nsplit == 1);  // this CTA produced the final fp16 outputs of its head group
  if (nsplit > 1) {
    __threadfence();
    __syncthreads();
    uint32_t* cnt = ws_cnt + static_cast<size_t>(b) * gridDim.x + blockIdx.x;
    if (threadIdx.x == 0) {
      const uint32_t old = atomicAdd(cnt, 1u);
      const bool last = (old == static_cast<uint32_t>(nsplit - 1));
      if (last) *cnt = 0;
      s_last = last ? 1u : 0u;
    }
    __syncthreads();
    final_written = (s_last != 0);
    if (s_last && threadIdx.x < kD) {
      const int d = threadIdx.x;
      __threadfence();
      for (int r = 0; r < Gc; ++r) {
        const float* pr = ws_part + (static_cast<size_t>(b) * num_heads + h0 + r) * nsplit * (kD + 2);
        float M = -CUDART_INF_F;
        for (int sp = 0; sp < nsplit; ++sp) M = fmaxf(M, __ldcg(pr + sp * (kD + 2) + kD));
        float L = 0.f, acc = 0.f;
        for (int sp = 0; sp < nsplit; ++sp) {
          const float ms = __ldcg(pr + sp * (kD + 2) + kD);
          const float e = (ms == -CUDART_INF_F) ? 0.f : exp2f(ms - M);
          L += __ldcg(pr + sp * (kD + 2) + kD + 1) * e;
          acc += __ldcg(pr + sp * (kD + 2) + d) * e;
        }
        out[(static_cast<size_t>(b) * num_heads + h0 + r) * kD + d] = __float2half_rn(acc * __fdividef(1.f, L + 1.e-6f));
      }
    }
  }
  if (q_out != nullptr && final_written) {
    // ---- fused per-token INT8 quantisation of the attention output (invoke_quant[_fuse_sum], fused_kernels.cu:92-137).
    //      `out` is an fp16 scratch row in the workspace (L2 resident); the last head-group CTA of a token to finish
    //      re-reads the row and quantises it: same arithmetic as quant_per_token_kernel ----
    __shared__ uint32_t s_last_tok;
    __shared__ float s_red_f[8];
    __shared__ long long s_red_l[8];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const uint32_t old = atomicAdd(tok_cnt + b, 1u);
      const bool last = (old == gridDim.x - 1);
      if (last) tok_cnt[b] = 0;
      s_last_tok = last ? 1u : 0u;
    }
    __syncthreads();
    if (s_last_tok) {
      __threadfence();
      const int nvec = num_heads * kD / 8;
      const uint4* row = reinterpret_cast<const uint4*>(out + static_cast<size_t>(b) * num_heads * kD);
      // one pass: the row (<= kRowRegs x 128 vectors: up to 64 query heads) stays in registers between the statistics and the quantisation
      constexpr int kRowRegs = 8;
      const bool in_regs = nvec <= kRowRegs * kAttnThreadsV2;
      uint4 rv[kRowRegs];
      float amax = 0.f;
      long long sum = 0;
      auto stats = [&](const uint4& v) {
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          if (q_sum) sum += __float2ll_rn(f.x * 16777216.f) + __float2ll_rn(f.y * 16777216.f);
          amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
        }
      };
      if (in_regs) {
#pragma unroll
        for (int c = 0; c < kRowRegs; ++c) {
          const int i = threadIdx.x + c * kAttnThreadsV2;
          rv[c] = (i < nvec) ? __ldcg(row + i) : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int c = 0; c < kRowRegs; ++c)
          if (threadIdx.x + c * kAttnThreadsV2 < nvec) stats(rv[c]);
      } else {
        for (int i = threadIdx.x; i < nvec; i += kAttnThreadsV2) stats(__ldcg(row + i));
      }
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, m));
        sum += __shfl_xor_sync(0xffffffffu, sum, m);
      }
      if (lane == 0) { s_red_f[warp] = amax; s_red_l[warp] = sum; }
      __syncthreads();
      amax = 0.f;
      sum = 0;
      for (int w = 0; w < kAttnThreadsV2 / 32; ++w) { amax = fmaxf(amax, s_red_f[w]); sum += s_red_l[w]; }
      if (threadIdx.x == 0) {
        q_scale[b] = __float2half_rn(__fdiv_rn(amax, 127.f));
        if (q_sum) q_sum[b] = __float2half_rn(__ll2float_rn(sum) * (1.f / 16777216.f));
      }
      const float qs_ = __fdiv_rn(127.f, amax);
      uint2* qrow = reinterpret_cast<uint2*>(q_out + static_cast<size_t>(b) * num_heads * kD);
      auto quantise = [&](int i, const uint4& v) {
        const __half* h = reinterpret_cast<const __half*>(&v);
        uint32_t w[2] = {0u, 0u};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          int32_t c;
          asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(c) : "f"(__fmul_rn(__half2float(h[j]), qs_)));
          w[j >> 2] |= (static_cast<uint32_t>(c) & 0xffu) << ((j & 3) * 8);
        }
        qrow[i] = make_uint2(w[0], w[1]);
      };
      if (in_regs) {
#pragma unroll
        for (int c = 0; c < kRowRegs; ++c) {
          const int i = threadIdx.x + c * kAttnThreadsV2;
          if (i < nvec) quantise(i, rv[c]);
        }
      } else {
        for (int i = threadIdx.x; i < nvec; i += kAttnThreadsV2) quantise(i, __ldcg(row + i));
      }
    }
  }
  if (threadIdx.x == 0) ATTN_PROF(9);
#undef ATTN_PROF
}

// ------------------------------------------------------------------------------------------------
// K2: prefill RoPE + KV quantise + page append: one warp per (token, KV head): it rotates the G query heads of the group and the key head with
//     ONE evaluation of the position's sines / cosines (the first version, one warp per query head, spent its time in 32 redundant
//     powf / sincosf per token: 365 us per layer for the 8 x 1024-token prompt batch), then quantises and appends K and V.
//     applyBiasRopeUpdateKVCache.h:94-455 (STORE_QKV = true, no bias, NeoX)
// ------------------------------------------------------------------------------------------------
template <int BITS, bool AT>  // AT: start_pos is given (qs_apply_bias_rope_update_kv_cache_at); otherwise it is ignored
__global__ void __launch_bounds__(128) prefill_append_kernel(__half* __restrict__ qkv, const int* __restrict__ seq_lens,
                                                             const int* __restrict__ padding_offset, const long long* __restrict__ kv_pointers,
                                                             const int* __restrict__ start_pos, int num_tokens, int max_blocks, int num_heads, int num_kv_heads, int seq_len,
                                                             PageGeom pg, float rotary_base, int rotary_dim, int max_positions) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int G = num_heads / num_kv_heads;
  const int warps_per_cta = blockDim.x >> 5;
  const long long n_work = static_cast<long long>(num_tokens) * num_kv_heads;
  const int n = (num_heads + 2 * num_kv_heads) * kD;
  const int half_rot = rotary_dim / 2;
  for (long long wi = static_cast<long long>(blockIdx.x) * warps_per_cta + (threadIdx.x >> 5); wi < n_work;
       wi += static_cast<long long>(gridDim.x) * warps_per_cta) {
    const int token = static_cast<int>(wi / num_kv_heads), kvh = static_cast<int>(wi - static_cast<long long>(token) * num_kv_heads);
    const int gtok = token + (padding_offset ? padding_offset[token] : 0);
    const int bidx = gtok / seq_len, cpos = gtok - bidx * seq_len;
    const int clen = seq_lens[bidx];
    if (cpos >= clen) continue;  // padded slot (cannot happen with un-padded inputs)
    // with start_pos (a chunk appended behind start_pos[b] cached tokens) the position and the total length are shifted; the RoPE angle, the
    // page / slot and the cyclic window all use the shifted values, so appending a prompt in chunks gives the bytes of a one-shot append
    const int start = AT ? __ldg(start_pos + bidx) : 0;
    const int pos = start + cpos, len = start + clen;
    __half* trow = qkv + static_cast<size_t>(token) * n;
    // lane handles rotary pairs i = 2*lane, 2*lane+1  (i in [0, 64)) -> dims i and i + half_rot: one half2 at each end
    float cs[2], sn[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int i = 2 * lane + e;
      const float inv_freq = __fdiv_rn(static_cast<float>(pos), powf(rotary_base, __fdiv_rn(static_cast<float>(2 * i), static_cast<float>(rotary_dim))));
      sincosf(inv_freq, &sn[e], &cs[e]);
    }
    auto rotate = [&](__half* row, float (&lo)[2], float (&hi)[2]) {  // in place; returns the rotated values (rounded to fp16) as floats
      __half2* p0 = reinterpret_cast<__half2*>(row + 2 * lane);
      __half2* p1 = reinterpret_cast<__half2*>(row + half_rot + 2 * lane);
      const float2 a = __half22float2(*p0), b = __half22float2(*p1);
      const float x0[2] = {a.x, a.y}, x1[2] = {b.x, b.y};
      __half r0[2], r1[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        r0[e] = __float2half_rn(__fsub_rn(__fmul_rn(cs[e], x0[e]), __fmul_rn(sn[e], x1[e])));
        r1[e] = __float2half_rn(__fadd_rn(__fmul_rn(cs[e], x1[e]), __fmul_rn(sn[e], x0[e])));
        lo[e] = __half2float(r0[e]);
        hi[e] = __half2float(r1[e]);
      }
      *p0 = __halves2half2(r0[0], r0[1]);
      *p1 = __halves2half2(r1[0], r1[1]);
    };
    float t0[2], t1[2];
    for (int g = 0; g < G; ++g) rotate(trow + static_cast<size_t>(kvh * G + g) * kD, t0, t1);
    float kx[4], vx[4];  // dims 2l, 2l+1, 64+2l, 65+2l
    rotate(trow + static_cast<size_t>(num_heads + kvh) * kD, t0, t1);
    kx[0] = t0[0]; kx[1] = t0[1]; kx[2] = t1[0]; kx[3] = t1[1];
    {
      const __half* vrow = trow + static_cast<size_t>(num_heads + num_kv_heads + kvh) * kD;
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(vrow + 2 * lane));
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(vrow + half_rot + 2 * lane));
      vx[0] = a.x; vx[1] = a.y; vx[2] = b.x; vx[3] = b.y;
    }
    if (kv_pointers == nullptr) continue;
    if (pos < max(len - max_positions, 0)) continue;  // outside the cyclic window (:268-271)
    const int blk = pos / pg.tokens_per_block, slot = pos - blk * pg.tokens_per_block;
    const float L = (BITS == 4) ? 15.f : 255.f;
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      const float* x = which ? vx : kx;
      float mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3]));
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, m));
      }
      __half sc, zp;
      kv_quant_params(mx, mn, L, sc, zp);
      const float inv_s = __fdiv_rn(1.0f, __half2float(sc)), zf = __half2float(zp);
      uint8_t* page = reinterpret_cast<uint8_t*>(kv_pointers[(static_cast<size_t>(bidx) * 2 + which) * max_blocks + blk]);
      const uint32_t c0 = kv_quant_code(x[0], inv_s, zf), c1 = kv_quant_code(x[1], inv_s, zf);
      const uint32_t c2 = kv_quant_code(x[2], inv_s, zf), c3 = kv_quant_code(x[3], inv_s, zf);
      if constexpr (BITS == 4) {
        uint8_t* row = page + static_cast<size_t>(kvh * pg.tokens_per_block + slot) * (kD / 2);
        row[lane] = static_cast<uint8_t>((c0 & 0xF) | ((c1 & 0xF) << 4));        // dims 2l, 2l+1
        row[32 + lane] = static_cast<uint8_t>((c2 & 0xF) | ((c3 & 0xF) << 4));   // dims 64+2l, 65+2l
      } else {
        uint8_t* row = page + static_cast<size_t>(kvh * pg.tokens_per_block + slot) * kD;
        reinterpret_cast<uint16_t*>(row)[lane] = static_cast<uint16_t>(c0 | (c1 << 8));
        reinterpret_cast<uint16_t*>(row + 64)[lane] = static_cast<uint16_t>(c2 | (c3 << 8));
      }
      if (lane == 0) {
        __half* meta = reinterpret_cast<__half*>(page + pg.code_bytes);
        meta[kvh * pg.tokens_per_block + slot] = sc;
        meta[pg.num_kv_heads * pg.tokens_per_block + kvh * pg.tokens_per_block + slot] = zp;
      }
    }
  }
}

__global__ void padding_offsets_kernel(int* __restrict__ out, const int* __restrict__ cu_seqlens, int max_seqlen) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const int beg = cu_seqlens[b], end = cu_seqlens[b + 1];
  const int off = b * max_seqlen - beg;
  for (int t = beg + threadIdx.x; t < end; t += blockDim.x) out[t] = off;
}

template <typename Kern, typename... Args>
int launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, void* stream, const char* what, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return check_cuda(cudaLaunchKernelEx(&cfg, kern, args...), what);
}

constexpr size_t kAttnCounterBytes = 256 * 1024;  // 49152 (sequence, head-group) split counters + 16384 per-token counters
constexpr size_t kAttnTokCounterOffset = 192 * 1024;

}  // namespace

size_t attention_workspace_bytes(int batch, int num_heads, int head_dim, int max_splits) {
  return kAttnCounterBytes + static_cast<size_t>(batch) * num_heads * max_splits * (head_dim + 2) * sizeof(float) +
         static_cast<size_t>(batch) * num_heads * head_dim * sizeof(__half);  // + fp16 scratch rows of the fused-quant form
}

int attention_trace_install(void* buf, unsigned cap) { return qs_trace_install(buf, cap); }

int decode_attention(const DecodeAttnArgs& a) {
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.head_dim == kD, "single_query_attention: head_dim=%d, only 128 is supported (as in the reference)", a.head_dim);
  QS_REQUIRE(a.kv_zeros, "single_query_attention: only kv_cache_with_zeros=True is supported (arg_utils.py:422 always sets it)");
  QS_REQUIRE(a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "single_query_attention: heads %d / kv heads %d", a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.tokens_per_block > 0 && a.tokens_per_block % kChunk == 0, "single_query_attention: tokens_per_block=%d must be a multiple of %d",
             a.tokens_per_block, kChunk);
  QS_REQUIRE(a.rotary_dim == kD, "single_query_attention: rotary_dim=%d must equal head_dim (llama_w4a8_unpad.py:258)", a.rotary_dim);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * kD * bits / 8, "single_query_attention: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
  QS_REQUIRE(a.batch <= 65535, "single_query_attention: batch=%d too large", a.batch);
  PageGeom pg{a.tokens_per_block, a.tokens_per_block * a.size_per_token, a.num_kv_heads};
  const int G = a.num_heads / a.num_kv_heads;
  const int gparts = (G + kMaxG - 1) / kMaxG;
  const int gx = a.num_kv_heads * gparts;
  // context splits: enough CTAs to fill the machine (4 resident CTAs per SM), never more than one split per 256 tokens
  int nsplit = 1;
  const int ctas = gx * a.batch;
  const int slots = num_sms() * 4;
  if (2 * ctas <= slots && a.timestep > 512) {
    nsplit = (slots + ctas - 1) / ctas;
    const int cap = (a.timestep + 255) / 256;
    if (nsplit > cap) nsplit = cap;
    if (nsplit > 32) nsplit = 32;
  }
  float* part = nullptr;
  uint32_t* cnt = nullptr;
  if (nsplit > 1) {
    const size_t need = attention_workspace_bytes(a.batch, a.num_heads, kD, nsplit);
    if (a.workspace == nullptr || need > a.workspace_bytes || static_cast<size_t>(a.batch) * gx * 4 > kAttnTokCounterOffset) {
      nsplit = 1;
    } else {
      cnt = static_cast<uint32_t*>(a.workspace);
      part = reinterpret_cast<float*>(static_cast<uint8_t*>(a.workspace) + kAttnCounterBytes);
    }
  }
  const bool fused_quant = a.q_out != nullptr;
  uint32_t* tok_cnt = nullptr;
  void* out = a.out;
  if (fused_quant) {
    QS_REQUIRE(a.q_scale != nullptr, "single_query_attention_quant: q_scale is null");
    const size_t row_bytes = static_cast<size_t>(a.batch) * a.num_heads * kD * sizeof(__half);
    const size_t part_bytes = nsplit > 1 ? attention_workspace_bytes(a.batch, a.num_heads, kD, nsplit) - kAttnCounterBytes - row_bytes : 0;
    QS_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= kAttnCounterBytes + part_bytes + row_bytes && a.batch <= 16384,
               "single_query_attention_quant: workspace too small (need qs_attention_workspace_bytes)");
    tok_cnt = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(a.workspace) + kAttnTokCounterOffset);
    out = static_cast<uint8_t*>(a.workspace) + kAttnCounterBytes + part_bytes;
  }
  dim3 grid(gx, a.batch, nsplit);
  auto run = [&](auto kern, size_t smem) {
    static bool attr_done[2][kMaxDevices] = {};
    bool& done = attr_done[a.int4_kv ? 0 : 1][device_ordinal()];
    if (!done) {
      int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)), "attention smem attribute");
      if (rc) return rc;
      done = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(kAttnThreadsV2);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = static_cast<cudaStream_t>(a.stream);
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = 1;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    return check_cuda(cudaLaunchKernelEx(&cfg, kern, static_cast<const __half*>(a.q),
                      static_cast<const __half*>(a.k), static_cast<const __half*>(a.v), a.q_stride, a.k_stride, a.v_stride, a.kv_pointers, a.lengths,
                      static_cast<__half*>(out), a.num_heads, a.num_kv_heads, a.max_blocks, pg, a.rotary_base, a.rotary_dim, a.timestep, nsplit,
                      part, cnt, tok_cnt, static_cast<int8_t*>(a.q_out), static_cast<__half*>(a.q_scale), static_cast<__half*>(a.q_sum), static_cast<unsigned long long*>(a.prof)), "single_query_attention");
  };
  QS_REQUIRE(a.tokens_per_block == kPageTokens, "single_query_attention: tokens_per_block=%d, only 64 is supported (cache_engine block_size)", a.tokens_per_block);
  return a.int4_kv ? run(decode_attention_kernel<4>, static_cast<size_t>(kWarps) * StageLayout<4>::kWarpBytes)
                   : run(decode_attention_kernel<8>, static_cast<size_t>(kWarps) * StageLayout<8>::kWarpBytes);
}

int prefill_rope_append(const PrefillAppendArgs& a) {
  if (a.num_tokens == 0) return QS_OK;
  QS_REQUIRE(a.head_dim == kD, "apply_bias_rope_update_kv_cache: head_dim=%d, only 128 is supported", a.head_dim);
  QS_REQUIRE(a.kv_zeros, "apply_bias_rope_update_kv_cache: only kv_cache_with_zeros=True is supported");
  QS_REQUIRE(a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "apply_bias_rope_update_kv_cache: heads %d / kv heads %d", a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.rotary_dim == kD, "apply_bias_rope_update_kv_cache: rotary_dim=%d must equal head_dim (update_kv_cache.cu:54)", a.rotary_dim);
  QS_REQUIRE(a.seq_len > 0, "apply_bias_rope_update_kv_cache: seq_len=%d", a.seq_len);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * kD * bits / 8, "apply_bias_rope_update_kv_cache: size_per_token=%d does not match", a.size_per_token);
  PageGeom pg{a.tokens_per_block, a.tokens_per_block * a.size_per_token, a.num_kv_heads};
  const long long work = static_cast<long long>(a.num_tokens) * a.num_kv_heads;  // one warp per (token, KV head)
  long long blocks = (work + 3) / 4;
  if (blocks > static_cast<long long>(num_sms()) * 16) blocks = static_cast<long long>(num_sms()) * 16;
  auto run = [&](auto kern) {
    return launch_pdl(kern, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, a.stream, "apply_bias_rope_update_kv_cache", static_cast<__half*>(a.qkv),
                      a.seq_lens, a.padding_offset, a.kv_pointers, a.start_pos, a.num_tokens, a.max_blocks, a.num_heads, a.num_kv_heads, a.seq_len, pg,
                      a.rotary_base, a.rotary_dim, a.max_positions);
  };
  if (a.start_pos) return a.int4_kv ? run(prefill_append_kernel<4, true>) : run(prefill_append_kernel<8, true>);
  return a.int4_kv ? run(prefill_append_kernel<4, false>) : run(prefill_append_kernel<8, false>);
}

int padding_offsets(int* out, const int* cu_seqlens, int batch, int max_seqlen, void* stream) {
  if (batch == 0) return QS_OK;
  return launch_pdl(padding_offsets_kernel, dim3(batch), dim3(256), 0, stream, "compute_padding_offsets", out, cu_seqlens, max_seqlen);
}

}  // namespace qs
