// qserve_b200 -- causal prompt attention over a cached prefix in the paged INT4 / INT8 KV cache (chunked prefill, prefix reuse), sm_90a.
//
// A batch of prompt CHUNKS: query i of sequence b sits at absolute position P_b + i, where P_b = prefix_lens[b] tokens of the sequence are
// already quantised in the pages.  It attends to the prefix keys 0 .. P_b - 1, dequantised from the pages element for element as the
// reference dequantises them (4 bit: hfma2(u, s, half(-s z)); 8 bit: half(s (u - z))), and to the chunk keys 0 .. i as the un-quantised fp16
// rows of the rotated qkv buffer (what flash-attn sees in the prompt step and what the decode kernel does for its current token).
//
// One CTA = one (sequence, query head, block of 128 chunk rows), 384 threads in three warpgroups:
//   WG0  producer (setmaxnreg 56): one thread per key row.  For a prefix block it loads that token's codes, scale and zero straight from the
//        page into registers and writes 256 B of fp16 into the K or V ring slot in exactly the 128-byte-swizzled [128 rows][64 halfs] x 2 layout
//        a TMA box produces (16-byte chunk c of row r at chunk c ^ (r & 7)); rows >= P_b are written as zeros (unwritten page slots hold
//        arbitrary bytes, and NaN * 0 is NaN).  For a chunk block one elected thread issues the TMA loads, as prefill_attention.cu does.
//   WG1, WG2  consumers (setmaxnreg 224), the two warpgroups of prefill_attention.cu unchanged: S = Q K^T from shared memory, online softmax
//        in registers, O += P V with P from registers and V as the MN-major operand.
// Key blocks: first the ceil(P_b / 128) prefix blocks (keys >= P_b of the last one masked to -inf), then the chunk blocks aligned to the chunk
// start, so that no block mixes prefix and chunk keys and the diagonal mask of the prompt kernel applies unchanged.  No atomics: the result is
// deterministic run to run.  Shared memory: the Q tile and the two-deep K / V ring, 160 KB, as in prefill_attention.cu.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include <climits>

#include "common.cuh"
#include "launch.h"

namespace qs {
namespace {

constexpr int kD = 128;         // head dim
constexpr int kBQ = 128;        // query rows per CTA (two consumer warpgroups x m64)
constexpr int kBKV = 128;       // keys per block
constexpr int kStages = 2;      // K / V ring depth
constexpr int kThreads = 384;   // warps 0..3: producer warpgroup, warps 4..11: two consumer warpgroups
constexpr int kProducers = 128;
constexpr int kPageTokens = 64;
constexpr int kTileBytes = kBQ * kD * 2;      // 32 KB: two swizzled [128 rows x 64 halfs] sub-tiles
constexpr int kSubBytes = kTileBytes / 2;     // 16 KB
constexpr int kOffQ = 0, kOffK = kTileBytes, kOffV = kOffK + kStages * kTileBytes, kOffBar = kOffV + kStages * kTileBytes;
constexpr int kSmemBytes = kOffBar + 128;
// register split of the 64 K-register file: 128 x 56 + 256 x 224 = 64512
constexpr int kProducerRegs = 56, kConsumerRegs = 224;

template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b, float& sum) {
  const __half2 h2 = __floats2half2_rn(a, b);
  const float2 f = __half22float2(h2);  // the row sum is taken over the ROUNDED probabilities, as in prefill_attention.cu
  sum += f.x + f.y;
  return *reinterpret_cast<const uint32_t*>(&h2);
}

struct PrefixAttnParams {
  const int* cu_seqlens;          // [B + 1] chunk token offsets
  const int* prefix_lens;         // [B] tokens already in the cache
  const long long* kv_pointers;   // [B, 2, max_blocks] absolute page addresses
  __half* out;                    // [T, Hq * 128] rows of out_stride halfs
  long long out_stride;
  int num_heads, num_kv_heads, max_blocks;
  int code_bytes;                 // bytes of codes per page (64 * size_per_token)
  float scale_log2;               // softmax scale * log2(e)
};

// Dequantise one cached token of kv head `hkv` (or write zeros when page == nullptr) into row r of a swizzled [128][64] x 2 fp16 tile.
template <int BITS>
__device__ __forceinline__ void dequant_row(uint8_t* tile, int r, const uint8_t* page, int slot, int hkv, const PrefixAttnParams& p) {
  uint8_t* row = tile + r * 128;
  const int sw = r & 7;
  auto store = [&](int c, uint4 v) {  // output chunk c = dims 8c .. 8c + 7
    *reinterpret_cast<uint4*>(row + (c >> 3) * kSubBytes + (((c & 7) ^ sw) << 4)) = v;
  };
  if (page == nullptr) {
#pragma unroll
    for (int c = 0; c < kD / 8; ++c) store(c, make_uint4(0u, 0u, 0u, 0u));
    return;
  }
  const __half* meta = reinterpret_cast<const __half*>(page + p.code_bytes);
  const __half s = meta[hkv * kPageTokens + slot];
  const __half z = meta[(p.num_kv_heads + hkv) * kPageTokens + slot];
  constexpr int kRow = kD * BITS / 8;
  const uint4* codes = reinterpret_cast<const uint4*>(page + static_cast<size_t>(hkv * kPageTokens + slot) * kRow);
  if constexpr (BITS == 4) {
    // x = fma_f16(half(u), s, half(-float(s) * float(z))): one fp16 rounding, as kv_dequant
    const __half c = __float2half_rn(__fmul_rn(-__half2float(s), __half2float(z)));
    const __half2 s2 = __halves2half2(s, s), c2 = __halves2half2(c, c);
    const __half2 magic = __float2half2_rn(1024.f);
#pragma unroll
    for (int q = 0; q < kRow / 16; ++q) {
      const uint4 w = codes[q];
      const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {  // word e: 8 dims, nibble d = dim d (byte i holds dims 2i low, 2i + 1 high)
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t x = ws[e] >> (8 * i);
          const uint32_t bits = (x & 0xFu) | ((x & 0xF0u) << 12) | 0x64006400u;  // half2(1024 + lo, 1024 + hi)
          const __half2 u = __hsub2(*reinterpret_cast<const __half2*>(&bits), magic);  // exact
          const __half2 v = __hfma2(u, s2, c2);
          o[i] = *reinterpret_cast<const uint32_t*>(&v);
        }
        store(4 * q + e, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  } else {
    // x = half(float(s) * (float(u) - float(z))), fp32 steps rounded as kv_dequant
    const float sf = __half2float(s), zf = __half2float(z);
#pragma unroll
    for (int q = 0; q < kRow / 16; ++q) {
      const uint4 w = codes[q];
      const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int hc = 0; hc < 2; ++hc) {  // 16 codes = two output chunks
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t x = ws[2 * hc + (i >> 1)] >> (16 * (i & 1));
          const float lo = __fmul_rn(sf, __fsub_rn(static_cast<float>(x & 0xFFu), zf));
          const float hi = __fmul_rn(sf, __fsub_rn(static_cast<float>((x >> 8) & 0xFFu), zf));
          const __half2 v = __halves2half2(__float2half_rn(lo), __float2half_rn(hi));
          o[i] = *reinterpret_cast<const uint32_t*>(&v);
        }
        store(2 * q + hc, make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

template <int BITS>
__global__ void __launch_bounds__(kThreads, 1)
prefix_attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const PrefixAttnParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int b = blockIdx.z, h = blockIdx.y;
  const int seq_start = __ldg(p.cu_seqlens + b);
  const int seq_len = __ldg(p.cu_seqlens + b + 1) - seq_start;
  const int n_qb = (seq_len + kBQ - 1) / kBQ;
  const int qb = n_qb - 1 - static_cast<int>(blockIdx.x);  // the longest (last) query blocks of a chunk are scheduled first
  if (qb < 0) return;                                      // uniform per CTA
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
  const int hkv = h / (p.num_heads / p.num_kv_heads);
  // prefix_lens is prepared by the host before the step (like the page table): read before the dependency wait
  const int P = __ldg(p.prefix_lens + b);
  const int n_pb = (P + kBKV - 1) / kBKV;  // prefix key blocks
  const int n_kb = n_pb + qb + 1;          // + causal chunk key blocks 0 .. qb

  uint8_t* s_q = smem + kOffQ;
  uint8_t* s_k = smem + kOffK;
  uint8_t* s_v = smem + kOffV;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* bar_q = bar;                      // Q tile landed
  uint64_t* bar_kfull = bar + 1;              // [kStages] K block ready: 128 producer arrivals (+ TMA bytes for a chunk block)
  uint64_t* bar_kfree = bar_kfull + kStages;  // [kStages] S = Q K^T retired in all eight consumer warps
  uint64_t* bar_vfull = bar_kfree + kStages;
  uint64_t* bar_vfree = bar_vfull + kStages;  // O += P V retired in all eight consumer warps

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(bar_q, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&bar_kfull[i], kProducers);
      mbar_init(&bar_kfree[i], 8);
      mbar_init(&bar_vfull[i], kProducers);
      mbar_init(&bar_vfree[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp < 4) {
    // ===================================== producer warpgroup: thread r fills key row r of every block =====================================
    setmaxnreg_dec<kProducerRegs>();
    const int r = threadIdx.x;
    const long long* kptrs = p.kv_pointers + static_cast<size_t>(b) * 2 * p.max_blocks;
    const long long* vptrs = kptrs + p.max_blocks;
    long long kpg = 0, vpg = 0;  // page addresses of this thread's token of the current prefix block
    if (r < P) {
      kpg = kptrs[r / kPageTokens];
      vpg = vptrs[r / kPageTokens];
    }
    pdl_wait();  // page contents and q / k / v are written by the preceding kernel (RoPE + KV append)
    if (r == 0) {
      const int q_row = seq_start + qb * kBQ;
      mbar_expect_tx(bar_q, kTileBytes);
      tma_load_2d(s_q, &tmap_q, h * kD, q_row, bar_q);
      tma_load_2d(s_q + kSubBytes, &tmap_q, h * kD + 64, q_row, bar_q);
    }
    for (int j = 0; j < n_kb; ++j) {
      const int st = j % kStages;
      const uint32_t ph = static_cast<uint32_t>(j / kStages) & 1u;
      uint8_t* sk = s_k + st * kTileBytes;
      uint8_t* sv = s_v + st * kTileBytes;
      if (j < n_pb) {
        const int t = j * kBKV + r;
        const bool live = t < P;
        const int slot = t & (kPageTokens - 1);
        if (j >= kStages) mbar_wait(&bar_kfree[st], ph ^ 1u);
        dequant_row<BITS>(sk, r, live ? reinterpret_cast<const uint8_t*>(kpg) : nullptr, slot, hkv, p);
        fence_proxy_async();  // generic-proxy writes, read by wgmma through the async proxy
        mbar_arrive(&bar_kfull[st]);
        if (j >= kStages) mbar_wait(&bar_vfree[st], ph ^ 1u);
        dequant_row<BITS>(sv, r, live ? reinterpret_cast<const uint8_t*>(vpg) : nullptr, slot, hkv, p);
        fence_proxy_async();
        mbar_arrive(&bar_vfull[st]);
        const int tn = t + kBKV;
        if (tn < P) {
          kpg = kptrs[tn / kPageTokens];
          vpg = vptrs[tn / kPageTokens];
        }
      } else {
        const int k_row = seq_start + (j - n_pb) * kBKV;
        if (j >= kStages) mbar_wait(&bar_kfree[st], ph ^ 1u);
        if (r == 0) {
          mbar_expect_tx(&bar_kfull[st], kTileBytes);
          tma_load_2d(sk, &tmap_k, hkv * kD, k_row, &bar_kfull[st]);
          tma_load_2d(sk + kSubBytes, &tmap_k, hkv * kD + 64, k_row, &bar_kfull[st]);
        } else {
          mbar_arrive(&bar_kfull[st]);
        }
        if (j >= kStages) mbar_wait(&bar_vfree[st], ph ^ 1u);
        if (r == 0) {
          mbar_expect_tx(&bar_vfull[st], kTileBytes);
          tma_load_2d(sv, &tmap_v, hkv * kD, k_row, &bar_vfull[st]);
          tma_load_2d(sv + kSubBytes, &tmap_v, hkv * kD + 64, k_row, &bar_vfull[st]);
        } else {
          mbar_arrive(&bar_vfull[st]);
        }
      }
    }
    return;
  }

  // ===================================== consumers: warpgroup g owns query rows [64 g, 64 g + 64) of the block =====================================
  setmaxnreg_inc<kConsumerRegs>();
  const int cw = warp - 4;
  const int g = cw >> 2;
  const int row_a = g * 64 + (cw & 3) * 16 + (lane >> 2);  // this thread's two rows: row_a and row_a + 8
  const int q_pos_a = qb * kBQ + row_a, q_pos_b = q_pos_a + 8;  // positions within the chunk
  const int col0 = (lane & 3) * 2;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_a = -CUDART_INF_F, m_b = -CUDART_INF_F;  // running maxima (log2 domain, scaled)
  float l_a = 0.f, l_b = 0.f;                      // this thread's share of the row sums
  mbar_wait(bar_q, 0);
  for (int j = 0; j < n_kb; ++j) {
    const int st = j % kStages;
    const uint32_t ph = static_cast<uint32_t>(j / kStages) & 1u;
    const uint8_t* sk = s_k + st * kTileBytes;
    const uint8_t* sv = s_v + st * kTileBytes;
    mbar_wait(&bar_kfull[st], ph);
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
    if (lane == 0) mbar_arrive(&bar_kfree[st]);

    // ---- masks: keys >= P of the last prefix block; the causal diagonal of the chunk.  Key k is visible to a row iff k <= lim ----
    const bool pre = j < n_pb;
    const int kbase = (pre ? j : j - n_pb) * kBKV;
    const bool masked = pre ? (kbase + kBKV > P) : (j - n_pb == qb);
    const int lim_a = pre ? P - 1 : q_pos_a, lim_b = pre ? P - 1 : q_pos_b;
    float mx_a = -CUDART_INF_F, mx_b = -CUDART_INF_F;
#pragma unroll
    for (int c = 0; c < kBKV / 8; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + c * 8 + col0 + (e & 1);
        float& v = s[c * 4 + e];
        if (e < 2) {
          if (masked && key > lim_a) v = -CUDART_INF_F;  // -inf: exp2 turns it into an exact 0
          mx_a = fmaxf(mx_a, v);
        } else {
          if (masked && key > lim_b) v = -CUDART_INF_F;
          mx_b = fmaxf(mx_b, v);
        }
      }
#pragma unroll
    for (int sh = 1; sh <= 2; sh <<= 1) {
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, sh));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, sh));
    }
    // the first key of every block (prefix key 128 j < P, or chunk key 128 jj <= q_pos) is visible: the maxima are finite from block 0 on
    const float mn_a = fmaxf(m_a, mx_a * p.scale_log2), mn_b = fmaxf(m_b, mx_b * p.scale_log2);
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
    uint32_t pa[kBKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float* sc = s + (2 * kk + hf) * 4;
        pa[kk][2 * hf + 0] = pack_half2(ex2_approx(fmaf(sc[0], p.scale_log2, -m_a)), ex2_approx(fmaf(sc[1], p.scale_log2, -m_a)), l_a);
        pa[kk][2 * hf + 1] = pack_half2(ex2_approx(fmaf(sc[2], p.scale_log2, -m_b)), ex2_approx(fmaf(sc[3], p.scale_log2, -m_b)), l_b);
      }
    mbar_wait(&bar_vfull[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBKV / 16; ++kk) wgmma_f16_rs_n128_tb(o, pa[kk], gmma_desc_sw128(smem_u32(sv + kk * 2048), kSubBytes));
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_vfree[st]);
  }
  // ---- epilogue: O / l -> fp16 ----
#pragma unroll
  for (int sh = 1; sh <= 2; sh <<= 1) {
    l_a += __shfl_xor_sync(0xffffffffu, l_a, sh);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, sh);
  }
  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
  __half* dst_a = p.out + static_cast<long long>(seq_start + q_pos_a) * p.out_stride + h * kD + col0;
  __half* dst_b = dst_a + 8 * p.out_stride;
  const bool valid_a = q_pos_a < seq_len, valid_b = q_pos_b < seq_len;
#pragma unroll
  for (int c = 0; c < kD / 8; ++c) {
    if (valid_a) *reinterpret_cast<__half2*>(dst_a + c * 8) = __floats2half2_rn(o[c * 4 + 0] * inv_a, o[c * 4 + 1] * inv_a);
    if (valid_b) *reinterpret_cast<__half2*>(dst_b + c * 8) = __floats2half2_rn(o[c * 4 + 2] * inv_b, o[c * 4 + 3] * inv_b);
  }
}

}  // namespace

int prefix_attention(const PrefixAttnArgs& a) {
  QS_REQUIRE(a.head_dim == kD, "prefix_prefill_attention: head_dim=%d (only 128 is built)", a.head_dim);
  QS_REQUIRE(a.num_heads > 0 && a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "prefix_prefill_attention: heads=%d kv_heads=%d", a.num_heads,
             a.num_kv_heads);
  QS_REQUIRE(a.batch >= 0 && a.num_tokens >= 0 && a.max_seqlen >= 0 && a.max_prefix_len >= 0, "prefix_prefill_attention: negative size");
  QS_REQUIRE(a.tokens_per_block == kPageTokens, "prefix_prefill_attention: tokens_per_block=%d, only 64 is supported", a.tokens_per_block);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * kD * bits / 8, "prefix_prefill_attention: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
  QS_REQUIRE(static_cast<long long>(a.max_prefix_len) + a.max_seqlen <= static_cast<long long>(a.max_blocks) * kPageTokens,
             "prefix_prefill_attention: max_prefix_len %d + max_seqlen %d exceed the page table (%d blocks of %d tokens)", a.max_prefix_len, a.max_seqlen,
             a.max_blocks, kPageTokens);
  if (a.batch == 0 || a.num_tokens == 0 || a.max_seqlen == 0) return QS_OK;
  QS_REQUIRE(a.batch <= 65535 && a.num_heads <= 65535, "prefix_prefill_attention: batch=%d / heads=%d exceed the grid limits", a.batch, a.num_heads);
  QS_REQUIRE(a.q && a.k && a.v && a.out && a.cu_seqlens && a.prefix_lens && a.kv_pointers, "prefix_prefill_attention: null pointer");
  QS_REQUIRE(a.q_stride % 8 == 0 && a.k_stride % 8 == 0 && a.v_stride % 8 == 0 && a.out_stride % 8 == 0,
             "prefix_prefill_attention: row strides must be multiples of 8 halfs");
  QS_REQUIRE(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) | reinterpret_cast<uintptr_t>(a.out)) & 15) == 0,
             "prefix_prefill_attention: q, k, v, out must be 16-byte aligned");
  QS_REQUIRE(a.q_stride >= a.num_heads * kD && a.k_stride >= a.num_kv_heads * kD && a.v_stride >= a.num_kv_heads * kD && a.out_stride >= a.num_heads * kD,
             "prefix_prefill_attention: row stride smaller than the row");
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_f16(&tq, a.q, a.num_tokens, static_cast<uint64_t>(a.num_heads) * kD, a.q_stride);
  if (rc) return rc;
  rc = make_tmap_f16(&tk, a.k, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.k_stride);
  if (rc) return rc;
  rc = make_tmap_f16(&tv, a.v, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.v_stride);
  if (rc) return rc;
  PrefixAttnParams p{};
  p.cu_seqlens = a.cu_seqlens;
  p.prefix_lens = a.prefix_lens;
  p.kv_pointers = a.kv_pointers;
  p.out = static_cast<__half*>(a.out);
  p.out_stride = a.out_stride;
  p.num_heads = a.num_heads;
  p.num_kv_heads = a.num_kv_heads;
  p.max_blocks = a.max_blocks;
  p.code_bytes = kPageTokens * a.size_per_token;
  p.scale_log2 = a.softmax_scale * 1.4426950408889634f;
  auto run = [&](auto kern) {
    static bool attr_set[2][kMaxDevices] = {};
    bool& done = attr_set[a.int4_kv ? 0 : 1][device_ordinal()];
    if (!done) {
      const int r = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes), "cudaFuncSetAttribute(prefix attention)");
      if (r) return r;
      done = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((a.max_seqlen + kBQ - 1) / kBQ, a.num_heads, a.batch);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmemBytes;
    cfg.stream = static_cast<cudaStream_t>(a.stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return check_cuda(cudaLaunchKernelEx(&cfg, kern, tq, tk, tv, p), "prefix prefill attention launch");
  };
  return a.int4_kv ? run(prefix_attention_kernel<4>) : run(prefix_attention_kernel<8>);
}

}  // namespace qs
