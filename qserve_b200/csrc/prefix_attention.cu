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
//   WG1, WG2  consumers (setmaxnreg 224), the two warpgroups of prompt_attention.cuh that prefill_attention.cu runs too: S = Q K^T from
//        shared memory, online softmax in registers, O += P V with P from registers and V as the MN-major operand.
// Key blocks: first the ceil(P_b / 128) prefix blocks (keys >= P_b of the last one masked to -inf), then the chunk blocks aligned to the chunk
// start, so that no block mixes prefix and chunk keys and the diagonal mask of the prompt kernel applies unchanged.  No atomics: the result is
// deterministic run to run.  Shared memory: the Q tile and the two-deep K / V ring, 160 KB, as in prefill_attention.cu.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <climits>

#include "common.cuh"
#include "launch.cuh"
#include "prompt_attention.cuh"

namespace qs {
namespace {

constexpr int kThreads = 384;   // warps 0..3: producer warpgroup, warps 4..11: two consumer warpgroups
constexpr int kProducers = 128;
constexpr int kPageTokens = 64;
// register split of the 64 K-register file: 128 x 56 + 256 x 224 = 64512
constexpr int kProducerRegs = 56, kConsumerRegs = 224;

template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

struct PrefixAttnParams {
  const int* cu_seqlens;          // [B + 1] chunk token offsets
  const int* prefix_lens;         // [B] tokens already in the cache
  const long long* kv_pointers;   // [B, 2, max_blocks] absolute page addresses
  __half* out;                    // [T, Hq * 128] rows of out_stride halfs
  long long out_stride;
  int num_heads, num_kv_heads, max_blocks;
  int num_tokens;                 // T: rows cu_seqlens[B] .. T - 1 are padding (zero output)
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
  if (b == static_cast<int>(gridDim.z) - 1 && seq_start + seq_len < p.num_tokens) {
    // rows cu_seqlens[B] .. num_tokens - 1 belong to no sequence (an in-flight step's chunk-segment padding): the CTAs (x, h) of the last
    // sequence write head h of those rows as zeros, so no NaN comes out of rows nobody reads.  Every existing call has cu_seqlens[B] = T.
    pdl_wait();  // the output buffer may still be read by the kernel before
    for (long long i = seq_start + seq_len + static_cast<long long>(blockIdx.x) * kBQ; i < p.num_tokens; i += static_cast<long long>(gridDim.x) * kBQ)
      for (int c = threadIdx.x; c < kBQ * kD / 8; c += kThreads) {
        const long long row = i + c / (kD / 8);
        if (row < p.num_tokens) reinterpret_cast<uint4*>(p.out + row * p.out_stride + static_cast<size_t>(h) * kD)[c % (kD / 8)] = make_uint4(0u, 0u, 0u, 0u);
      }
  }
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
  const RingBarriers bar = ring_barriers(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) init_ring(bar, kProducers, &tmap_q, &tmap_k, &tmap_v);  // K / V block ready: 128 arrivals (+ TMA bytes for a chunk block)
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
      mbar_expect_tx(bar.q, kTileBytes);
      tma_load_2d(s_q, &tmap_q, h * kD, q_row, bar.q);
      tma_load_2d(s_q + kSubBytes, &tmap_q, h * kD + 64, q_row, bar.q);
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
        if (j >= kStages) mbar_wait(&bar.kfree[st], ph ^ 1u);
        dequant_row<BITS>(sk, r, live ? reinterpret_cast<const uint8_t*>(kpg) : nullptr, slot, hkv, p);
        fence_proxy_async();  // generic-proxy writes, read by wgmma through the async proxy
        mbar_arrive(&bar.kfull[st]);
        if (j >= kStages) mbar_wait(&bar.vfree[st], ph ^ 1u);
        dequant_row<BITS>(sv, r, live ? reinterpret_cast<const uint8_t*>(vpg) : nullptr, slot, hkv, p);
        fence_proxy_async();
        mbar_arrive(&bar.vfull[st]);
        const int tn = t + kBKV;
        if (tn < P) {
          kpg = kptrs[tn / kPageTokens];
          vpg = vptrs[tn / kPageTokens];
        }
      } else {
        const int k_row = seq_start + (j - n_pb) * kBKV;
        if (j >= kStages) mbar_wait(&bar.kfree[st], ph ^ 1u);
        if (r == 0) {
          mbar_expect_tx(&bar.kfull[st], kTileBytes);
          tma_load_2d(sk, &tmap_k, hkv * kD, k_row, &bar.kfull[st]);
          tma_load_2d(sk + kSubBytes, &tmap_k, hkv * kD + 64, k_row, &bar.kfull[st]);
        } else {
          mbar_arrive(&bar.kfull[st]);
        }
        if (j >= kStages) mbar_wait(&bar.vfree[st], ph ^ 1u);
        if (r == 0) {
          mbar_expect_tx(&bar.vfull[st], kTileBytes);
          tma_load_2d(sv, &tmap_v, hkv * kD, k_row, &bar.vfull[st]);
          tma_load_2d(sv + kSubBytes, &tmap_v, hkv * kD + 64, k_row, &bar.vfull[st]);
        } else {
          mbar_arrive(&bar.vfull[st]);
        }
      }
    }
    return;
  }

  // ---- consumers.  Masks: keys >= P of the last prefix block; the causal diagonal of the chunk ----
  setmaxnreg_inc<kConsumerRegs>();
  consume(smem, warp - 4, lane, qb, n_kb, p.scale_log2, p.out, p.out_stride, seq_start, seq_len, h, [&](int j, int q_pos_a, int q_pos_b) {
    const bool pre = j < n_pb;
    const int kbase = (pre ? j : j - n_pb) * kBKV;
    return BlockMask{pre ? (kbase + kBKV > P) : (j - n_pb == qb), kbase, pre ? P - 1 : q_pos_a, pre ? P - 1 : q_pos_b};
  });
}

}  // namespace

int prefix_attention(const PrefixAttnArgs& a) {
  QS_REQUIRE(a.max_prefix_len >= 0, "prefix_prefill_attention: negative size");
  QS_REQUIRE(a.tokens_per_block == kPageTokens, "prefix_prefill_attention: tokens_per_block=%d, only 64 is supported", a.tokens_per_block);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * kD * bits / 8, "prefix_prefill_attention: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
  QS_REQUIRE(static_cast<long long>(a.max_prefix_len) + a.max_seqlen <= static_cast<long long>(a.max_blocks) * kPageTokens,
             "prefix_prefill_attention: max_prefix_len %d + max_seqlen %d exceed the page table (%d blocks of %d tokens)", a.max_prefix_len, a.max_seqlen,
             a.max_blocks, kPageTokens);
  bool empty = false;
  CUtensorMap tq, tk, tv;
  int rc = prompt_attention_prepare(a, "prefix_prefill_attention", &empty, &tq, &tk, &tv);
  if (rc || empty) return rc;
  QS_REQUIRE(a.prefix_lens && a.kv_pointers, "prefix_prefill_attention: null pointer");
  PrefixAttnParams p{};
  p.cu_seqlens = a.cu_seqlens;
  p.prefix_lens = a.prefix_lens;
  p.kv_pointers = a.kv_pointers;
  p.out = static_cast<__half*>(a.out);
  p.out_stride = a.out_stride;
  p.num_heads = a.num_heads;
  p.num_kv_heads = a.num_kv_heads;
  p.max_blocks = a.max_blocks;
  p.num_tokens = a.num_tokens;
  p.code_bytes = kPageTokens * a.size_per_token;
  p.scale_log2 = a.softmax_scale * 1.4426950408889634f;
  auto kern = a.int4_kv ? prefix_attention_kernel<4> : prefix_attention_kernel<8>;
  rc = raise_smem_limit(kern, kSmemBytes, "cudaFuncSetAttribute(prefix attention)");
  if (rc) return rc;
  return launch(kern, dim3((a.max_seqlen + kBQ - 1) / kBQ, a.num_heads, a.batch), dim3(kThreads), kSmemBytes, 0, a.stream,
                "prefix prefill attention launch", tq, tk, tv, p);
}

}  // namespace qs
