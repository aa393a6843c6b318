// qserve_b200 -- causal variable-length prefill attention on the sm_90a tensor cores (wgmma, fp32 accumulators in registers).
//
// Replaces the third-party call on the reference's prompt path: flash_attn_varlen_func(q, k, v, cu_seqlens, cu_seqlens, max_seqlen, max_seqlen,
// dropout_p=0, causal=True) in qserve/modeling/models/llama_w4a8_unpad.py:232-242, where q / k / v are strided views of the post-RoPE fp16 qkv
// buffer that fused_attention.apply_bias_rope_update_kv_cache has just rotated in place (SURVEY.md section 8 row f-3).
//
// One CTA = one (sequence, query head, block of 128 query rows); two consumer warpgroups own 64 query rows each.  Per block of 128 keys:
//     S = Q K^T      8 x wgmma m64n128k16, both operands K-major in shared memory (TMA, 128-byte swizzle), fp32 accumulators in registers
//     softmax        online, in the accumulator fragment (a row lives in the four threads of a quad): running max / sum in the log2 domain,
//                    P = exp2(..) rounded to fp16 and re-packed in registers as the A operand of the next MMA
//     O += P V       8 x wgmma m64n128k16, A = P from registers, B = the V tile exactly as TMA delivers it ([key][dim] rows: an MN-major
//                    operand, transposed B)
// K and V blocks travel in a two-deep ring filled by a producer warp (TMA), each slot refilled once both warpgroups' MMAs that read it retired.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include <mutex>

#include "common.cuh"
#include "launch.h"

namespace qs {
namespace {

constexpr int kD = 128;         // head dim
constexpr int kBQ = 128;        // query rows per CTA (two warpgroups x m64)
constexpr int kBKV = 128;       // keys per block (N of S, K extent of PV)
constexpr int kStages = 2;      // K / V ring depth
constexpr int kThreads = 288;   // warps 0..7: two consumer warpgroups, warp 8: TMA producer
constexpr int kTileBytes = kBQ * kD * 2;      // 32 KB: two swizzled [128 rows x 64 halfs] sub-tiles
constexpr int kSubBytes = kTileBytes / 2;     // 16 KB
constexpr int kOffQ = 0, kOffK = kTileBytes, kOffV = kOffK + kStages * kTileBytes, kOffBar = kOffV + kStages * kTileBytes;
constexpr int kSmemBytes = kOffBar + 128;

// 2^x on the SFU (MUFU.EX2), flush-to-zero: -inf must give 0
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b, float& sum) {
  const __half2 h2 = __floats2half2_rn(a, b);
  // the row sum is taken over the ROUNDED probabilities: numerator (the MMA sees fp16 P) and denominator then agree
  const float2 f = __half22float2(h2);
  sum += f.x + f.y;
  return *reinterpret_cast<const uint32_t*>(&h2);
}

struct PrefillAttnParams {
  const int* cu_seqlens;  // [B + 1]
  __half* out;            // [T, Hq * 128] rows of out_stride halfs
  long long out_stride;
  int num_heads, num_kv_heads;
  float scale_log2;       // softmax scale * log2(e)
};

__global__ void __launch_bounds__(kThreads, 1)
prefill_attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                         const __grid_constant__ CUtensorMap tmap_v, const PrefillAttnParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int b = blockIdx.z, h = blockIdx.y;
  const int seq_start = __ldg(p.cu_seqlens + b);
  const int seq_len = __ldg(p.cu_seqlens + b + 1) - seq_start;
  const int n_qb = (seq_len + kBQ - 1) / kBQ;
  const int qb = n_qb - 1 - static_cast<int>(blockIdx.x);  // the longest (last) query blocks of a sequence are scheduled first
  if (qb < 0) return;                                      // uniform per CTA
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
  const int hkv = h / (p.num_heads / p.num_kv_heads);
  const int n_kb = qb + 1;  // causal, q and k positions coincide: key blocks 0 .. qb

  uint8_t* s_q = smem + kOffQ;
  uint8_t* s_k = smem + kOffK;
  uint8_t* s_v = smem + kOffV;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* bar_q = bar;                      // Q tile landed
  uint64_t* bar_kfull = bar + 1;              // [kStages] K block landed
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
      mbar_init(&bar_kfull[i], 1);
      mbar_init(&bar_kfree[i], 8);
      mbar_init(&bar_vfull[i], 1);
      mbar_init(&bar_vfree[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == 8) {
    // ===================================== TMA producer =====================================
    if (lane == 0) {
      pdl_wait();  // q / k / v are written by the preceding kernel (RoPE + KV append)
      const int q_row = seq_start + qb * kBQ;
      mbar_expect_tx(bar_q, kTileBytes);
      tma_load_2d(s_q, &tmap_q, h * kD, q_row, bar_q);
      tma_load_2d(s_q + kSubBytes, &tmap_q, h * kD + 64, q_row, bar_q);
      for (int j = 0; j < n_kb; ++j) {
        const int k_row = seq_start + j * kBKV;
        const int st = j % kStages;
        const uint32_t ph = static_cast<uint32_t>(j / kStages) & 1u;
        uint8_t* sk = s_k + st * kTileBytes;
        uint8_t* sv = s_v + st * kTileBytes;
        if (j >= kStages) mbar_wait(&bar_kfree[st], ph ^ 1u);
        mbar_expect_tx(&bar_kfull[st], kTileBytes);
        tma_load_2d(sk, &tmap_k, hkv * kD, k_row, &bar_kfull[st]);
        tma_load_2d(sk + kSubBytes, &tmap_k, hkv * kD + 64, k_row, &bar_kfull[st]);
        if (j >= kStages) mbar_wait(&bar_vfree[st], ph ^ 1u);
        mbar_expect_tx(&bar_vfull[st], kTileBytes);
        tma_load_2d(sv, &tmap_v, hkv * kD, k_row, &bar_vfull[st]);
        tma_load_2d(sv + kSubBytes, &tmap_v, hkv * kD + 64, k_row, &bar_vfull[st]);
      }
    }
    return;
  }

  // ===================================== consumers: warpgroup g owns query rows [64 g, 64 g + 64) of the block =====================================
  const int g = warp >> 2;
  const int row_a = g * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's two rows: row_a and row_a + 8
  const int q_pos_a = qb * kBQ + row_a, q_pos_b = q_pos_a + 8;
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

    // ---- causal mask (diagonal block only) and row maxima ----
    float mx_a = -CUDART_INF_F, mx_b = -CUDART_INF_F;
    const bool diag = (j == qb);
#pragma unroll
    for (int c = 0; c < kBKV / 8; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = j * kBKV + c * 8 + col0 + (e & 1);
        float& v = s[c * 4 + e];
        if (e < 2) {
          if (diag && key > q_pos_a) v = -CUDART_INF_F;  // -inf: exp2 turns it into an exact 0
          mx_a = fmaxf(mx_a, v);
        } else {
          if (diag && key > q_pos_b) v = -CUDART_INF_F;
          mx_b = fmaxf(mx_b, v);
        }
      }
#pragma unroll
    for (int sh = 1; sh <= 2; sh <<= 1) {
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, sh));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, sh));
    }
    // key 0 is visible to every row, so the maxima are finite from the first block on
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
    // ---- P = exp2(s * scale - m), fp16, as wgmma A fragments: 16 keys (two accumulator column groups) per fragment ----
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
    // O += P V: B = V rows [key][dim] = MN-major, 16 keys (2 KB of each 64-dim sub-tile) per instruction, the second sub-tile 16 KB on
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

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
namespace {
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p) fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}
}  // namespace

// fp16 [rows, cols] with a row pitch of `stride` elements; box = 64 columns (128 B, swizzled) x 128 rows
int make_tmap_f16(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t stride) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {stride * 2};
  cuuint32_t box[2] = {64, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled(f16) failed (%d): ptr=%p rows=%llu cols=%llu stride=%llu", (int)r, ptr, (unsigned long long)rows,
                     (unsigned long long)cols, (unsigned long long)stride);
  return QS_OK;
}

int prefill_attention(const PrefillAttnArgs& a) {
  QS_REQUIRE(a.head_dim == kD, "prefill_attention: head_dim=%d (only 128 is built, as in the reference)", a.head_dim);
  QS_REQUIRE(a.num_heads > 0 && a.num_kv_heads > 0 && a.num_heads % a.num_kv_heads == 0, "prefill_attention: heads=%d kv_heads=%d", a.num_heads, a.num_kv_heads);
  QS_REQUIRE(a.batch >= 0 && a.num_tokens >= 0 && a.max_seqlen >= 0, "prefill_attention: negative size");
  if (a.batch == 0 || a.num_tokens == 0 || a.max_seqlen == 0) return QS_OK;
  QS_REQUIRE(a.batch <= 65535 && a.num_heads <= 65535, "prefill_attention: batch=%d / heads=%d exceed the grid limits", a.batch, a.num_heads);
  QS_REQUIRE(a.q && a.k && a.v && a.out && a.cu_seqlens, "prefill_attention: null pointer");
  QS_REQUIRE(a.q_stride % 8 == 0 && a.k_stride % 8 == 0 && a.v_stride % 8 == 0 && a.out_stride % 8 == 0, "prefill_attention: row strides must be multiples of 8 halfs");
  QS_REQUIRE(((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v) | reinterpret_cast<uintptr_t>(a.out)) & 15) == 0,
             "prefill_attention: q, k, v, out must be 16-byte aligned");
  QS_REQUIRE(a.q_stride >= a.num_heads * kD && a.k_stride >= a.num_kv_heads * kD && a.v_stride >= a.num_kv_heads * kD && a.out_stride >= a.num_heads * kD,
             "prefill_attention: row stride smaller than the row");
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_f16(&tq, a.q, a.num_tokens, static_cast<uint64_t>(a.num_heads) * kD, a.q_stride);
  if (rc) return rc;
  rc = make_tmap_f16(&tk, a.k, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.k_stride);
  if (rc) return rc;
  rc = make_tmap_f16(&tv, a.v, a.num_tokens, static_cast<uint64_t>(a.num_kv_heads) * kD, a.v_stride);
  if (rc) return rc;
  static bool attr_set[kMaxDevices] = {};
  bool& done = attr_set[device_ordinal()];
  if (!done) {
    rc = check_cuda(cudaFuncSetAttribute(prefill_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes), "cudaFuncSetAttribute(prefill attention)");
    if (rc) return rc;
    done = true;
  }
  PrefillAttnParams p{};
  p.cu_seqlens = a.cu_seqlens;
  p.out = static_cast<__half*>(a.out);
  p.out_stride = a.out_stride;
  p.num_heads = a.num_heads;
  p.num_kv_heads = a.num_kv_heads;
  p.scale_log2 = a.softmax_scale * 1.4426950408889634f;
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
  return check_cuda(cudaLaunchKernelEx(&cfg, prefill_attention_kernel, tq, tk, tv, p), "prefill attention launch");
}

}  // namespace qs
