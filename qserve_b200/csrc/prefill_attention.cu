// qserve_b200 -- causal variable-length prefill attention on the sm_90a tensor cores (wgmma, fp32 accumulators in registers).
//
// Replaces the third-party call on the reference's prompt path: flash_attn_varlen_func(q, k, v, cu_seqlens, cu_seqlens, max_seqlen, max_seqlen,
// dropout_p=0, causal=True) in qserve/modeling/models/llama_w4a8_unpad.py:232-242, where q / k / v are strided views of the post-RoPE fp16 qkv
// buffer that fused_attention.apply_bias_rope_update_kv_cache has just rotated in place (SURVEY.md section 8 row f-3).
//
// One CTA = one (sequence, query head, block of 128 query rows); the two consumer warpgroups of prompt_attention.cuh own 64 query rows each
// (S = Q K^T, online softmax in registers, O += P V) and mask only the diagonal key block.  K and V blocks travel in a two-deep ring filled
// by a producer warp (TMA), each slot refilled once both warpgroups' MMAs that read it retired.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <mutex>

#include "common.cuh"
#include "launch.cuh"
#include "prompt_attention.cuh"

namespace qs {
namespace {

constexpr int kThreads = 288;   // warps 0..7: two consumer warpgroups, warp 8: TMA producer

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
  const RingBarriers bar = ring_barriers(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) init_ring(bar, 1, &tmap_q, &tmap_k, &tmap_v);
  __syncthreads();
  if (threadIdx.x == 0) pdl_launch_dependents();

  if (warp == 8) {
    // ===================================== TMA producer =====================================
    if (lane == 0) {
      pdl_wait();  // q / k / v are written by the preceding kernel (RoPE + KV append)
      const int q_row = seq_start + qb * kBQ;
      mbar_expect_tx(bar.q, kTileBytes);
      tma_load_2d(s_q, &tmap_q, h * kD, q_row, bar.q);
      tma_load_2d(s_q + kSubBytes, &tmap_q, h * kD + 64, q_row, bar.q);
      for (int j = 0; j < n_kb; ++j) {
        const int k_row = seq_start + j * kBKV;
        const int st = j % kStages;
        const uint32_t ph = static_cast<uint32_t>(j / kStages) & 1u;
        uint8_t* sk = s_k + st * kTileBytes;
        uint8_t* sv = s_v + st * kTileBytes;
        if (j >= kStages) mbar_wait(&bar.kfree[st], ph ^ 1u);
        mbar_expect_tx(&bar.kfull[st], kTileBytes);
        tma_load_2d(sk, &tmap_k, hkv * kD, k_row, &bar.kfull[st]);
        tma_load_2d(sk + kSubBytes, &tmap_k, hkv * kD + 64, k_row, &bar.kfull[st]);
        if (j >= kStages) mbar_wait(&bar.vfree[st], ph ^ 1u);
        mbar_expect_tx(&bar.vfull[st], kTileBytes);
        tma_load_2d(sv, &tmap_v, hkv * kD, k_row, &bar.vfull[st]);
        tma_load_2d(sv + kSubBytes, &tmap_v, hkv * kD + 64, k_row, &bar.vfull[st]);
      }
    }
    return;
  }

  // causal, q and k positions coincide: only the diagonal block qb is masked
  consume(smem, warp, lane, qb, n_kb, p.scale_log2, p.out, p.out_stride, seq_start, seq_len, h, [&](int j, int q_pos_a, int q_pos_b) {
    return BlockMask{j == qb, j * kBKV, q_pos_a, q_pos_b};
  });
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
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
  bool empty = false;
  CUtensorMap tq, tk, tv;
  int rc = prompt_attention_prepare(a, "prefill_attention", &empty, &tq, &tk, &tv);
  if (rc || empty) return rc;
  rc = raise_smem_limit(prefill_attention_kernel, kSmemBytes, "cudaFuncSetAttribute(prefill attention)");
  if (rc) return rc;
  PrefillAttnParams p{};
  p.cu_seqlens = a.cu_seqlens;
  p.out = static_cast<__half*>(a.out);
  p.out_stride = a.out_stride;
  p.num_heads = a.num_heads;
  p.num_kv_heads = a.num_kv_heads;
  p.scale_log2 = a.softmax_scale * 1.4426950408889634f;
  return launch(prefill_attention_kernel, dim3((a.max_seqlen + kBQ - 1) / kBQ, a.num_heads, a.batch), dim3(kThreads), kSmemBytes, 0, a.stream,
                "prefill attention launch", tq, tk, tv, p);
}

}  // namespace qs
