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
#include "launch.cuh"
#include "paged_attention.cuh"

namespace qs {
namespace {

__device__ __forceinline__ unsigned long long attn_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
  return t;
}

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
// This kernel, multi_token_attention_kernel and shared_prefix_attention_kernel are built on paged_attention.cuh (one n8 tile here: the <= 8
// heads of the group); the output bits of this kernel are pinned by tests/test_gpu_attention.py::test_decode_attention_output_bits_are_pinned.
constexpr int kAttnThreadsV2 = kAttnConsumers;  // no dedicated producer warp: every warp streams its own half pages

// SHARED (the row pass of qs_shared_prefix_decode_attention, DESIGN.md 3.10): the row's pages start at row_pages[b]; a row with
// row_pages[b] > 0 has part_stride - nsplit more partials per head, written by shared_prefix_attention_kernel at slots nsplit .., and its final
// merge takes them after its own splits.  Without SHARED the two trailing arguments are not read.
template <int BITS, bool SHARED = false>
__global__ void __launch_bounds__(kAttnThreadsV2, 4)
decode_attention_kernel(const __half* __restrict__ q_in, const __half* __restrict__ k_in, const __half* __restrict__ v_in, long long q_stride,
                        long long k_stride, long long v_stride, const long long* __restrict__ kv_pointers, const int* __restrict__ lengths,
                        __half* __restrict__ out, int num_heads, int num_kv_heads, int max_blocks, PageGeom pg, float rotary_base, int rotary_dim,
                        int timestep, int nsplit, float* __restrict__ ws_part, uint32_t* __restrict__ ws_cnt, uint32_t* __restrict__ tok_cnt, int8_t* __restrict__ q_out,
                        __half* __restrict__ q_scale, __half* __restrict__ q_sum, unsigned long long* __restrict__ prof, const int* __restrict__ row_pages,
                        int part_stride) {
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
  if (tlen < 0) {
    // idle row (length 0, an in-flight step's free or prefilling row): no page byte, a zero output row (with the fused quantisation: the zero
    // int8 row, scale and sum that invoke_quant gives a zero row), and no split or per-token counter is touched.  Uniform per CTA.
    pdl_wait();  // the outputs may still be read by the kernel before (q_out aliases the qkv GEMM's input)
    if (split != 0) return;
    if (q_out == nullptr) {
      for (int i = threadIdx.x; i < Gc * kD; i += kAttnThreadsV2) out[(static_cast<size_t>(b) * num_heads + h0) * kD + i] = __float2half_rn(0.f);
    } else if (blockIdx.x == 0) {
      int8_t* qrow = q_out + static_cast<size_t>(b) * num_heads * kD;
      for (int i = threadIdx.x; i < num_heads * kD; i += kAttnThreadsV2) qrow[i] = 0;
      if (threadIdx.x == 0) {
        q_scale[b] = __float2half_rn(0.f);
        if (q_sum) q_sum[b] = __float2half_rn(0.f);
      }
    }
    return;
  }
  const long long* kptrs = kv_pointers + (static_cast<size_t>(b) * 2 + 0) * max_blocks;
  const long long* vptrs = kv_pointers + (static_cast<size_t>(b) * 2 + 1) * max_blocks;
  const int n_pages = (tlen + kPageTokens - 1) / kPageTokens;
  const int p_first = SHARED ? row_pages[b] : 0;  // pages below p_first are the group's: the shared pass reads them
  const int pps = (n_pages - p_first + nsplit - 1) / nsplit;
  const int p_begin = p_first + split * pps, p_end = min(n_pages, p_begin + pps);
  const int last_blk = tlen / pg.tokens_per_block;  // page receiving the new token
  // partials of the final merge per (row, head): this launch's splits, then (SHARED, rows in a group) the shared pass's
  const int ptot = (SHARED && p_first > 0) ? part_stride : nsplit;
  const int pstride = SHARED ? part_stride : nsplit;

  // ---- this warp's stream: token slice [32 (warp & 1), +32) of the pages p_begin + (warp >> 1), +2, ...  ----
  const int hslice = warp & 1;
  const int my_first = p_begin + (warp >> 1);
  const int n_my = (p_end > my_first) ? (p_end - my_first + 1) / 2 : 0;
  uint8_t* my_ring = s_ring + warp * SL::kWarpBytes;
  uint64_t* my_full = &s_full[warp][0];
  const int zoff = pg.num_kv_heads * pg.tokens_per_block * 2;  // bytes from a scale row to the zero row
  long long kp_l = 0, vp_l = 0;  // lane l: page pointers of this warp's slice (batch * 32 + l)
  auto load_ptr_batch = [&](int j0) { slice_ptrs(kptrs, vptrs, my_first + 2 * (j0 + lane), p_end, kp_l, vp_l); };
  auto issue = [&](int j, int slot) {
    issue_slice<BITS>(lane, kp_l, vp_l, j, my_ring + slot * SL::kBytes, &my_full[slot], hk, hslice, pg.code_bytes, zoff);
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
    rope_sincos(tlen, ri, rotary_base, rotary_dim, sn, cs);
#pragma unroll
    for (int e = 0; e < kRowsPerThread; ++e) {
      const int r = r0 + 2 * e;
      if (r <= Gc) rope_store((r < Gc) ? (s_q + r * kD) : s_k, ri, half_rot, x0[e], x1[e], sn, cs);
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
    float sumq[1][2], biasq[1][2];  // heads 2*q4 and 2*q4+1 (this thread's S^T columns)
    q_operand<BITS>(s_q + g * kD + 32 * q4, q4, qb0, qb1, sumq[0], biasq[0]);
    auto qb = [&](int, int ks, uint32_t& b0, uint32_t& b1) {  // the Q fragments stay in registers
      b0 = qb0[ks];
      b1 = qb1[ks];
    };

    const float sm_scale = rsqrtf(static_cast<float>(kD)) * 1.4426950408889634f;  // 1/sqrt(D) * log2(e)
    // O^T accumulators: m-tile i (dims 16g + 2i, 16g + 2i + 1) x heads (2q4, 2q4+1)
    float o[1][8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[0][i][0] = o[0][i][1] = o[0][i][2] = o[0][i][3] = 0.f;
    // running max, sum p, sum p*c (zero-point correction), sum p' (bias correction of the V operand) per head
    float m[2] = {-CUDART_INF_F, -CUDART_INF_F}, l[2] = {0.f, 0.f}, cr[2] = {0.f, 0.f};
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
      if (t0 < tlen) {  // every processed slice holds at least one valid token, so no column's running max stays -inf
        slice_meta<BITS>(st, lane, t0 + lane >= tlen, sm_scale, s_meta[warp][0], s_meta[warp][1]);
        __syncwarp();
        // ---- S^T (2 x 16 tokens x 8 heads) on biased codes: 16 MMAs ----
        float sc[2][1][4];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          sc[c][0][0] = sc[c][0][1] = sc[c][0][2] = sc[c][0][3] = 0.f;
          qk_chunk<BITS, 1>(st + SL::kOffK + (c * kChunk + tokA) * kRow, q4, sc[c], qb);
        }
        // ---- logits (log2 units) of tokens A = tokA, B = 8 + tokA of both chunks for heads 2q4, 2q4+1 ----
        float tl[2][1][4], vs[2][2], vc[2][2];
#pragma unroll
        for (int c = 0; c < 2; ++c) chunk_logits<1>(s_meta[warp][0], s_meta[warp][1], c, tokA, sc[c], biasq, sumq, tl[c], vs[c], vc[c]);
        if (t0 + 2 * kChunk > tlen) {  // only the last page of a sequence
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (t0 + c * kChunk + tokA >= tlen) tl[c][0][0] = tl[c][0][1] = -CUDART_INF_F;
            if (t0 + c * kChunk + 8 + tokA >= tlen) tl[c][0][2] = tl[c][0][3] = -CUDART_INF_F;
          }
        }
        uint32_t bp[2][1][2];
        softmax_tile<1, false>(0, tl, vs, vc, m, l, cr, spa, o[0], bp);
        // ---- O^T += V^T P'^T on biased codes: 2 x 8 MMAs (m-tile = 16 dims) ----
#pragma unroll
        for (int c = 0; c < 2; ++c) pv_chunk<BITS, 1>(st + SL::kOffV + (c * kChunk + q4) * kRow, g, o, bp[c]);
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
    reduce_tile_sums(l, cr);
    if (g == 0) {
      s_m[warp][2 * q4] = m[0]; s_m[warp][2 * q4 + 1] = m[1];
      s_l[warp][2 * q4] = l[0]; s_l[warp][2 * q4 + 1] = l[1];
    }
    __syncwarp();  // every lane is done with the ring slots this overwrites
    store_partial<BITS>(reinterpret_cast<float*>(my_ring) + (2 * q4) * kOStride + g, o[0], spa, cr);
    // new token logit: fp32 dot of the rotated, un-quantised q and k
    if (split == 0) {
      for (int r = warp; r < Gc; r += kWarps) {
        const float acc = own_logit(s_q + r * kD, s_k, lane);
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
  const int nparts = kWarps + (split == 0 ? 1 : 0);
  if (threadIdx.x < kMaxG) merge_weights<kMaxG>(threadIdx.x, nparts, ptot, s_m, s_l, s_f);
  __syncthreads();
  if (threadIdx.x < kD) {
    const int d = 16 * (threadIdx.x & 7) + (threadIdx.x >> 3);  // the dim whose partials sit at offset threadIdx.x
    float* part = nullptr;
    if (ptot > 1) part = ws_part + ((static_cast<size_t>(b) * num_heads + h0) * pstride + split) * (kD + 2);
    const float vd = __half2float(s_v[d]);
#pragma unroll
    for (int r = 0; r < kMaxG; ++r) {
      if (r < Gc) {
        const float acc = merge_warps<BITS, kMaxG>(s_ring, r, vd, s_f);
        if (ptot == 1) {
          out[(static_cast<size_t>(b) * num_heads + h0 + r) * kD + d] = __float2half_rn(acc);
        } else {
          float* pr = part + static_cast<size_t>(r) * pstride * (kD + 2);
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
  bool final_written = (ptot == 1);  // this CTA produced the final fp16 outputs of its head group
  if (ptot > 1) {
    // SHARED: the shared pass finished before this grid passed its dependency wait, so its partials are complete
    final_written = arrive_last(ws_cnt + static_cast<size_t>(b) * gridDim.x + blockIdx.x, nsplit, s_last);
    if (final_written && threadIdx.x < kD) {
      const int d = threadIdx.x;
      __threadfence();
      for (int r = 0; r < Gc; ++r) {
        const float* pr = ws_part + (static_cast<size_t>(b) * num_heads + h0 + r) * pstride * (kD + 2);
        out[(static_cast<size_t>(b) * num_heads + h0 + r) * kD + d] = __float2half_rn(merge_splits(pr, ptot, d));
      }
    }
  }
  if (q_out != nullptr && final_written) {
    // ---- fused per-token INT8 quantisation of the attention output (invoke_quant[_fuse_sum], fused_kernels.cu:92-137).
    //      `out` is an fp16 scratch row in the workspace (L2 resident); the last head-group CTA of a token to finish
    //      re-reads the row and quantises it: same arithmetic as quant_per_token_kernel ----
    __shared__ uint32_t s_last_tok;
    __shared__ float s_red_f[8], s_red_nf[8];
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
      float amax = 0.f, nf = 0.f;
      long long sum = 0;
      auto stats = [&](const uint4& v) {
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          if (q_sum) {
            sum += fx_of_finite(f.x) + fx_of_finite(f.y);
            nf += f.x + f.y;  // a thread's fp32 sum of fp16 values cannot overflow: it is non-finite only where the side sum is, and then equals it
          }
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
      nf = nonfinite_part(nf);
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, m));
        sum += __shfl_xor_sync(0xffffffffu, sum, m);
        nf += __shfl_xor_sync(0xffffffffu, nf, m);
      }
      if (lane == 0) { s_red_f[warp] = amax; s_red_l[warp] = sum; s_red_nf[warp] = nf; }
      __syncthreads();
      amax = 0.f;
      sum = 0;
      nf = 0.f;
      for (int w = 0; w < kAttnThreadsV2 / 32; ++w) { amax = fmaxf(amax, s_red_f[w]); sum += s_red_l[w]; nf += s_red_nf[w]; }
      if (threadIdx.x == 0) {
        q_scale[b] = __float2half_rn(__fdiv_rn(amax, 127.f));
        if (q_sum) q_sum[b] = __float2half_rn(row_sum(sum, nf));
      }
      const float qs_ = __fdiv_rn(127.f, amax);
      int8_t* qrow = q_out + static_cast<size_t>(b) * num_heads * kD;
      auto quantise = [&](int i, const uint4& v) {
        const __half* h = reinterpret_cast<const __half*>(&v);
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = __half2float(h[j]);
        store_q8(qrow, i, x, qs_);
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
// K1s: shared pass of qs_shared_prefix_decode_attention (DESIGN.md 3.10).  Rows forked from one prompt share the pages 0 .. S_g - 1 of their
//   group g.  One CTA owns (KV head, column part, group, context split); column c of part cp is (member j, query head h) with C cp + c = j G + h,
//   so every code a warp unpacks feeds C = 8 NT columns: the page stream is column_tile_stream, shared with multi_token_attention_kernel
//   (DESIGN.md 3.6).  Member j's q is rotated at its own position lengths[row_j] - 1 (members diverge once a finished row stops advancing)
//   through the decode kernel's RoPE functions.  Every shared token is valid for every member (the caller guarantees 64 S_g cached tokens),
//   so there is no causal tail, no own token and no append.  The CTA writes one unnormalised partial (O, max, sum) per (member row, head) at split slot part_off + split of the row's
//   partials; the row pass (decode_attention_kernel<BITS, true>) merges them after its own splits.
// ------------------------------------------------------------------------------------------------
struct SharedPrefixParams {
  const __half* q;                // [B, Hq * 128] rows of q_stride halfs (un-rotated)
  long long q_stride;
  const int* lengths;             // [B] context length including the new token
  const long long* kv_pointers;   // [B, 2, max_blocks]
  const int* group_offsets;       // [num_groups + 1]
  const int* group_rows;          // rows of group g: group_rows[group_offsets[g] .. group_offsets[g + 1])
  const int* group_pages;         // [num_groups] shared pages S_g, read through the table of the group's first row
  int num_heads, num_kv_heads, max_blocks;
  int cparts, nsplit;             // column parts per KV head, context splits of the shared pages
  int part_off, part_stride;      // slot of split 0 among a row's partials, partials per (row, head)
  PageGeom pg;
  float rotary_base;
  int rotary_dim;
  float* ws_part;                 // [B, Hq, part_stride, 130]
};

template <int BITS, int NT>
__global__ void __launch_bounds__(kAttnConsumers, kColumnMinBlocks<NT>) shared_prefix_attention_kernel(const SharedPrefixParams p) {
  constexpr int C = 8 * NT;
  const int G = p.num_heads / p.num_kv_heads;
  const int hk = blockIdx.x / p.cparts;
  const int col0 = (blockIdx.x - hk * p.cparts) * C;
  const int grp = blockIdx.y;
  const int split = blockIdx.z;

  // the layout and the tables are prepared by the host before the step: read before the dependency wait; q and the pages after it
  const int mem0 = p.group_offsets[grp];
  const int nmem = p.group_offsets[grp + 1] - mem0;
  const int S = p.group_pages[grp];
  const int ncol = min(C, G * nmem - col0);
  if (ncol <= 0 || S <= 0) return;  // uniform over the CTA; a group without shared pages has no partials (its rows have row_pages 0)

  extern __shared__ __align__(128) uint8_t smem_attn[];
  uint8_t* s_ring = smem_attn;
  __shared__ ColumnShared<BITS, NT> sh;

  auto stage = [&] {
    // thread t rotates the pair (ri, ri + 64) of columns t / 64, t / 64 + 2, ...: the member rows and positions of those columns
    const int ri = threadIdx.x & 63, c0 = threadIdx.x >> 6;
    const int half_rot = p.rotary_dim / 2;
    int last_pos = -1;
    float sn = 0.f, cs = 1.f;
    for (int c = c0; c < C; c += 2) {
      __half* dst = sh.q + c * kD;
      if (c < ncol) {
        const int j = (col0 + c) / G, h = col0 + c - j * G;
        const int row = p.group_rows[mem0 + j];
        const int pos = p.lengths[row] - 1;
        const __half* src = p.q + static_cast<size_t>(row) * p.q_stride + static_cast<size_t>(hk * G + h) * kD;
        const __half x0 = src[ri], x1 = src[ri + half_rot];
        if (pos != last_pos) {
          rope_sincos(pos, ri, p.rotary_base, p.rotary_dim, sn, cs);
          last_pos = pos;
        }
        rope_store(dst, ri, half_rot, x0, x1, sn, cs);
      } else {
        dst[ri] = dst[ri + half_rot] = __float2half_rn(0.f);
      }
    }
  };
  auto none_unread = [](int) { return false; };
  auto no_tail = [](int, int, float (&)[2][NT][4]) {};
  // the shared pages through the table of the group's first row; the decode kernel's softmax scale
  column_tile_stream<BITS, NT, false>(sh, s_ring, p.kv_pointers, p.group_rows[mem0], p.max_blocks, p.pg, hk, S, p.nsplit,
                                      rsqrtf(static_cast<float>(kD)) * 1.4426950408889634f, stage, none_unread, no_tail);
  __syncthreads();

  // merge the warps; never normalised here (nsplit argument 0): the row pass normalises after its merge of every part
  if (threadIdx.x < C) merge_weights<C>(threadIdx.x, kWarps, 0, sh.m, sh.l, sh.f);
  __syncthreads();
  if (threadIdx.x < kD) {
    const int d = 16 * (threadIdx.x & 7) + (threadIdx.x >> 3);
#pragma unroll
    for (int r = 0; r < C; ++r) {
      if (r < ncol) {
        const float acc = merge_warps<BITS, C>(s_ring, r, 0.f, sh.f);
        const int j = (col0 + r) / G, h = col0 + r - j * G;
        const int row = p.group_rows[mem0 + j];
        float* pr = p.ws_part + ((static_cast<size_t>(row) * p.num_heads + hk * G + h) * p.part_stride + p.part_off + split) * (kD + 2);
        pr[d] = acc;
        if (threadIdx.x == 0) {
          pr[kD] = sh.m[0][r];
          pr[kD + 1] = sh.l[0][r];
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K2: prefill RoPE + KV quantise + page append: one warp per (token, KV head): it rotates the G query heads of the group and the key head with
//     ONE evaluation of the position's sines / cosines (the first version, one warp per query head, spent its time in 32 redundant
//     powf / sincosf per token: 365 us per layer for the 8 x 1024-token prompt batch), then quantises and appends K and V.
//     applyBiasRopeUpdateKVCache.h:94-455 (STORE_QKV = true, no bias, NeoX)
// ------------------------------------------------------------------------------------------------
// AT: start_pos is given (qs_apply_bias_rope_update_kv_cache_at); otherwise it is ignored.  TREE (with AT): the tokens are draft-tree nodes,
// node cpos is rotated at start + depth(cpos) (the popcount of its ancestor word tree_mask[token]) and stored in slot start + cpos.
template <int BITS, bool AT, bool TREE = false>
__global__ void __launch_bounds__(128) prefill_append_kernel(__half* __restrict__ qkv, const int* __restrict__ seq_lens,
                                                             const int* __restrict__ padding_offset, const long long* __restrict__ kv_pointers,
                                                             const int* __restrict__ start_pos, int num_tokens, int max_blocks, int num_heads, int num_kv_heads, int seq_len,
                                                             PageGeom pg, float rotary_base, int rotary_dim, int max_positions,
                                                             const int* __restrict__ tree_mask) {
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
    const int rpos = TREE ? start + __popc(static_cast<uint32_t>(tree_mask[token]) & ((1u << cpos) - 1u)) : pos;  // RoPE position
    __half* trow = qkv + static_cast<size_t>(token) * n;
    // lane handles rotary pairs i = 2*lane, 2*lane+1  (i in [0, 64)) -> dims i and i + half_rot: one half2 at each end
    float cs[2], sn[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int i = 2 * lane + e;
      const float inv_freq = __fdiv_rn(static_cast<float>(rpos), powf(rotary_base, __fdiv_rn(static_cast<float>(2 * i), static_cast<float>(rotary_dim))));
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

constexpr size_t kAttnCounterBytes = 256 * 1024;  // 49152 (sequence, head-group) split counters + 16384 per-token counters
constexpr size_t kAttnTokCounterOffset = 192 * 1024;

struct SharedPrefixPlan {
  int gx;          // row pass: KV heads x head groups of <= 8 query heads
  int nsplit;      // row pass context splits (decode_attention's)
  ColumnPlan sp;   // shared pass over (member, query head) columns; sp.nsplit = 0: no shared pass
  size_t part_bytes, row_bytes;
};

// shared_prefix_attention_kernel<bits, ntile>: the one place the plan's occupancy lookup and the launch pick it
ColumnKernel<void (*)(SharedPrefixParams)> shared_prefix_kernel(int bits, int ntile) {
  if (bits == 4) return ntile == 1 ? column_kernel<shared_prefix_attention_kernel<4, 1>>() : column_kernel<shared_prefix_attention_kernel<4, 2>>();
  return ntile == 1 ? column_kernel<shared_prefix_attention_kernel<8, 1>>() : column_kernel<shared_prefix_attention_kernel<8, 2>>();
}

// The launch plan of qs_shared_prefix_decode_attention: a function of host integers only, so the call can be captured in a graph
SharedPrefixPlan plan_shared_prefix(int bits, int batch, int num_heads, int num_kv_heads, int timestep, int num_groups, int max_group, int max_pages) {
  SharedPrefixPlan pl{};
  const int G = num_heads / num_kv_heads;
  pl.gx = num_kv_heads * ((G + kMaxG - 1) / kMaxG);
  pl.nsplit = context_splits(static_cast<long long>(pl.gx) * batch, num_sms() * 4, timestep);
  if (num_groups > 0 && max_group > 0 && max_pages > 0) {
    auto per_sm = [&](int ntile) { return shared_prefix_kernel(bits, ntile).resident(ring_bytes(bits), "shared_prefix_decode_attention smem attribute"); };
    pl.sp = plan_columns(G * max_group, static_cast<long long>(num_kv_heads) * num_groups, max_pages * kPageTokens, per_sm);
  }
  pl.part_bytes = static_cast<size_t>(batch) * num_heads * (pl.nsplit + pl.sp.nsplit) * (kD + 2) * sizeof(float);
  pl.row_bytes = static_cast<size_t>(batch) * num_heads * kD * sizeof(__half);
  return pl;
}

}  // namespace

size_t shared_prefix_attention_workspace_bytes(int batch, int num_heads, int num_kv_heads, int timestep, int num_groups, int max_group, int max_pages,
                                               int int4_kv) {
  if (batch <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0) return 0;
  const SharedPrefixPlan pl = plan_shared_prefix(int4_kv ? 4 : 8, batch, num_heads, num_kv_heads, timestep, num_groups, max_group, max_pages);
  return kAttnCounterBytes + pl.part_bytes + pl.row_bytes;
}

int shared_prefix_decode_attention(const SharedPrefixAttnArgs& s) {
  const DecodeAttnArgs& a = s.d;
  const int rc = check_page_geometry("shared_prefix_decode_attention", a.head_dim, a.num_heads, a.num_kv_heads, a.tokens_per_block, a.size_per_token,
                                     a.int4_kv);
  if (rc) return rc;
  QS_REQUIRE(a.kv_zeros, "shared_prefix_decode_attention: only kv_cache_with_zeros=True is supported");
  QS_REQUIRE(a.rotary_dim == kD, "shared_prefix_decode_attention: rotary_dim=%d must equal head_dim", a.rotary_dim);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.batch >= 0 && a.batch <= 16384, "shared_prefix_decode_attention: batch=%d, must be 0 .. 16384", a.batch);
  QS_REQUIRE(s.num_groups >= 0 && s.num_groups <= 65535 && s.max_group >= 0 && s.max_pages >= 0,
             "shared_prefix_decode_attention: num_groups=%d, max_group=%d, max_pages=%d", s.num_groups, s.max_group, s.max_pages);
  QS_REQUIRE(s.max_pages <= a.max_blocks, "shared_prefix_decode_attention: max_pages=%d exceeds the page table (%d blocks)", s.max_pages, a.max_blocks);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.q && a.k && a.v && a.kv_pointers && a.lengths && s.row_pages && (a.out != nullptr) != (a.q_out != nullptr),
             "shared_prefix_decode_attention: null tensor, or not exactly one of out / out_q");
  QS_REQUIRE(s.num_groups == 0 || (s.group_offsets && s.group_rows && s.group_pages), "shared_prefix_decode_attention: null group layout");
  QS_REQUIRE(a.q_out == nullptr || a.q_scale != nullptr, "shared_prefix_decode_attention: q_scale is null");
  QS_REQUIRE(a.q_stride % 8 == 0 && (reinterpret_cast<uintptr_t>(a.q) & 15) == 0, "shared_prefix_decode_attention: q rows must be 16-byte aligned");
  const SharedPrefixPlan pl = plan_shared_prefix(bits, a.batch, a.num_heads, a.num_kv_heads, a.timestep, s.num_groups, s.max_group, s.max_pages);
  QS_REQUIRE(static_cast<size_t>(a.batch) * pl.gx * 4 <= kAttnTokCounterOffset, "shared_prefix_decode_attention: batch %d x %d head groups too large",
             a.batch, pl.gx);
  const size_t need = kAttnCounterBytes + pl.part_bytes + pl.row_bytes;
  QS_REQUIRE(a.workspace != nullptr && a.workspace_bytes >= need,
             "shared_prefix_decode_attention: workspace of %zu bytes, need %zu (qs_shared_prefix_attention_workspace_bytes)", a.workspace_bytes, need);
  uint8_t* ws = static_cast<uint8_t*>(a.workspace);
  uint32_t* cnt = reinterpret_cast<uint32_t*>(ws);
  uint32_t* tok_cnt = reinterpret_cast<uint32_t*>(ws + kAttnTokCounterOffset);
  float* part = reinterpret_cast<float*>(ws + kAttnCounterBytes);
  void* out = a.q_out != nullptr ? ws + kAttnCounterBytes + pl.part_bytes : a.out;
  const int pstride = pl.nsplit + pl.sp.nsplit;
  PageGeom pg{kPageTokens, kPageTokens * a.size_per_token, a.num_kv_heads};
  const size_t smem = ring_bytes(bits);
  if (pl.sp.nsplit > 0) {
    SharedPrefixParams p{};
    p.q = static_cast<const __half*>(a.q);
    p.q_stride = a.q_stride;
    p.lengths = a.lengths;
    p.kv_pointers = a.kv_pointers;
    p.group_offsets = s.group_offsets;
    p.group_rows = s.group_rows;
    p.group_pages = s.group_pages;
    p.num_heads = a.num_heads; p.num_kv_heads = a.num_kv_heads; p.max_blocks = a.max_blocks;
    p.cparts = pl.sp.cparts; p.nsplit = pl.sp.nsplit;
    p.part_off = pl.nsplit; p.part_stride = pstride;
    p.pg = pg;
    p.rotary_base = a.rotary_base; p.rotary_dim = a.rotary_dim;
    p.ws_part = part;
    const dim3 grid(static_cast<unsigned>(a.num_kv_heads * pl.sp.cparts), s.num_groups, pl.sp.nsplit);
    const auto kern = shared_prefix_kernel(bits, pl.sp.ntile).fn;
    if (const int err = raise_smem_limit(kern, smem, "shared_prefix_decode_attention smem attribute")) return err;
    if (const int err = launch(kern, grid, dim3(kAttnConsumers), smem, 0, a.stream, "shared_prefix_decode_attention", p)) return err;
  }
  const dim3 grid(pl.gx, a.batch, pl.nsplit);
  auto run = [&](auto kern) {
    const int rc = raise_smem_limit(kern, smem, "attention smem attribute");
    if (rc) return rc;
    return launch(kern, grid, dim3(kAttnThreadsV2), smem, 1, a.stream, "shared_prefix_decode_attention rows", static_cast<const __half*>(a.q),
                  static_cast<const __half*>(a.k), static_cast<const __half*>(a.v), a.q_stride, a.k_stride, a.v_stride, a.kv_pointers, a.lengths,
                  static_cast<__half*>(out), a.num_heads, a.num_kv_heads, a.max_blocks, pg, a.rotary_base, a.rotary_dim, a.timestep, pl.nsplit, part, cnt,
                  a.q_out != nullptr ? tok_cnt : nullptr, static_cast<int8_t*>(a.q_out), static_cast<__half*>(a.q_scale), static_cast<__half*>(a.q_sum),
                  static_cast<unsigned long long*>(nullptr), s.row_pages, pstride);
  };
  return bits == 4 ? run(decode_attention_kernel<4, true>) : run(decode_attention_kernel<8, true>);
}

size_t attention_workspace_bytes(int batch, int num_heads, int head_dim, int max_splits) {
  return kAttnCounterBytes + static_cast<size_t>(batch) * num_heads * max_splits * (head_dim + 2) * sizeof(float) +
         static_cast<size_t>(batch) * num_heads * head_dim * sizeof(__half);  // + fp16 scratch rows of the fused-quant form
}

int attention_trace_install(void* buf, unsigned cap) { return qs_trace_install(buf, cap); }

int decode_attention(const DecodeAttnArgs& a) {
  if (a.batch == 0) return QS_OK;
  const int rc = check_page_geometry("single_query_attention", a.head_dim, a.num_heads, a.num_kv_heads, a.tokens_per_block, a.size_per_token, a.int4_kv);
  if (rc) return rc;
  QS_REQUIRE(a.kv_zeros, "single_query_attention: only kv_cache_with_zeros=True is supported (arg_utils.py:422 always sets it)");
  QS_REQUIRE(a.rotary_dim == kD, "single_query_attention: rotary_dim=%d must equal head_dim (llama_w4a8_unpad.py:258)", a.rotary_dim);
  QS_REQUIRE(a.batch <= 65535, "single_query_attention: batch=%d too large", a.batch);
  PageGeom pg{kPageTokens, kPageTokens * a.size_per_token, a.num_kv_heads};
  const int G = a.num_heads / a.num_kv_heads;
  const int gparts = (G + kMaxG - 1) / kMaxG;
  const int gx = a.num_kv_heads * gparts;
  int nsplit = context_splits(static_cast<long long>(gx) * a.batch, num_sms() * 4, a.timestep);  // over 4 resident CTAs per SM
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
    const int rc = raise_smem_limit(kern, smem, "attention smem attribute");
    if (rc) return rc;
    return launch(kern, grid, dim3(kAttnThreadsV2), smem, 1, a.stream, "single_query_attention", static_cast<const __half*>(a.q),
                  static_cast<const __half*>(a.k), static_cast<const __half*>(a.v), a.q_stride, a.k_stride, a.v_stride, a.kv_pointers, a.lengths,
                  static_cast<__half*>(out), a.num_heads, a.num_kv_heads, a.max_blocks, pg, a.rotary_base, a.rotary_dim, a.timestep, nsplit, part, cnt,
                  tok_cnt, static_cast<int8_t*>(a.q_out), static_cast<__half*>(a.q_scale), static_cast<__half*>(a.q_sum),
                  static_cast<unsigned long long*>(a.prof), static_cast<const int*>(nullptr), 0);
  };
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
    return launch(kern, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, 0, a.stream, "apply_bias_rope_update_kv_cache", static_cast<__half*>(a.qkv),
                  a.seq_lens, a.padding_offset, a.kv_pointers, a.start_pos, a.num_tokens, a.max_blocks, a.num_heads, a.num_kv_heads, a.seq_len, pg,
                  a.rotary_base, a.rotary_dim, a.max_positions, a.tree_mask);
  };
  if (a.tree_mask) {
    QS_REQUIRE(a.start_pos && a.seq_len <= 16, "apply_bias_rope_update_kv_cache_tree: needs start_pos and at most 16 draft nodes per sequence (seq_len=%d)",
               a.seq_len);
    return a.int4_kv ? run(prefill_append_kernel<4, true, true>) : run(prefill_append_kernel<8, true, true>);
  }
  if (a.start_pos) return a.int4_kv ? run(prefill_append_kernel<4, true>) : run(prefill_append_kernel<8, true>);
  return a.int4_kv ? run(prefill_append_kernel<4, false>) : run(prefill_append_kernel<8, false>);
}

int padding_offsets(int* out, const int* cu_seqlens, int batch, int max_seqlen, void* stream) {
  if (batch == 0) return QS_OK;
  return launch(padding_offsets_kernel, dim3(batch), dim3(256), 0, 0, stream, "compute_padding_offsets", out, cu_seqlens, max_seqlen);
}

}  // namespace qs
