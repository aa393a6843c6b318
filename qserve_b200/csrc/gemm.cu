// qserve_b200 -- W4A8 (per-channel / per-group) and W8A8 GEMM for sm_90a.
//
// Replaces  kernels/csrc/qgemm/w4a8_per_chn/gemm_cuda.cu:303-652,
//           kernels/csrc/qgemm/w4a8_per_group/gemm_cuda.cu:328-702,
//           kernels/csrc/qgemm/w8a8/w8a8_gemm_cuda.cu:267-577        (reference: mma.sync + ldmatrix + cp.async)
//
// Hopper design (see DESIGN.md "GEMM"):
//   * swap-AB: the 128 output channels of a tile are the MMA M dimension (two m64 wgmmas), the tokens are MMA N (32 / 64 / 128),
//     so decode-sized batches (M = 64 tokens) still use full-height tensor-core instructions.
//   * the packed INT4 weights are consumed in the checkpoint's own "compute-aware reordered" layout
//     (w4a8_linear.py:292-322): one 32x32 tile is 512 contiguous bytes, a 32-channel band is contiguous in K.
//     ONE TMA tensor copy per 128-K block stages 4 bands x 2 KB into shared memory; each of the four consumer warps reads one
//     16-byte lane chunk per 32 K (LDS.128), splits nibbles in registers (per-group: level-2 dequant q*s2+z2 with the reference's
//     exact 32-bit multiply + vadd4) and hands the INT8 values to wgmma as the REGISTER A operand: the mma.sync B-fragment order of the
//     checkpoint is exactly the wgmma A-fragment order, so no shuffle and no shared-memory round trip is needed.  Channel rows of a
//     band split into the two m64 wgmmas: warp w's lanes give channels 32 w + [0, 16) to the first and 32 w + [16, 32) to the second.
//   * W8A8: the INT8 weight tile comes by TMA with the 128-byte swizzle and is read by wgmma from shared memory.
//   * B (INT8 activations) is TMA-loaded with the 128-byte swizzle; INT32 accumulators live in registers.
//   * weights and activations travel in separate rings with separate producer warps: the weight producer never waits for the previous
//     kernel, so with programmatic dependent launch the weight ring fills while the preceding norm / quant kernel runs.
//   * decode shapes have too few 128-channel tiles to fill 132 SMs, so K is split across a thread-block CLUSTER
//     (2/4/8 CTAs); every CTA stages its INT32 partials in its own shared memory and sends each peer the channels that peer finishes
//     with one bulk copy through DISTRIBUTED SHARED MEMORY (cp.async.bulk.shared::cluster, completing on the peer's mbarrier); each
//     CTA sums and finishes a 1/S slice of the channels -- integer adds, so the result is bit-identical for every split.
//   * epilogue fused: acc*s1[n]*sa[m] - s1z[n]*asum[m] (per-channel) or acc*(s1[n]*sa[m]) (per-group, W8A8) -> fp16,
//     IEEE fp32 in the reference's source order (bit-exact against the oracle).
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "launch.cuh"

namespace qs {

namespace {

constexpr int kBM = 128;  // output channels per tile (two m64 wgmmas)
constexpr int kBK = 128;  // K sub-block (= one g128 group, one 128-byte swizzled activation row)
constexpr int kSub = 2;    // sub-blocks per pipeline stage: per-stage barrier latencies are amortised over 256 K
constexpr int kConsumers = 128;  // warps 0..3: one warpgroup (unpack, wgmma, epilogue)
constexpr int kNumThreads = 192; // + warp 4: weight producer, warp 5: activation producer
constexpr int kFrag = 4;         // W4: wgmma pairs whose A fragments are held in registers at once (kFrag - 1 in flight)

enum { kModeW4Chn = 0, kModeW4Grp = 1, kModeW8 = 2 };

struct GemmParams {
  const uint8_t* s2_scales;  // per-group: [K/128, N] (shuffled per 32 columns, as stored in the checkpoint)
  const uint8_t* s2_zeros;   // per-group: [K/128, N]
  const __half* wscales;     // [N]
  const __half* w_szs;       // [N]  (per-channel only)
  const __half* ascales;     // [M]
  const __half* a_ssums;     // [M]  (per-channel only)
  __half* out;               // [M, N]
  int32_t* acc_out;          // optional: raw INT32 accumulators [M, N] (parity tests)
  int M, N, K;
  int m_tiles, kb_per_tile, split;
  unsigned long long* prof;  // optional: 16 globaltimer stamps per CTA (tools/gemm_timeline.py); slots 13 / 14 / 15 hold NT, the split, the SM id
};

// WS = depth of the WEIGHT ring in shared memory.  Weights are static, so the producer streams them before the
// programmatic-dependent-launch wait: everything that fits in the ring is already on chip when the preceding activation kernel finishes.
template <int MODE, int NT, int WS, int AS>
struct Cfg {
  static constexpr int kActSub = NT * kBK;                                       // one swizzled [NT x 128 B] activation sub-tile
  static constexpr int kWSub = (MODE == kModeW8) ? kBM * kBK : kBM * kBK / 2;   // int8 rows or packed int4 tiles of one sub-block
  static constexpr int kS2Sub = (MODE == kModeW4Grp) ? 2 * kBM : 0;             // scales | zeros of one group
  static constexpr int kActBytes = kSub * kActSub;
  static constexpr int kWBytes = kSub * kWSub;
  static constexpr int kS2Bytes = kSub * kS2Sub;
  static constexpr int kWStageTx = kWBytes + kS2Bytes;
  // shared memory carve-up (offsets from a 1024-aligned base; activation and W8 weight stages are 1024-byte multiples)
  static constexpr int kOffAct = 0;
  static constexpr int kOffW = kOffAct + AS * kActBytes;
  static constexpr int kOffS2 = kOffW + WS * kWBytes;
  static constexpr int kPipeBytes = kOffS2 + WS * kS2Bytes;
  // INT32 partials, aliasing the drained pipeline buffers.  S == 1: the CTA's own tile [NT][128] at offset 0.  Split-K (cluster) launches:
  // at offset 0 the receive buffer [sender][token][128 / S channels], into which the peers copy the partials of the channels this CTA
  // finishes -- only after a cluster barrier has seen every CTA's mainloop drain; behind it the staging buffer [owner][token][128 / S
  // channels], which only this CTA writes, so it may be filled as soon as this CTA's own rings have drained.
  static constexpr int kRedBytes = NT * kBM * 4;
  static constexpr int kOffTx = kRedBytes;
  static_assert(2 * kRedBytes <= kPipeBytes, "receive and staging buffer must both fit in the drained rings");
  static constexpr int kOffRow = (kPipeBytes > kRedBytes ? kPipeBytes : kRedBytes);  // float ascales[NT], asums[NT]
  static constexpr int kOffBar = kOffRow + 2 * NT * 4;
  static constexpr int kNumBars = 2 * WS + 2 * AS + 1;  // + the split-K receive barrier
  static constexpr int kSmemBytes = kOffBar + kNumBars * 8;
  // two co-resident CTAs per SM for the narrow tiles (NT accumulator registers per thread; <= 113 KB of shared memory each), split or not:
  // one CTA's prologue / epilogue overlaps the other's weight stream.  128-token tiles keep 128 accumulators per thread and run one CTA per SM.
  static constexpr int kCtasPerSm = (NT <= 64 && kSmemBytes <= 113 * 1024) ? 2 : 1;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory overflow");
};

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)::"memory");
  return t;
}
#define QS_PROF(slot) do { if (p.prof) p.prof[blockIdx.x * 16 + (slot)] = gtime(); } while (0)

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// split phases of the same barrier (every thread of every CTA arrives once, then waits once): work between them overlaps the peers
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ uint32_t smid() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// bulk copy from this CTA's shared memory into a peer's (dst and bar are shared::cluster addresses of the same peer); the peer's mbarrier
// receives the byte count
__device__ __forceinline__ void bulk_copy_s2peer(uint32_t dst, uint32_t src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "r"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// word swizzle of a row of `width` (16 .. 128) INT32 partials of token `tok`
__device__ __forceinline__ int red_swizzle(int tok, int width) { return (((tok >> 1) & 3) << 3) & (width - 1); }

template <int V>
struct IntTag { static constexpr int value = V; };

template <int MODE>
__device__ __forceinline__ float epilogue_one(int32_t acc, float ws, float wsz, float as, float asum) {
  // IEEE fp32, reference source order, no FMA contraction (bit-exact against oracle/w4a8.py)
  float ps = __int2float_rn(acc);
  if constexpr (MODE == kModeW4Chn) {
    // w4a8_per_chn/gemm_cuda.cu:586  psum * wscale * ascale - w_sz * a_ssum
    float t = __fmul_rn(__fmul_rn(ps, ws), as);
    float u = __fmul_rn(wsz, asum);
    return __fsub_rn(t, u);
  } else {
    // w4a8_per_group/gemm_cuda.cu:619, w8a8_gemm_cuda.cu:522   psum *= wscale * ascale
    return __fmul_rn(ps, __fmul_rn(ws, as));
  }
}

// channel (inside the 128-channel tile) of accumulator row r (0..15) of warp w in m64 wgmma h
template <int MODE>
__device__ __forceinline__ int acc_channel(int h, int w, int r) {
  return (MODE == kModeW8) ? 64 * h + 16 * w + r : 32 * w + 16 * h + r;
}

// grid.x = tiles * split; the `split` CTAs of a cluster share one (n_tile, m_tile) and own disjoint K ranges
template <int MODE, int NT, int WS, int AS, bool ACC>
__global__ void __launch_bounds__(kNumThreads, Cfg<MODE, NT, WS, AS>::kCtasPerSm)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_act, const __grid_constant__ CUtensorMap tmap_w, const GemmParams p) {
  using C = Cfg<MODE, NT, WS, AS>;
  extern __shared__ __align__(1024) uint8_t smem[];  // no static shared memory in this kernel: the window starts 1024-aligned
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* s_act = smem + C::kOffAct;
  uint8_t* s_w = smem + C::kOffW;
  uint8_t* s_s2 = smem + C::kOffS2;
  int32_t* s_red = reinterpret_cast<int32_t*>(smem);  // aliases the pipeline buffers once the mainloop has drained
  float* s_asc = reinterpret_cast<float*>(smem + C::kOffRow);
  float* s_asum = s_asc + NT;
  uint64_t* bar_wfull = reinterpret_cast<uint64_t*>(smem + C::kOffBar);  // weight TMA -> consumers
  uint64_t* bar_wempty = bar_wfull + WS;                                   // consumers (4 warps) -> weight producer
  uint64_t* bar_xfull = bar_wempty + WS;                                   // activation TMA -> consumers
  uint64_t* bar_xempty = bar_xfull + AS;                                   // consumers (4 warps) -> activation producer
  uint64_t* bar_red = bar_xempty + AS;                                     // split-K: the peers' bulk copies -> consumers

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int S = p.split;
  const int rank = (S > 1) ? static_cast<int>(cluster_ctarank()) : 0;
  const int tile = blockIdx.x / S;
  const int m_tile = tile % p.m_tiles, n_tile = tile / p.m_tiles;
  // balanced K split: rank r owns pipeline stages (256 K each) [kb_begin, kb_end)
  const int KB = p.kb_per_tile;
  const int kb_begin = (KB * rank) / S, kb_end = (KB * (rank + 1)) / S;
  const int n_kb = kb_end - kb_begin;
  if (threadIdx.x == 0) {
    QS_PROF(0);
    if (p.prof) {
      p.prof[blockIdx.x * 16 + 13] = NT;
      p.prof[blockIdx.x * 16 + 14] = S;
      p.prof[blockIdx.x * 16 + 15] = smid();
    }
  }
  qs_trace(QS_K_GEMM, 0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_act);
    tma_prefetch_desc(&tmap_w);
    for (int i = 0; i < WS; ++i) {
      mbar_init(&bar_wfull[i], 1);
      mbar_init(&bar_wempty[i], 4);
    }
    for (int i = 0; i < AS; ++i) {
      mbar_init(&bar_xfull[i], 1);
      mbar_init(&bar_xempty[i], 4);
    }
    // split-K: one phase per launch, complete when the S - 1 peer slices (NT x 128 / S partials each) have landed.  The peers copy only
    // after cluster barrier A, which this thread joins after the fence below.
    mbar_init(bar_red, 1);
    if (S > 1) mbar_expect_tx(bar_red, static_cast<uint32_t>((S - 1) * NT * (kBM / S) * 4));
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) { pdl_launch_dependents(); QS_PROF(1); }

  if (warp == 4) {
    // ===================================== weight producer: never waits for the previous kernel =====================================
    if (lane == 0) {
      const int w_row = (MODE == kModeW8) ? n_tile * kBM : n_tile * 4;  // W8: row of [N,K]; W4: band index
      const uint8_t* s2s = p.s2_scales + static_cast<size_t>(n_tile) * kBM;
      const uint8_t* s2z = p.s2_zeros + static_cast<size_t>(n_tile) * kBM;
      // one stage = kSub sub-blocks of 128 K.  A sub-block past the end of K (K % 256 == 128) is zero-filled by the
      // tensor maps (weights and activations), so it contributes nothing; its g128 params are re-read from the last group.
      int s = 0;
      uint32_t ph = 0;  // parity of the (it / WS - 1)-th completion of wempty[s]
      for (int it = 0; it < n_kb; ++it) {
        if (it >= WS) mbar_wait_nocall(&bar_wempty[s], ph);
        mbar_expect_tx(&bar_wfull[s], C::kWStageTx);
#pragma unroll
        for (int u = 0; u < kSub; ++u) {
          const int kb = (kb_begin + it) * kSub + u;
          // W4: u64 elements, 256 per 128-K block of one band (4 tiles x 512 B); W8: bytes
          tma_load_2d(s_w + s * C::kWBytes + u * C::kWSub, &tmap_w, (MODE == kModeW8) ? kb * kBK : kb * 256, w_row, &bar_wfull[s]);
          if constexpr (MODE == kModeW4Grp) {
            const int kg = kb < p.K / kBK ? kb : p.K / kBK - 1;
            bulk_copy_g2s(s_s2 + s * C::kS2Bytes + u * C::kS2Sub, s2s + static_cast<size_t>(kg) * p.N, kBM, &bar_wfull[s]);
            bulk_copy_g2s(s_s2 + s * C::kS2Bytes + u * C::kS2Sub + kBM, s2z + static_cast<size_t>(kg) * p.N, kBM, &bar_wfull[s]);
          }
        }
        if (++s == WS) { s = 0; if (it >= WS) ph ^= 1; }
      }
      QS_PROF(3);
    }
  } else if (warp == 5) {
    // ===================================== activation producer =====================================
    if (lane == 0) {
      const int a_row = m_tile * NT;
      pdl_wait();  // the activations are the previous kernel's output
      QS_PROF(2);
      qs_trace(QS_K_GEMM, 1, 5 * 32);
      int s = 0;
      uint32_t ph = 0;
      for (int it = 0; it < n_kb; ++it) {
        if (it >= AS) mbar_wait_nocall(&bar_xempty[s], ph);
        mbar_expect_tx(&bar_xfull[s], C::kActBytes);
#pragma unroll
        for (int u = 0; u < kSub; ++u)
          tma_load_2d(s_act + s * C::kActBytes + u * C::kActSub, &tmap_act, ((kb_begin + it) * kSub + u) * kBK, a_row, &bar_xfull[s]);
        if (++s == AS) { s = 0; if (it >= AS) ph ^= 1; }
      }
    }
  } else {
    // ===================================== consumer warpgroup: unpack + wgmma + epilogue =====================================
    // warp w owns accumulator rows [16 w, 16 w + 16) of both m64 wgmmas (see acc_channel for the channel each row stands for)
    int32_t acc[2][NT / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[h][i] = 0;
    // No divergent branch and no call may sit between a wgmma issue and its wait (ptxas would serialise every wgmma of the kernel):
    // the first-stage stamp is taken before the loop, stage releases are predicated arrives, barrier waits trap without a printf.
    mbar_wait_nocall(&bar_wfull[0], 0);
    mbar_wait_nocall(&bar_xfull[0], 0);
    if (threadIdx.x == 0) QS_PROF(4);
    const bool leader = lane == 0;
    int sw = 0, sx = 0, prev_sw = WS - 1, prev_sx = AS - 1;
    uint32_t phw = 0, phx = 0;
    for (int it = 0; it < n_kb; ++it) {
      mbar_wait_nocall(&bar_wfull[sw], phw);
      mbar_wait_nocall(&bar_xfull[sx], phx);
      if constexpr (MODE == kModeW8) {
#pragma unroll
        for (int u = 0; u < kSub; ++u) {
          const uint64_t bdesc = gmma_desc_sw128(smem_u32(s_act + sx * C::kActBytes + u * C::kActSub));
          const uint64_t adesc = gmma_desc_sw128(smem_u32(s_w + sw * C::kWBytes + u * C::kWSub));
          wgmma_fence();
#pragma unroll
          for (int t = 0; t < kBK / 32; ++t) {
            wgmma_s8_ss(acc[0], adesc + t * 2, bdesc + t * 2);
            wgmma_s8_ss(acc[1], adesc + (64 * kBK >> 4) + t * 2, bdesc + t * 2);
          }
          wgmma_commit();
        }
        // everything but this stage's kSub groups has retired: the previous stage's weight and activation buffers are free
        wgmma_wait<kSub>();
        mbar_arrive_if(&bar_wempty[prev_sw], it > 0 && leader);
        mbar_arrive_if(&bar_xempty[prev_sx], it > 0 && leader);
      } else {
        // fragment registers of the last kFrag wgmma pairs [pair % kFrag][wgmma h][register]: up to kFrag - 1 pairs stay in flight
        // while the next one is unpacked
        uint32_t fr[kFrag][2][4];
#pragma unroll
        for (int u = 0; u < kSub; ++u) {
          const uint64_t bdesc = gmma_desc_sw128(smem_u32(s_act + sx * C::kActBytes + u * C::kActSub));
          const uint8_t* wsrc = s_w + sw * C::kWBytes + u * C::kWSub + warp * 2048 + lane * 16;
          uint32_t sc4 = 0, zp4 = 0;
          if constexpr (MODE == kModeW4Grp) {
            const uint8_t* s2 = s_s2 + sw * C::kS2Bytes + u * C::kS2Sub + warp * 32 + (lane >> 2) * 4;
            sc4 = *reinterpret_cast<const uint32_t*>(s2);
            zp4 = *reinterpret_cast<const uint32_t*>(s2 + kBM);
          }
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const int j = u * 4 + t;  // pair index inside the stage
            const uint4 v = *reinterpret_cast<const uint4*>(wsrc + t * 512);
            uint32_t xl = v.x & 0x0F0F0F0Fu, xh = (v.x >> 4) & 0x0F0F0F0Fu;
            uint32_t yl = v.y & 0x0F0F0F0Fu, yh = (v.y >> 4) & 0x0F0F0F0Fu;
            uint32_t zl = v.z & 0x0F0F0F0Fu, zh = (v.z >> 4) & 0x0F0F0F0Fu;
            uint32_t wl = v.w & 0x0F0F0F0Fu, wh = (v.w >> 4) & 0x0F0F0F0Fu;
            if constexpr (MODE == kModeW4Grp) {
              // w4a8_per_group/gemm_cuda.cu:298-324: 32-bit multiply of four nibble-bytes, then vadd4 with the s8 zero
              const uint32_t s0 = sc4 & 0xFF, s1 = (sc4 >> 8) & 0xFF, s2 = (sc4 >> 16) & 0xFF, s3 = sc4 >> 24;
              const uint32_t z0 = __byte_perm(zp4, 0, 0x0000), z1 = __byte_perm(zp4, 0, 0x1111);
              const uint32_t z2 = __byte_perm(zp4, 0, 0x2222), z3 = __byte_perm(zp4, 0, 0x3333);
              xl = __vadd4(xl * s0, z0); zl = __vadd4(zl * s0, z0);   // channel c
              yl = __vadd4(yl * s1, z1); wl = __vadd4(wl * s1, z1);   // channel c + 8
              xh = __vadd4(xh * s2, z2); zh = __vadd4(zh * s2, z2);   // channel c + 16
              yh = __vadd4(yh * s3, z3); wh = __vadd4(wh * s3, z3);   // channel c + 24
            }
            // the pair that last read this fragment buffer (kFrag pairs back) must have retired
            wgmma_wait<kFrag - 1>();
            // once pair kFrag - 1 of the stage may be issued, every wgmma of the previous stage has retired: its activation buffer is free
            if (j == kFrag - 1) mbar_arrive_if(&bar_xempty[prev_sx], it > 0 && leader);
            uint32_t(&f)[2][4] = fr[j % kFrag];
            // rows lane/4 (+8) of the band's first 16 channels -> wgmma 0, of its last 16 -> wgmma 1; 32 K per fragment
            f[0][0] = xl; f[0][1] = yl; f[0][2] = zl; f[0][3] = wl;
            f[1][0] = xh; f[1][1] = yh; f[1][2] = zh; f[1][3] = wh;
            wgmma_fence();
            wgmma_s8_rs(acc[0], f[0], bdesc + t * 2);
            wgmma_s8_rs(acc[1], f[1], bdesc + t * 2);
            wgmma_commit();
          }
        }
        // the weight stage has been consumed into registers (every lane's loads fed the last, warp-aligned, wgmma)
        mbar_arrive_if(&bar_wempty[sw], leader);
      }
      prev_sw = sw;
      prev_sx = sx;
      if (++sw == WS) { sw = 0; phw ^= 1; }
      if (++sx == AS) { sx = 0; phx ^= 1; }
    }
    wgmma_wait<0>();
    if (threadIdx.x == 0) QS_PROF(6);
    // Cluster barrier A (split-K): the partials of the peers land in this CTA's pipeline buffers, so every CTA of the cluster must have
    // drained its rings before any partial is sent.  Arrive now; the wait comes after the work below, which touches this CTA only.
    if (S > 1) cluster_arrive();

    // ------------------------------------------ epilogue ------------------------------------------
    // every warp's wgmmas and weight reads are done: this CTA's own rings are free
    named_bar_sync(1, kConsumers);
    const int tid = threadIdx.x;  // 0..127
    const int cps_log2 = 8 - __ffs(S), cps = 1 << cps_log2;  // channels finished per CTA: 128 / S, S a power of two
    // registers -> this CTA's shared memory, [owner][token][channel % cps] (S == 1: [token][channel]), 8-word groups of a token row swizzled
    // by the token so that the four tokens and eight channels of a warp's store fall in 32 banks
    int32_t* s_tx = s_red + (S > 1 ? C::kOffTx / 4 : 0);
    {
      const int r0 = lane >> 2, c0 = (lane & 3) * 2;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) {
          const int ch = acc_channel<MODE>(h, warp, r0 + 8 * ((i >> 1) & 1));
          const int tok = (i >> 2) * 8 + c0 + (i & 1);
          s_tx[(((ch >> cps_log2) * NT + tok) << cps_log2) + ((ch & (cps - 1)) ^ red_swizzle(tok, cps))] = acc[h][i];
        }
    }
    // this CTA finishes channel pairs [64 rank / S, 64 (rank + 1) / S) of the tile for all NT tokens: npairs divides 128, so a thread keeps
    // one channel pair and walks the tokens.  Its weight scales are static; the loads are in flight across the waits below.
    const int npairs = 64 / S;
    const int prl = tid % npairs;  // channel pair inside this CTA's slice
    const int n = n_tile * kBM + 2 * ((64 * rank) / S + prl);
    const float ws0 = __half2float(__ldg(p.wscales + n)), ws1 = __half2float(__ldg(p.wscales + n + 1));
    float wz0 = 0.f, wz1 = 0.f;
    if constexpr (MODE == kModeW4Chn) {
      wz0 = __half2float(__ldg(p.w_szs + n));
      wz1 = __half2float(__ldg(p.w_szs + n + 1));
    }
    pdl_wait();  // ascales / a_ssums / out belong to the dependency chain; every storing thread observes it
    const int m0 = m_tile * NT;
    for (int j = tid; j < NT; j += kConsumers) {
      const bool ok = (m0 + j) < p.M;
      s_asc[j] = ok ? __half2float(p.ascales[m0 + j]) : 0.f;
      if constexpr (MODE == kModeW4Chn) s_asum[j] = ok ? __half2float(p.a_ssums[m0 + j]) : 0.f;
    }
    if (S > 1) {
      fence_proxy_async();  // the staged partials are read by bulk copies
      cluster_wait();       // barrier A: every ring of the cluster has drained
    }
    if (tid == 0) QS_PROF(8);
    named_bar_sync(1, kConsumers);  // staged partials and row scales are visible to the warpgroup
    if (S > 1) {
      // one bulk copy per peer: its slice of the staging buffer -> slot `rank` of its receive buffer, completing on ITS mbarrier
      if (tid < S && tid != rank) {
        const uint32_t slice = static_cast<uint32_t>(NT * cps * 4);
        bulk_copy_s2peer(map_to_cta(smem_u32(s_red) + rank * slice, tid), smem_u32(s_tx) + tid * slice, slice, map_to_cta(smem_u32(bar_red), tid));
      }
      if (tid == 0) QS_PROF(9);
      mbar_wait_nocall(bar_red, 0);  // the S - 1 peer slices have landed
      // Cluster barrier B: a CTA may exit only when the peers' copies have read its staging buffer.  Every CTA arrives after it has
      // received all its slices, so once all have arrived every copy of the cluster is complete.  The wait is at the end of the kernel.
      cluster_arrive();
    } else if (tid == 0) {
      QS_PROF(9);
    }
    if (tid == 0) QS_PROF(10);

    const int tstep = kConsumers / npairs;  // 2 * S tokens are finished per pass of the warpgroup
    const int tok_end = min(NT, p.M - m0);  // tokens of this tile that exist
    const int tok0 = tid / npairs;
    __half* optr = p.out + static_cast<size_t>(m0 + tok0) * p.N + n;
    const size_t ostep = static_cast<size_t>(tstep) * p.N;
    auto finish = [&](int tok, int2 acc, __half* dst) {
      const float as = s_asc[tok], asum = s_asum[tok];
      const float o0 = epilogue_one<MODE>(acc.x, ws0, wz0, as, asum);
      const float o1 = epilogue_one<MODE>(acc.y, ws1, wz1, as, asum);
      *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(o0, o1);  // one packed conversion, each half rounded to nearest even
      if constexpr (ACC) *reinterpret_cast<int2*>(p.acc_out + (dst - p.out)) = acc;
    };
    // S is a launch constant of the cluster: specialise so that the S partials of several tokens are loaded together, then summed
    auto reduce_rows = [&](auto s_tag) {
      constexpr int SS = decltype(s_tag)::value;
      constexpr int CPS = kBM / SS;
      constexpr int TPT = NT / (2 * SS) > 0 ? NT / (2 * SS) : 1;
      constexpr int kChunk = TPT * SS > 16 ? 16 / SS : TPT;  // at most 16 int2 loads in flight per thread
#pragma unroll 1
      for (int i0 = 0; i0 < TPT; i0 += kChunk) {
        int2 v[kChunk][SS];
#pragma unroll
        for (int i = 0; i < kChunk; ++i) {
          const int tok = tok0 + (i0 + i) * tstep;
#pragma unroll
          for (int r = 0; r < SS; ++r) {
            // sender r's partials: in the receive buffer, but this CTA's own never left its staging buffer
            const int32_t* src = (SS > 1 && r != rank) ? s_red + r * NT * CPS : s_tx + rank * NT * CPS;
            v[i][r] = (tok < NT) ? *reinterpret_cast<const int2*>(src + tok * CPS + ((2 * prl) ^ red_swizzle(tok, CPS))) : make_int2(0, 0);
          }
        }
#pragma unroll
        for (int i = 0; i < kChunk; ++i) {
          const int tok = tok0 + (i0 + i) * tstep;
          int2 acc = v[i][0];
#pragma unroll
          for (int r = 1; r < SS; ++r) { acc.x += v[i][r].x; acc.y += v[i][r].y; }
          if (tok < tok_end) finish(tok, acc, optr + (i0 + i) * ostep);
        }
      }
    };
    if (S == 1) reduce_rows(IntTag<1>{});
    else if (S == 2) reduce_rows(IntTag<2>{});
    else if (S == 4) reduce_rows(IntTag<4>{});
    else reduce_rows(IntTag<8>{});
    if (tid == 0) QS_PROF(11);
    if (S > 1) cluster_wait();  // barrier B
    if (tid == 0) QS_PROF(12);
    qs_trace(QS_K_GEMM, 2);
    return;
  }
  // the producer warps take part in both cluster barriers (every thread of the cluster arrives at each) and otherwise stay out of the tail
  if (S > 1) {
    cluster_arrive();
    cluster_wait();
    cluster_arrive();
    cluster_wait();
  }
  // griddepcontrol.wait holds the whole warp: lanes 1..31 get here at once, and the weight producer's lane 0 must go on streaming weights
  // while the previous kernel runs, so the warp reconverges first
  __syncwarp();
  pdl_wait();
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------

// Tensor maps are pure functions of (address, shape, box): cuTensorMapEncodeTiled costs ~1 us of host time and an eager decode step issues
// ~260 of them, so they are memoised (weights: one entry per layer and projection; activations: a handful of buffers).
struct TmapKey {
  const void* ptr; uint64_t a, b; uint32_t box, kind;
  bool operator==(const TmapKey& o) const { return ptr == o.ptr && a == o.a && b == o.b && box == o.box && kind == o.kind; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr) * 0x9E3779B97F4A7C15ull;
    h ^= (k.a + 0x7F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.b * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2));
    return h ^ (static_cast<size_t>(k.box) << 7) ^ k.kind;
  }
};
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash>& tmap_cache() {
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> c;
  return c;
}
std::mutex& tmap_mutex() { static std::mutex m; return m; }
bool tmap_lookup(const TmapKey& k, CUtensorMap* m) {
  std::lock_guard<std::mutex> g(tmap_mutex());
  auto it = tmap_cache().find(k);
  if (it == tmap_cache().end()) return false;
  memcpy(m, &it->second, sizeof(CUtensorMap));
  return true;
}
void tmap_store(const TmapKey& k, const CUtensorMap* m) {
  std::lock_guard<std::mutex> g(tmap_mutex());
  if (tmap_cache().size() > 16384) tmap_cache().clear();  // bounded: a serving loop cycles through a fixed set of buffers
  memcpy(&tmap_cache()[k], m, sizeof(CUtensorMap));
}

// 2-D uint8 tensor [rows, cols] row-major, box {128 bytes, box_rows}, 128-byte swizzle, zero fill out of bounds
int make_tmap_u8(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  const TmapKey key{ptr, rows, cols, box_rows, 0u};
  if (tmap_lookup(key, m)) return QS_OK;
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {128, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): ptr=%p rows=%llu cols=%llu box_rows=%u", (int)r, ptr,
                                          (unsigned long long)rows, (unsigned long long)cols, box_rows);
  tmap_store(key, m);
  return QS_OK;
}

// packed INT4 weights [N, K/2] seen as [N/32 bands][K*16 bytes] of uint64 elements; box = 4 bands x 2 KB (one 128-K block)
int make_tmap_w4(CUtensorMap* m, const void* ptr, uint64_t N, uint64_t K, uint32_t box_bands = 4) {
  const TmapKey key{ptr, N, K, box_bands, 1u};
  if (tmap_lookup(key, m)) return QS_OK;
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {K * 16 / 8, N / 32};
  cuuint64_t strides[1] = {K * 16};
  cuuint32_t box[2] = {256, box_bands};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_INT64, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(QS_ERR_CUDA, "cuTensorMapEncodeTiled(w4) failed (%d): ptr=%p N=%llu K=%llu", (int)r, ptr, (unsigned long long)N,
                                          (unsigned long long)K);
  tmap_store(key, m);
  return QS_OK;
}

// How many clusters of `s` CTAs of `kern` the device holds at once (s == 1: CTAs): the occupancy API's answer for the exact launch
// configuration -- clusters must fit inside one GPC, so this is less than (SMs x CTAs per SM) / s.
int resident_clusters(const void* kern, int smem, int s) {
  int n = 0;
  if (s == 1) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kNumThreads, smem) != cudaSuccess) n = 0;
    return n * num_sms();
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(s);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = s;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) n = 0;
  return n;
}

// resident clusters of `s` CTAs of one instantiation on the current device, queried once per (instantiation, accumulator dump, device, s)
template <int MODE, int NT, int WS, int AS>
int resident_gemm(const GemmArgs& a, int s) {
  using C = Cfg<MODE, NT, WS, AS>;
  auto kern = a.acc_out ? gemm_kernel<MODE, NT, WS, AS, true> : gemm_kernel<MODE, NT, WS, AS, false>;
  static int cache[2][kMaxDevices][4] = {};  // 0 = not yet asked
  int& r = cache[a.acc_out ? 1 : 0][device_ordinal()][s == 1 ? 0 : s == 2 ? 1 : s == 4 ? 2 : 3];
  if (r == 0 && raise_smem_limit(kern, C::kSmemBytes, "cudaFuncSetAttribute(gemm smem)") == QS_OK)
    r = resident_clusters(reinterpret_cast<const void*>(kern), C::kSmemBytes, s);
  return r;
}

template <int MODE, int NT, int WS, int AS>
int launch_gemm(const GemmArgs& a, int split) {
  using C = Cfg<MODE, NT, WS, AS>;
  GemmParams p{};
  p.s2_scales = static_cast<const uint8_t*>(a.s2_scales);
  p.s2_zeros = static_cast<const uint8_t*>(a.s2_zeros);
  p.wscales = static_cast<const __half*>(a.wscales);
  p.w_szs = static_cast<const __half*>(a.w_szs);
  p.ascales = static_cast<const __half*>(a.ascales);
  p.a_ssums = static_cast<const __half*>(a.a_ssums);
  p.out = static_cast<__half*>(a.out);
  p.acc_out = static_cast<int32_t*>(a.acc_out);
  p.prof = static_cast<unsigned long long*>(a.prof);
  p.M = a.M; p.N = a.N; p.K = a.K;
  const int n_tiles = a.N / kBM;
  p.m_tiles = (a.M + NT - 1) / NT;
  p.kb_per_tile = (a.K + kSub * kBK - 1) / (kSub * kBK);  // pipeline stages of 256 K (the last one may be half zero-filled)
  const int tiles = n_tiles * p.m_tiles;

  CUtensorMap tm_act, tm_w;
  int rc = make_tmap_u8(&tm_act, a.act, a.M, a.K, NT);
  if (rc) return rc;
  rc = (MODE == kModeW8) ? make_tmap_u8(&tm_w, a.weight, a.N, a.K, kBM) : make_tmap_w4(&tm_w, a.weight, a.N, a.K);
  if (rc) return rc;

  auto kern = a.acc_out ? gemm_kernel<MODE, NT, WS, AS, true> : gemm_kernel<MODE, NT, WS, AS, false>;
  rc = raise_smem_limit(kern, C::kSmemBytes, "cudaFuncSetAttribute(gemm smem)");
  if (rc) return rc;
  p.split = split;
  if (p.prof)  // profiled launches (tools/gemm_timeline.py) report their plan
    fprintf(stderr, "qs_gemm_plan mode=%d nt=%d ws=%d as=%d M=%d N=%d K=%d tiles=%d split=%d ctas=%d smem=%d resident_clusters=%d\n", MODE, NT, WS,
            AS, a.M, a.N, a.K, tiles, p.split, tiles * p.split, C::kSmemBytes, resident_gemm<MODE, NT, WS, AS>(a, p.split));
  return launch(kern, dim3(tiles * p.split), dim3(kNumThreads), C::kSmemBytes, p.split, a.stream, "gemm launch", tm_act, tm_w, p);
}

// one (MODE, NT) instantiation with its ring depths, as the planner sees it
struct TileImpl {
  int nt;
  int (*resident)(const GemmArgs&, int);
  int (*launch)(const GemmArgs&, int);
};

// The plan of a launch: tokens per tile NT in {32, 64, 128} x cluster split S in {1, 2, 4, 8}.  Candidates: every NT up to the smallest
// one that covers M in one tile (a larger one would be mostly empty), every S that leaves each CTA >= 2 pipeline stages, and only plans
// whose clusters are all resident at once by the occupancy API's answer for that exact instantiation -- one wave by construction.
// `force_nt` / `force_split` (tests, tuning) restrict the candidates to the given value, a forced S without the stage rule (it is
// halved only until every CTA has a stage).  Without a one-wave candidate (prompt-sized M) the launch is the covering tile, unsplit.
// Rule, in this order: fewest stages per CTA, then fewest token tiles (larger NT), then smaller S.
// Measured on an H100 80GB HBM3 (700 W, 1980 MHz max SM clock), us per launch over 32 weight sets in a CUDA graph
// (tools/gemm_split_sweep.py), as NT/S: us.  Llama-3-8B W4A8 per-channel, M = 64:
//   qkv      32/2: 11.17  64/2: 12.12  64/4: 11.19  64/8: 17.05    o     32/2: 10.14  64/2: 10.19  64/4:  9.66  64/8: 15.42
//   gate_up  32/1: 33.97  64/1: 27.78  64/2: 33.18  128/1: 45.49   down  32/2: 22.40  32/4: 25.73  64/2: 23.51  64/4: 18.51  64/8: 24.41
// g128, M = 64:  qkv 32/2: 15.12  64/4: 11.71;  o 32/2: 13.88  64/4: 11.58;  gate_up 64/1: 29.59;  down 32/4: 32.91  64/4: 25.17.
// W8A8, M = 128:  qkv 32/1: 23.70  64/2: 17.10  128/2: 16.94;  o 32/2: 15.17  64/2: 14.77  128/2: 15.00;
//   gate_up 64/1: 60.20 (two waves)  128/1: 61.32;  down 32/2: 41.89  64/2: 40.93  128/2: 39.78.
// Qwen1.5-72B TP = 4 shards, per-channel, M = 64:  qkv (6144 x 8192) 32/2: 15.89  64/4: 15.08;  o (8192 x 2048) 32/2: 9.72  64/2: 9.65;
//   gate_up (12288 x 8192) 32/1: 26.78  64/2: 23.73;  down (8192 x 6144) 32/2: 15.74  64/2: 15.47.
// The rule picks the fastest plan of each of these shapes or one within 2 % of it.  Two token tiles unpack every weight twice, so a
// smaller NT pays only where it buys a deeper split; 32 clusters of 8 do not fit (30 resident), so S = 8 is a second wave.  With the
// scalar remote-store tail this kernel had before, 32/2 measured 1.5 (qkv) and 0.9 us (o) faster than 64/4; the bulk-copy tail removed
// that difference.
inline long plan_cost(int nt, int s, int stages) { return stages * 1000L + (128 - nt) + s; }

template <int MODE>
int dispatch_gemm(const GemmArgs& a) {
  QS_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "gemm: empty problem M=%d N=%d K=%d", a.M, a.N, a.K);
  QS_REQUIRE(a.N % kBM == 0, "gemm: N=%d must be a multiple of %d", a.N, kBM);
  QS_REQUIRE(a.K % kBK == 0, "gemm: K=%d must be a multiple of %d", a.K, kBK);
  QS_REQUIRE((reinterpret_cast<uintptr_t>(a.act) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.weight) & 15) == 0, "gemm: operands must be 16-byte aligned");
  QS_REQUIRE(a.force_split == 0 || a.force_split == 1 || a.force_split == 2 || a.force_split == 4 || a.force_split == 8, "gemm: split must be 1, 2, 4 or 8");
  QS_REQUIRE(a.force_nt == 0 || a.force_nt == 32 || a.force_nt == 64 || a.force_nt == 128, "gemm: tile tokens must be 32, 64 or 128");
  // ring depths (256-K stages): NT <= 64 fits two CTAs per SM (<= 113 KB of shared memory each); 128-token tiles run one CTA per SM and
  // take deeper weight rings.  The split-K receive and staging buffers alias the drained rings, so they cost no shared memory.
  constexpr bool w8 = (MODE == kModeW8), grp = (MODE == kModeW4Grp);
  constexpr int kWs32 = w8 ? 2 : grp ? 4 : 5, kWs64 = w8 ? 2 : grp ? 3 : 4, kAs64 = w8 ? 2 : 3;
  static const TileImpl impls[3] = {{32, resident_gemm<MODE, 32, kWs32, 4>, launch_gemm<MODE, 32, kWs32, 4>},
                                    {64, resident_gemm<MODE, 64, kWs64, kAs64>, launch_gemm<MODE, 64, kWs64, kAs64>},
                                    {128, resident_gemm<MODE, 128, 4, 2>, launch_gemm<MODE, 128, 4, 2>}};
  const int kb = (a.K + kSub * kBK - 1) / (kSub * kBK);
  const int nt_cover = a.M <= 32 ? 32 : a.M <= 64 ? 64 : 128;  // the smallest tile that covers M, or the largest there is
  int forced_s = a.force_split;
  while (forced_s > 1 && kb < forced_s) forced_s /= 2;
  const TileImpl* best = nullptr;
  int best_s = 0;
  long best_cost = 0;
  for (const TileImpl& t : impls) {
    if (a.force_nt > 0 ? t.nt != a.force_nt : t.nt > nt_cover) continue;
    const int tiles = (a.N / kBM) * ((a.M + t.nt - 1) / t.nt);
    for (int s = 1; s <= 8; s *= 2) {
      if (forced_s > 0 ? s != forced_s : (s > 1 && kb < 2 * s)) continue;
      if (tiles > t.resident(a, s)) continue;
      const long cost = plan_cost(t.nt, s, (kb + s - 1) / s);
      if (best == nullptr || cost < best_cost) best = &t, best_s = s, best_cost = cost;
    }
  }
  if (best == nullptr) {  // no one-wave plan (prompt-sized M, or a forced value that does not fit): the widest tile, unsplit unless forced
    best = &impls[(a.force_nt > 0 ? a.force_nt : nt_cover) == 32 ? 0 : (a.force_nt > 0 ? a.force_nt : nt_cover) == 64 ? 1 : 2];
    best_s = forced_s > 0 ? forced_s : 1;
  }
  return best->launch(a, best_s);
}

}  // namespace

int gemm_w4a8_per_chn(const GemmArgs& a) { return dispatch_gemm<kModeW4Chn>(a); }
int gemm_w4a8_per_group(const GemmArgs& a) { return dispatch_gemm<kModeW4Grp>(a); }
int gemm_w8a8(const GemmArgs& a) { return dispatch_gemm<kModeW8>(a); }
size_t gemm_workspace_bytes() { return 4096; }
int gemm_trace_install(void* buf, unsigned cap) { return qs_trace_install(buf, cap); }  // the cluster/DSMEM split-K needs no global workspace; kept for ABI stability

}  // namespace qs
