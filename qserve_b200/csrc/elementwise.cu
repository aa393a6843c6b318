// qserve_b200 -- fused norm / activation / per-token INT8 quantisation kernels (fp16 activations).
//
// Replaces kernels/csrc/layernorm_kernels.cu, fused_kernels.cu, activation_kernels.cu of the reference.
// Each op reads its row from HBM exactly once (row cached in shared memory as fp16), uses 128-bit vector
// accesses, IEEE fp32 arithmetic in the reference's source order, and is PDL-aware (griddepcontrol.wait /
// launch_dependents) so back-to-back launches of the decode step overlap their prologues.
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kThreads = 512;

template <typename Op>
__device__ __forceinline__ float warp_reduce(float v, Op op) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, m));
  return v;
}
struct OpSum { __device__ float operator()(float a, float b) const { return a + b; } };
struct OpMax { __device__ float operator()(float a, float b) const { return fmaxf(a, b); } };

// block-wide all-reduce for kThreads threads; red must hold >= 32 floats; result broadcast to all threads
template <typename Op>
__device__ __forceinline__ float block_reduce(float v, float* red, Op op, float identity) {
  v = warp_reduce(v, op);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();  // protect red reuse
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = (l < (blockDim.x >> 5)) ? red[l] : identity;
  r = warp_reduce(r, op);
  return r;
}

// block-wide sum of the fixed-point row sums (fx_of_half, common.cuh)
__device__ __forceinline__ long long block_sum_ll(long long v, long long* red) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  long long r = (l < (blockDim.x >> 5)) ? red[l] : 0ll;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) r += __shfl_xor_sync(0xffffffffu, r, m);
  return r;
}

// cluster exchange of the silu_mul_quant kernels: one 64-bit word carries the CTA's amax (low half) and non-finite sum (high half)
__device__ __forceinline__ long long pack_amax_nf(float amax, float nf) {
  return static_cast<long long>((static_cast<unsigned long long>(__float_as_uint(nf)) << 32) | __float_as_uint(amax));
}
__device__ __forceinline__ float unpack_amax(long long v) { return __uint_as_float(static_cast<uint32_t>(v)); }
__device__ __forceinline__ float unpack_nf(long long v) { return __uint_as_float(static_cast<uint32_t>(static_cast<unsigned long long>(v) >> 32)); }

__device__ __forceinline__ void load_row_to_smem(__half* dst, const __half* src, int H) {
  // H % 8 == 0 guaranteed by the host wrapper
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) d[i] = __ldg(s + i);
}

// ------------------------------------------------------------------------------------------------
// N1: rms_norm_general[_fuse_sum]  (generalLayerNorm[_fuse_sum], layernorm_kernels.cu:53-326)
//     mean-subtracting layer norm + per-token INT8 quant (+ fp16-accumulated row sum, reference thread grouping)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) layernorm_quant_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                  const __half* __restrict__ gamma, __half* __restrict__ input_sum,
                                                                  __half* __restrict__ scaling, float eps, int H, int ref_block,
                                                                  bool per_token) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sx = reinterpret_cast<__half*>(sm);  // x row
  __half* sy = sx + H;                         // half(y) row (only for the fused sum)
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  qs_trace(QS_K_NORM, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  pdl_wait();
  qs_trace(QS_K_NORM, 1);
  load_row_to_smem(sx, in + static_cast<size_t>(row) * H, H);
  __syncthreads();

  float s = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      s += f.x + f.y;
    }
  }
  const float mean = __fdiv_rn(block_reduce(s, red, OpSum(), 0.f), static_cast<float>(H));
  float vs = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      const float a = f.x - mean, b = f.y - mean;
      vs += a * a + b * b;
    }
  }
  const float var = block_reduce(vs, red, OpSum(), 0.f);
  const float rstd = __frsqrt_rn(__fadd_rn(__fdiv_rn(var, static_cast<float>(H)), eps));

  if (!per_token) {
    // per-tensor static scale: q = rni_sat(half(y) * scale)   (layernorm_kernels.cu:159-163)
    const float sc = __half2float(scaling[0]);
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      const float y = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(sx[i]), mean), rstd), __half2float(gamma[i]));
      out[static_cast<size_t>(row) * H + i] = cvt_s8(__fmul_rn(__half2float(__float2half_rn(y)), sc));
    }
    return;
  }

  // pass 3: amax of half(y) (init 1e-6 in fp16), optionally stash half(y) for the sum
  float amax = __half2float(__float2half_rn(1e-6f));
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(gamma) + i);
    const __half* h = reinterpret_cast<const __half*>(&v);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    uint4 yv;
    __half* yh = reinterpret_cast<__half*>(&yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float y = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(h[j]), mean), rstd), __half2float(gh[j]));
      yh[j] = __float2half_rn(y);
      amax = fmaxf(amax, fabsf(__half2float(yh[j])));
    }
    if (input_sum) reinterpret_cast<uint4*>(sy)[i] = yv;
  }
  amax = block_reduce(amax, red, OpMax(), 0.f);  // (includes the barrier that publishes sy)
  if (input_sum) {
    // reference thread t (of ref_block threads) accumulates y_h[t], y_h[t+B], ... sequentially IN FP16 (:275,286)
    long long part = 0;
    for (int t = threadIdx.x; t < ref_block; t += blockDim.x) {
      __half acc = __float2half_rn(0.f);
      for (int i = t; i < H; i += ref_block) acc = __hadd(acc, sy[i]);
      part += fx_of_half(__half2float(acc));
    }
    const long long total = block_sum_ll(part, red_ll);
    if (threadIdx.x == 0) input_sum[row] = __float2half_rn(fx_to_float(total));
  }
  if (threadIdx.x == 0) scaling[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
  const float qs_ = __fdiv_rn(127.f, amax);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(gamma) + i);
    const __half* h = reinterpret_cast<const __half*>(&v);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(h[j]), mean), rstd), __half2float(gh[j]));
    store_q8(out + static_cast<size_t>(row) * H, i, y, qs_);  // quantises the UN-rounded fp32 y (:307-318)
  }
}

// ------------------------------------------------------------------------------------------------
// Fused extensions (bit-identical to the unfused op sequences they replace; tests/test_gpu_fused.py)
//   add_layernorm_quant : hidden = half(x + delta)  [torch `residual + out_buf`, llama_w4a8_unpad.py:348,360]  -> N1
//   silu_mul_quant      : act = silu_and_mul(in)    [activation.py:24-29]                                      -> Q1
// ------------------------------------------------------------------------------------------------
constexpr int kFusedThreads = kThreads;  // same thread count and loop order as the unfused kernels -> bit-identical sums

constexpr int kGammaPre = 4;  // gamma chunks (8 halves each) a thread keeps in registers: covers H <= 8192 at 256 threads

// Tensor parallelism: the sum-all-reduce of the row-parallel GEMM output FUSED into the consumer (residual add + norm + quant).
// Every rank's GEMM writes its fp16 partial [M, H] into a peer-mapped (NVLink / NVSwitch symmetric-memory) buffer; this kernel
//   1. (after its own GEMM is complete: griddepcontrol.wait) raises a flag in every peer's flag pad:  flags[r][phase * 8 + me] = epoch,
//   2. waits until all peers' flags have reached the epoch in ITS pad (their partials are complete),
//   3. pulls the token row of all ranks with 128-bit peer loads, sums them in fp32 IN RANK ORDER (every rank computes the same bits),
//      rounds once to fp16 -- the value an fp16 all-reduce would have delivered, without its per-hop roundings -- and continues as
//      add_rms_norm_general.  No NCCL call, no extra kernel boundary, the NVLink transfer overlaps the other rows' norm arithmetic.
// Two phases (o_proj / down_proj) use two buffers, so a rank that runs ahead can never overwrite a partial a slower peer still reads:
// buffer p is rewritten only after a kernel that waited for the peers' NEXT-phase flags (see DESIGN.md 6).
struct PeerArgs {
  const __half* delta[8];   // partial-output buffer of this phase on every rank (peer-mapped addresses), indexed by rank
  uint32_t* flags[8];       // flag pad of every rank (peer-mapped): 16 x u32, [phase * 8 + source rank]
  uint32_t* state;          // local: [phase] = epoch of the last completed launch, [2 + phase] = finished-CTA counter
  int world, rank, phase;
};
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint4 ld_peer_v4(const uint4* p) {  // peer memory: bypass the (incoherent) L1
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

template <bool PEER>
__global__ void __launch_bounds__(kFusedThreads) add_layernorm_quant_kernel(int8_t* __restrict__ out, __half* __restrict__ hidden_out,
                                                                           const __half* __restrict__ x, const __half* __restrict__ delta,
                                                                           const __half* __restrict__ gamma, __half* __restrict__ input_sum,
                                                                           __half* __restrict__ scaling, float eps, int H, int ref_block, const PeerArgs peer) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sx = reinterpret_cast<__half*>(sm);
  __half* sy = sx + H;
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  qs_trace(QS_K_ADDNORM, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  // gamma is a static weight: fetch this thread's chunks before waiting for the producer of x / delta
  uint4 gpre[kGammaPre];
#pragma unroll
  for (int e = 0; e < kGammaPre; ++e) {
    const int i = threadIdx.x + e * blockDim.x;
    gpre[e] = (i < H / 8) ? __ldg(reinterpret_cast<const uint4*>(gamma) + i) : make_uint4(0u, 0u, 0u, 0u);
  }
  pdl_wait();
  qs_trace(QS_K_ADDNORM, 1);
  uint32_t epoch = 0;
  if constexpr (PEER) {
    epoch = *reinterpret_cast<volatile uint32_t*>(peer.state + peer.phase) + 1u;
    if (blockIdx.x == 0 && threadIdx.x < peer.world) st_release_sys(peer.flags[threadIdx.x] + peer.phase * 8 + peer.rank, epoch);
    if (threadIdx.x < peer.world) {
      const uint32_t* mine = peer.flags[peer.rank] + peer.phase * 8 + threadIdx.x;
      unsigned spins = 0;
      while (static_cast<int32_t>(ld_acquire_sys(mine) - epoch) < 0) {
        __nanosleep(40);
        if (++spins > (1u << 27)) {  // several seconds: a peer died or the ranks disagree on the launch sequence
          printf("qserve_b200: peer all-reduce timed out (rank %d waits for rank %d, phase %d, epoch %u)\n", peer.rank, threadIdx.x, peer.phase, epoch);
          __trap();
        }
      }
    }
    __syncthreads();
  }
  {
    const uint4* a = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * H);
    const uint4* b = reinterpret_cast<const uint4*>(delta + static_cast<size_t>(row) * H);
    uint4* ho = reinterpret_cast<uint4*>(hidden_out + static_cast<size_t>(row) * H);
    for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
      const uint4 va = __ldg(a + i);
      uint4 vb;
      if constexpr (PEER) {
        // all ranks' partials of this 16-byte column chunk: issue every peer load first, then sum in rank order (fp32), round once
        uint4 pv[8];
#pragma unroll
        for (int r = 0; r < 8; ++r)
          if (r < peer.world) pv[r] = ld_peer_v4(reinterpret_cast<const uint4*>(peer.delta[r] + static_cast<size_t>(row) * H) + i);
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          if (r < peer.world) {
            const __half2* hp = reinterpret_cast<const __half2*>(&pv[r]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 f = __half22float2(hp[j]);
              acc[2 * j] = __fadd_rn(acc[2 * j], f.x);
              acc[2 * j + 1] = __fadd_rn(acc[2 * j + 1], f.y);
            }
          }
        }
        __half2* hb2 = reinterpret_cast<__half2*>(&vb);
#pragma unroll
        for (int j = 0; j < 4; ++j) hb2[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
      } else {
        vb = __ldg(b + i);
      }
      uint4 vo;
      const __half2* ha = reinterpret_cast<const __half2*>(&va);
      const __half2* hb = reinterpret_cast<const __half2*>(&vb);
      __half2* ho2 = reinterpret_cast<__half2*>(&vo);
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // torch half add: float(a) + float(b), rounded once to fp16
        const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
        ho2[j] = __floats2half2_rn(__fadd_rn(fa.x, fb.x), __fadd_rn(fa.y, fb.y));
      }
      reinterpret_cast<uint4*>(sx)[i] = vo;
      ho[i] = vo;
    }
  }
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      s += f.x + f.y;
    }
  }
  const float mean = __fdiv_rn(block_reduce(s, red, OpSum(), 0.f), static_cast<float>(H));
  float vs = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      const float a = f.x - mean, b = f.y - mean;
      vs += a * a + b * b;
    }
  }
  const float var = block_reduce(vs, red, OpSum(), 0.f);
  const float rstd = __frsqrt_rn(__fadd_rn(__fdiv_rn(var, static_cast<float>(H)), eps));
  float amax = __half2float(__float2half_rn(1e-6f));
  auto norm_chunk = [&](int i, const uint4& g) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half* h = reinterpret_cast<const __half*>(&v);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    uint4 yv;
    __half* yh = reinterpret_cast<__half*>(&yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float y = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(h[j]), mean), rstd), __half2float(gh[j]));
      yh[j] = __float2half_rn(y);
      amax = fmaxf(amax, fabsf(__half2float(yh[j])));
    }
    if (input_sum) reinterpret_cast<uint4*>(sy)[i] = yv;
  };
#pragma unroll
  for (int e = 0; e < kGammaPre; ++e) {
    const int i = threadIdx.x + e * blockDim.x;
    if (i < H / 8) norm_chunk(i, gpre[e]);
  }
  for (int i = threadIdx.x + kGammaPre * blockDim.x; i < H / 8; i += blockDim.x) norm_chunk(i, __ldg(reinterpret_cast<const uint4*>(gamma) + i));
  amax = block_reduce(amax, red, OpMax(), 0.f);
  if (input_sum) {
    long long part = 0;
    for (int t = threadIdx.x; t < ref_block; t += blockDim.x) {
      __half acc = __float2half_rn(0.f);
      for (int i = t; i < H; i += ref_block) acc = __hadd(acc, sy[i]);
      part += fx_of_half(__half2float(acc));
    }
    const long long total = block_sum_ll(part, red_ll);
    if (threadIdx.x == 0) input_sum[row] = __float2half_rn(fx_to_float(total));
  }
  if (threadIdx.x == 0) scaling[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
  const float qs_ = __fdiv_rn(127.f, amax);
  auto quant_chunk = [&](int i, const uint4& g) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half* h = reinterpret_cast<const __half*>(&v);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(h[j]), mean), rstd), __half2float(gh[j]));
    store_q8(out + static_cast<size_t>(row) * H, i, y, qs_);
  };
#pragma unroll
  for (int e = 0; e < kGammaPre; ++e) {
    const int i = threadIdx.x + e * blockDim.x;
    if (i < H / 8) quant_chunk(i, gpre[e]);
  }
  for (int i = threadIdx.x + kGammaPre * blockDim.x; i < H / 8; i += blockDim.x) quant_chunk(i, __ldg(reinterpret_cast<const uint4*>(gamma) + i));
  if constexpr (PEER) {
    // the last CTA of the launch to get here publishes the epoch for the next launch of this phase (stream order separates the two)
    if (threadIdx.x == 0) {
      const uint32_t old = atomicAdd(peer.state + 2 + peer.phase, 1u);
      if (old == gridDim.x - 1) {
        peer.state[2 + peer.phase] = 0u;
        *reinterpret_cast<volatile uint32_t*>(peer.state + peer.phase) = epoch;
      }
    }
  }
}

__device__ __forceinline__ __half silu_h_fused(__half x) {
  const float f = __half2float(x);
  return __float2half_rn(__fdiv_rn(f, __fadd_rn(1.0f, expf(-f))));
}

// One row is split across a cluster of `csize` CTAs (all SMs busy even at 64 tokens); the row amax / sum are exchanged
// through distributed shared memory.  grid.x = tokens * csize.
constexpr int kSiluQuantThreads = 256;  // exact sums / max: the result does not depend on the thread count (measured: 256 beats 512 here)
__global__ void __launch_bounds__(kSiluQuantThreads) silu_mul_quant_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                      __half* __restrict__ input_sum, __half* __restrict__ scale, int d, int csize) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sa = reinterpret_cast<__half*>(sm);  // this CTA's slice of the activation row (fp16)
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  __shared__ __align__(16) long long s_part[2];  // [0] = pack_amax_nf(local amax, local non-finite sum), [1] = local fixed-point sum
  const int row = blockIdx.x / csize;
  const int rank = blockIdx.x - row * csize;
  const int dl = d / csize;  // columns of this CTA (multiple of 8)
  qs_trace(QS_K_SILUQ, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  pdl_wait();
  qs_trace(QS_K_SILUQ, 1);
  const uint4* gx = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * 2 * d + static_cast<size_t>(rank) * dl);
  const uint4* gy = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * 2 * d + d + static_cast<size_t>(rank) * dl);
  float amax = 0.f, nf = 0.f;
  long long s = 0;
  for (int i = threadIdx.x; i < dl / 8; i += blockDim.x) {
    const uint4 x = __ldg(gx + i), y = __ldg(gy + i);
    const __half* xh = reinterpret_cast<const __half*>(&x);
    const __half* yh = reinterpret_cast<const __half*>(&y);
    uint4 o;
    __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      oh[j] = __hmul(silu_h_fused(xh[j]), yh[j]);
      const float f = __half2float(oh[j]);
      if (input_sum) { s += fx_of_finite(f); nf += nonfinite_part(f); }
      amax = fmaxf(amax, fabsf(f));
    }
    reinterpret_cast<uint4*>(sa)[i] = o;
  }
  amax = block_reduce(amax, red, OpMax(), 0.f);  // (the barriers inside also publish sa)
  long long total = 0;
  if (input_sum) {
    total = block_sum_ll(s, red_ll);
    nf = block_reduce(nf, red, OpSum(), 0.f);
  }
  if (csize > 1) {
    if (threadIdx.x == 0) {
      s_part[0] = pack_amax_nf(amax, nf);
      s_part[1] = total;
    }
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    const uint32_t base = static_cast<uint32_t>(__cvta_generic_to_shared(s_part));
    amax = 0.f;
    nf = 0.f;
    total = 0;
    for (int r = 0; r < csize; ++r) {
      uint32_t peer;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer) : "r"(base), "r"(r));
      long long a, b;
      asm volatile("ld.shared::cluster.v2.s64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "r"(peer) : "memory");
      amax = fmaxf(amax, unpack_amax(a));
      nf += unpack_nf(a);
      total += b;
    }
  }
  if (rank == 0 && threadIdx.x == 0) {
    scale[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
    if (input_sum) input_sum[row] = __float2half_rn(row_sum(total, nf));
  }
  const float qs_ = __fdiv_rn(127.f, amax);
  int8_t* orow = out + static_cast<size_t>(row) * d + static_cast<size_t>(rank) * dl;
  for (int i = threadIdx.x; i < dl / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sa)[i];
    const __half* h = reinterpret_cast<const __half*>(&v);
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = __half2float(h[j]);
    store_q8(orow, i, x, qs_);
  }
  // peers may still be reading s_part
  if (csize > 1) asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
}

// Register-resident form of silu_mul_quant_kernel for slices of at most 2 x 256 vectors per CTA (every benchmark shape): the activation
// stays in registers, the two block reductions need one barrier each, and the cluster exchange is PUSH based -- every CTA stores its
// (amax, sum) into all peers' tables before ONE cluster barrier and reads only its own shared memory afterwards, so no trailing barrier keeps
// the CTAs alive.  Same arithmetic (exact sums, max) as the kernel above: bit-identical results.
template <int CHS>
__global__ void __launch_bounds__(kSiluQuantThreads) silu_mul_quant_fast_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                           __half* __restrict__ input_sum, __half* __restrict__ scale, int d, int csize) {
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  __shared__ float red_nf[32];
  __shared__ __align__(16) long long s_rx[8][2];  // [sender]: pack_amax_nf(its amax, its non-finite sum), its fixed-point sum
  const int row = blockIdx.x / csize;
  const int rank = blockIdx.x - row * csize;
  const int dl = d / csize;
  const int nvec = dl / 8;
  qs_trace(QS_K_SILUQ, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  qs_trace(QS_K_SILUQ, 1);
  const uint4* gx = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * 2 * d + static_cast<size_t>(rank) * dl);
  const uint4* gy = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * 2 * d + d + static_cast<size_t>(rank) * dl);
  uint4 xin[CHS], yin[CHS];
#pragma unroll
  for (int c = 0; c < CHS; ++c) {  // all loads of the thread in flight together
    const int i = threadIdx.x + c * kSiluQuantThreads;
    if (i < nvec) { xin[c] = __ldg(gx + i); yin[c] = __ldg(gy + i); }
  }
  float act[CHS][8];
  float amax = 0.f, nf = 0.f;
  long long s = 0;
#pragma unroll
  for (int c = 0; c < CHS; ++c) {
    if (threadIdx.x + c * kSiluQuantThreads < nvec) {
      const __half* xh = reinterpret_cast<const __half*>(&xin[c]);
      const __half* yh = reinterpret_cast<const __half*>(&yin[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float f = __half2float(__hmul(silu_h_fused(xh[j]), yh[j]));
        act[c][j] = f;
        if (input_sum) { s += fx_of_finite(f); nf += nonfinite_part(f); }
        amax = fmaxf(amax, fabsf(f));
      }
    }
  }
  // one barrier for both block reductions: warp partials of amax and of the exact sum are published together
  amax = warp_reduce(amax, OpMax());
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if (input_sum) nf = warp_reduce(nf, OpSum());
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[w] = amax; red_ll[w] = s; red_nf[w] = nf; }
  __syncthreads();
  amax = (l < (kSiluQuantThreads >> 5)) ? red[l] : 0.f;
  amax = warp_reduce(amax, OpMax());
  long long total = (l < (kSiluQuantThreads >> 5)) ? red_ll[l] : 0ll;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) total += __shfl_xor_sync(0xffffffffu, total, m);
  if (input_sum) nf = warp_reduce((l < (kSiluQuantThreads >> 5)) ? red_nf[l] : 0.f, OpSum());
  if (csize > 1) {
    if (threadIdx.x < csize) {  // thread r pushes this CTA's pair into CTA r's table
      uint32_t peer;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer) : "r"(static_cast<uint32_t>(__cvta_generic_to_shared(&s_rx[rank][0]))), "r"(threadIdx.x));
      asm volatile("st.shared::cluster.v2.s64 [%0], {%1, %2};" ::"r"(peer), "l"(pack_amax_nf(amax, nf)), "l"(total) : "memory");
    }
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    amax = 0.f;
    nf = 0.f;
    total = 0;
    for (int r = 0; r < csize; ++r) {
      amax = fmaxf(amax, unpack_amax(s_rx[r][0]));
      nf += unpack_nf(s_rx[r][0]);
      total += s_rx[r][1];
    }
  }
  if (rank == 0 && threadIdx.x == 0) {
    scale[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
    if (input_sum) input_sum[row] = __float2half_rn(row_sum(total, nf));
  }
  const float qs_ = __fdiv_rn(127.f, amax);
  int8_t* orow = out + static_cast<size_t>(row) * d + static_cast<size_t>(rank) * dl;
#pragma unroll
  for (int c = 0; c < CHS; ++c) {
    const int i = threadIdx.x + c * kSiluQuantThreads;
    if (i < nvec) store_q8(orow, i, act[c], qs_);
  }
}

// ------------------------------------------------------------------------------------------------
// Q1: invoke_quant / invoke_quant_fuse_sum (per-token)   fused_kernels.cu:52-137
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) quant_per_token_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                  __half* __restrict__ input_sum, __half* __restrict__ scale, int H) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sx = reinterpret_cast<__half*>(sm);
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  qs_trace(QS_K_QUANT, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  pdl_wait();
  qs_trace(QS_K_QUANT, 1);
  load_row_to_smem(sx, in + static_cast<size_t>(row) * H, H);
  __syncthreads();
  float amax = 0.f, nf = 0.f;
  long long s = 0;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      if (input_sum) {
        s += fx_of_finite(f.x) + fx_of_finite(f.y);
        nf += nonfinite_part(f.x) + nonfinite_part(f.y);
      }
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  amax = block_reduce(amax, red, OpMax(), 0.f);
  if (input_sum) {
    const long long total = block_sum_ll(s, red_ll);
    nf = block_reduce(nf, red, OpSum(), 0.f);
    if (threadIdx.x == 0) input_sum[row] = __float2half_rn(row_sum(total, nf));
  }
  if (threadIdx.x == 0) scale[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
  const float qs_ = __fdiv_rn(127.f, amax);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half* h = reinterpret_cast<const __half*>(&v);
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = __half2float(h[j]);
    store_q8(out + static_cast<size_t>(row) * H, i, x, qs_);
  }
}

// Tensor-parallel parity rule (SURVEY.md 8e): a row-parallel GEMM keeps INT32 partial sums that add up to the single-GPU
// accumulators only if every rank quantises its K shard of a token with the SAME per-token scale.  row_absmax -> [M] fp32
// max-allreduce -> quant_given_amax does exactly the arithmetic of quant_per_token_kernel with the global amax; the row sum
// (per-channel W4A8 zero-point term) stays the LOCAL shard's sum.
__global__ void __launch_bounds__(kThreads) row_absmax_kernel(float* __restrict__ amax_out, const __half* __restrict__ in, int H) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const uint4* src = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * H);
  float amax = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = src[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  amax = block_reduce(amax, red, OpMax(), 0.f);
  if (threadIdx.x == 0) amax_out[row] = amax;
}

__global__ void __launch_bounds__(kThreads) quant_given_amax_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                   const float* __restrict__ amax_in, __half* __restrict__ input_sum,
                                                                   __half* __restrict__ scale, int H) {
  __shared__ float red[32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const float amax = amax_in[row];
  const float qs_ = __fdiv_rn(127.f, amax);
  const uint4* src = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * H);
  long long s = 0;
  float nf = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = src[i];
    const __half* h = reinterpret_cast<const __half*>(&v);
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      x[j] = __half2float(h[j]);
      if (input_sum) { s += fx_of_finite(x[j]); nf += nonfinite_part(x[j]); }
    }
    store_q8(out + static_cast<size_t>(row) * H, i, x, qs_);
  }
  if (input_sum) {
    const long long total = block_sum_ll(s, red_ll);
    nf = block_reduce(nf, red, OpSum(), 0.f);
    if (threadIdx.x == 0) input_sum[row] = __float2half_rn(row_sum(total, nf));
  }
  if (threadIdx.x == 0) scale[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
}

// Register-resident form of quant_per_token_kernel for rows of at most 4 x 512 vectors (H <= 16384: every benchmark shape): one global pass, the
// max and the exact sum are reduced behind a single barrier.  Same arithmetic: bit-identical results.
template <int CH>
__global__ void __launch_bounds__(kThreads) quant_per_token_fast_kernel(int8_t* __restrict__ out, const __half* __restrict__ in,
                                                                       __half* __restrict__ input_sum, __half* __restrict__ scale, int H) {
  __shared__ float red[32];
  __shared__ float red_nf[32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  const int nvec = H / 8;
  qs_trace(QS_K_QUANT, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  qs_trace(QS_K_QUANT, 1);
  const uint4* src = reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * H);
  uint4 xv[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    xv[c] = (i < nvec) ? __ldg(src + i) : make_uint4(0u, 0u, 0u, 0u);
  }
  float amax = 0.f, nf = 0.f;
  long long s = 0;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (threadIdx.x + c * kThreads < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&xv[c]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        if (input_sum) {
          s += fx_of_finite(f.x) + fx_of_finite(f.y);
          nf += nonfinite_part(f.x) + nonfinite_part(f.y);
        }
        amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
  }
  amax = warp_reduce(amax, OpMax());
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
  if (input_sum) nf = warp_reduce(nf, OpSum());
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[w] = amax; red_ll[w] = s; red_nf[w] = nf; }
  __syncthreads();
  amax = (l < (kThreads >> 5)) ? red[l] : 0.f;
  amax = warp_reduce(amax, OpMax());
  if (input_sum && threadIdx.x < 32) {
    long long total = (l < (kThreads >> 5)) ? red_ll[l] : 0ll;
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) total += __shfl_xor_sync(0xffffffffu, total, m);
    nf = warp_reduce((l < (kThreads >> 5)) ? red_nf[l] : 0.f, OpSum());
    if (threadIdx.x == 0) input_sum[row] = __float2half_rn(row_sum(total, nf));
  }
  if (threadIdx.x == 0) scale[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
  const float qs_ = __fdiv_rn(127.f, amax);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    if (i < nvec) {
      const __half* h = reinterpret_cast<const __half*>(&xv[c]);
      float x[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = __half2float(h[j]);
      store_q8(out + static_cast<size_t>(row) * H, i, x, qs_);
    }
  }
}

__global__ void quant_scalar_kernel(int8_t* __restrict__ out, const __half* __restrict__ in, float scale, size_t n) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = cvt_s8(__fdiv_rn(__half2float(in[i]), scale));
}

// ------------------------------------------------------------------------------------------------
// N2: rms_norm   layernorm_kernels.cu:330-360
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) rms_norm_kernel(void* __restrict__ out, const __half* __restrict__ in,
                                                           const __half* __restrict__ weight, float eps, int H, bool use_quant) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sx = reinterpret_cast<__half*>(sm);
  __shared__ float red[32];
  const int row = blockIdx.x;
  qs_trace(QS_K_RMS, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  pdl_wait();
  qs_trace(QS_K_RMS, 1);
  load_row_to_smem(sx, in + static_cast<size_t>(row) * H, H);
  __syncthreads();
  float vs = 0.f;
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      vs += f.x * f.x + f.y * f.y;
    }
  }
  const float var = block_reduce(vs, red, OpSum(), 0.f);
  const float rstd = __frsqrt_rn(__fadd_rn(__fdiv_rn(var, static_cast<float>(H)), eps));
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) {
    const uint4 v = reinterpret_cast<const uint4*>(sx)[i];
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(weight) + i);
    const __half* h = reinterpret_cast<const __half*>(&v);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    if (use_quant) {
      float y[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = __fmul_rn(__fmul_rn(__half2float(h[j]), rstd), __half2float(gh[j]));
      store_q8(static_cast<int8_t*>(out) + static_cast<size_t>(row) * H, i, y, 1.0f);
    } else {
      uint4 o;
      __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) oh[j] = __hmul(__float2half_rn(__fmul_rn(__half2float(h[j]), rstd)), gh[j]);  // fp16 product (:356-357)
      reinterpret_cast<uint4*>(static_cast<__half*>(out) + static_cast<size_t>(row) * H)[i] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// A0: silu_and_mul   activation_kernels.cu:10-30
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ __half silu_h(__half x) {
  const float f = __half2float(x);
  return __float2half_rn(__fdiv_rn(f, __fadd_rn(1.0f, expf(-f))));
}
// Grid-stride over 16-byte vectors of the [tokens, d] output with two vectors per thread in flight: at prompt sizes (8192 x 14336) the first version
// -- one CTA per 1024 outputs, 114688 short-lived CTAs -- left a third of the HBM bandwidth unused; now 705 MB in 143 us = 4.9 TB/s.
__global__ void __launch_bounds__(256) silu_and_mul_kernel(__half* __restrict__ out, const __half* __restrict__ in, int d, long long n_vec) {
  qs_trace(QS_K_SILU, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();  // dependents may become resident (and prefetch static data) right away
  pdl_wait();
  qs_trace(QS_K_SILU, 1);
  const int vpr = d / 8;  // vectors per output row
  auto one = [&](long long v, uint4& x, uint4& y) {
    const long long row = v / vpr;
    const int c = static_cast<int>(v - row * vpr);
    const uint4* gx = reinterpret_cast<const uint4*>(in + row * 2 * d);
    x = __ldg(gx + c);
    y = __ldg(gx + vpr + c);
  };
  auto act = [&](const uint4& x, const uint4& y) {
    const __half* xh = reinterpret_cast<const __half*>(&x);
    const __half* yh = reinterpret_cast<const __half*>(&y);
    uint4 o;
    __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
#pragma unroll
    for (int j = 0; j < 8; ++j) oh[j] = __hmul(silu_h(xh[j]), yh[j]);
    return o;
  };
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  uint4* go = reinterpret_cast<uint4*>(out);
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < n_vec; v += 2 * stride) {
    uint4 x0, y0, x1 = make_uint4(0, 0, 0, 0), y1 = x1;
    const bool two = v + stride < n_vec;
    one(v, x0, y0);
    if (two) one(v + stride, x1, y1);
    go[v] = act(x0, y0);
    if (two) go[v + stride] = act(x1, y1);
  }
}

// ------------------------------------------------------------------------------------------------
// legacy exports (not reached by llama_w4a8 / llama_w8a8; API completeness)
// ------------------------------------------------------------------------------------------------
__global__ void gelu_kernel(__half* __restrict__ out, const __half* __restrict__ in, size_t n, bool fast) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const __half x = in[i];
    __half t;
    if (!fast) {  // activation_kernels.cu:166-170, every T expression rounded to fp16
      const float x3 = __half2float(__hmul(__hmul(x, x), x));
      const __half inner = __float2half_rn(__fmul_rn(0.044715f, x3));
      const __half arg = __float2half_rn(__fmul_rn(0.79788456f, __half2float(__hadd(x, inner))));
      t = __float2half_rn(tanhf(__half2float(arg)));
    } else {  // :172-178
      const float f = __half2float(x);
      const __half a = __float2half_rn(__fmul_rn(f, 0.79788456f));
      const __half b = __hadd(__float2half_rn(1.0f), __hmul(__float2half_rn(__fmul_rn(0.044715f, f)), x));
      t = __float2half_rn(tanhf(__half2float(__hmul(a, b))));
    }
    out[i] = __hmul(__hmul(__float2half_rn(0.5f), x), __hadd(__float2half_rn(1.0f), t));
  }
}

__global__ void dequant_add_residual_kernel(__half* __restrict__ out, const int32_t* __restrict__ in, const __half* __restrict__ residual,
                                            const __half* __restrict__ scale_vec, float scale, int H) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const float sc = scale_vec ? __half2float(scale_vec[row]) : scale;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const size_t o = static_cast<size_t>(row) * H + i;
    out[o] = __float2half_rn(__fadd_rn(__fmul_rn(__int2float_rn(in[o]), sc), __half2float(residual[o])));
  }
}

__global__ void dequant_kernel(__half* __restrict__ out, const int32_t* __restrict__ in, float scale, int H, int in_stride, int out_stride) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  for (int i = threadIdx.x; i < H; i += blockDim.x)
    out[static_cast<size_t>(row) * out_stride + i] = __float2half_rn(__fmul_rn(__int2float_rn(in[static_cast<size_t>(row) * in_stride + i]), scale));
}

__global__ void __launch_bounds__(kThreads) dequant_add_residual_rms_norm_quant_kernel(int8_t* __restrict__ out, const int32_t* __restrict__ in,
                                                                                      __half* __restrict__ residual, const __half* __restrict__ gamma,
                                                                                      const __half* __restrict__ scale_vec, float scale, float eps, int H) {
  __shared__ float red[32];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const float sc = scale_vec ? __half2float(scale_vec[row]) : scale;
  float vs = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const size_t o = static_cast<size_t>(row) * H + i;
    const float d = __fadd_rn(__fmul_rn(__int2float_rn(in[o]), sc), __half2float(residual[o]));
    residual[o] = __float2half_rn(d);
    vs += d * d;
  }
  const float var = block_reduce(vs, red, OpSum(), 0.f);
  const float rstd = __frsqrt_rn(__fadd_rn(__fdiv_rn(var, static_cast<float>(H)), eps));
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const size_t o = static_cast<size_t>(row) * H + i;
    out[o] = cvt_s8(__fmul_rn(__fmul_rn(__half2float(residual[o]), rstd), __half2float(gamma[i])));
  }
}

__global__ void __launch_bounds__(kThreads) dequant_silu_and_mul_quant_kernel(int8_t* __restrict__ out, const int32_t* __restrict__ in, int d,
                                                                             float scale_gate, float scale_up, float scale_out,
                                                                             float* __restrict__ scale_out_vec, float* __restrict__ tmp) {
  __shared__ float red[32];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const int32_t* g = in + static_cast<size_t>(row) * 2 * d;
  if (scale_out_vec == nullptr) {
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
      const float x = __fmul_rn(__int2float_rn(g[i]), scale_gate), y = __fmul_rn(__int2float_rn(g[d + i]), scale_up);
      const float s = __fdiv_rn(x, __fadd_rn(1.0f, expf(-x)));
      out[static_cast<size_t>(row) * d + i] = cvt_s8(__fdiv_rn(__fmul_rn(s, y), scale_out));
    }
    return;
  }
  float amax = 0.f;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    const float x = __fmul_rn(__int2float_rn(g[i]), scale_gate), y = __fmul_rn(__int2float_rn(g[d + i]), scale_up);
    const float t = __fmul_rn(__fdiv_rn(x, __fadd_rn(1.0f, expf(-x))), y);
    tmp[static_cast<size_t>(row) * d + i] = t;
    amax = fmaxf(amax, fabsf(t));
  }
  amax = block_reduce(amax, red, OpMax(), 0.f);
  if (threadIdx.x == 0) scale_out_vec[row] = __fdiv_rn(amax, 127.f);
  const float qs_ = __fdiv_rn(127.f, amax);
  for (int i = threadIdx.x; i < d; i += blockDim.x)
    out[static_cast<size_t>(row) * d + i] = cvt_s8(__fmul_rn(qs_, tmp[static_cast<size_t>(row) * d + i]));
}

// ---------------------------------------------------------------------------------------------
// greedy sampling: argmax over the vocabulary of fp16 logits [rows, V] (the reference samples with torch.argmax).
// A cluster of 8 CTAs per row: each scans V/8 logits with 128-bit loads, the (value, index) pairs are combined through
// distributed shared memory.  First maximal index wins, NaN counts as the maximum (torch semantics).
// ---------------------------------------------------------------------------------------------
constexpr int kArgmaxCluster = 8;
__global__ void __launch_bounds__(kThreads) argmax_rows_kernel(long long* __restrict__ out, const __half* __restrict__ logits, int V) {
  __shared__ float s_v[kThreads / 32];
  __shared__ int s_i[kThreads / 32];
  __shared__ __align__(8) int2 s_part;  // (float bits, index) of this CTA
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x / kArgmaxCluster, part = blockIdx.x % kArgmaxCluster;
  const __half* src = logits + static_cast<size_t>(row) * V;
  const int nvec = V / 8;  // V % 8 == 0 (checked on the host)
  const int v0 = static_cast<int>((static_cast<long long>(nvec) * part) / kArgmaxCluster);
  const int v1 = static_cast<int>((static_cast<long long>(nvec) * (part + 1)) / kArgmaxCluster);
  float best = __int_as_float(0xff800000);  // -inf
  int bi = 0x7fffffff;
  for (int i = v0 + threadIdx.x; i < v1; i += blockDim.x) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + i);
    const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = __half2float(h[j]);
      if (argmax_better(f, i * 8 + j, best, bi)) { best = f; bi = i * 8 + j; }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, m);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, m);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = best; s_i[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w)
      if (argmax_better(s_v[w], s_i[w], best, bi)) { best = s_v[w]; bi = s_i[w]; }
    s_part = make_int2(__float_as_int(best), bi);
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  if (part == 0 && threadIdx.x == 0) {
    const uint32_t base = static_cast<uint32_t>(__cvta_generic_to_shared(&s_part));
    for (int r = 1; r < kArgmaxCluster; ++r) {
      uint32_t peer;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer) : "r"(base), "r"(r));
      int pv, pi;
      asm volatile("ld.shared::cluster.v2.s32 {%0, %1}, [%2];" : "=r"(pv), "=r"(pi) : "r"(peer) : "memory");
      if (argmax_better(__int_as_float(pv), pi, best, bi)) { best = __int_as_float(pv); bi = pi; }
    }
    out[row] = bi;
  }
  asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");  // peers' smem stays valid
}

// ------------------------------------------------------------------------------------------------
// Register-resident fast path of N1 and of its fused forms (per-token quantisation, H <= 8 * kThreads * CH, CH <= 2: every model of the
// benchmark).  ONE body serves rms_norm_general[_fuse_sum], add_rms_norm_general and its peer (fused all-reduce) form, so the fused and the
// unfused ops are bit-identical by construction.  Against the shared-memory kernels above it keeps the row in registers (no re-reads) and needs
// 4 block barriers instead of 9: a decode-size row op is a pure latency chain, every barrier and round trip counts.
// Arithmetic and reduction trees are those of layernorm_quant_kernel (same thread -> element map, same shuffle order).
// ------------------------------------------------------------------------------------------------
template <typename Op>
__device__ __forceinline__ float block_reduce_1sync(float v, float* buf, Op op, float identity) {
  // `buf` must not be the buffer of the immediately preceding call (the callers alternate two buffers): then one barrier suffices
  v = warp_reduce(v, op);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) buf[w] = v;
  __syncthreads();
  float r = (l < (blockDim.x >> 5)) ? buf[l] : identity;
  return warp_reduce(r, op);
}

template <bool ADD, bool PEER, int CH>
__global__ void __launch_bounds__(kThreads) norm_quant_fast_kernel(int8_t* __restrict__ out, __half* __restrict__ hidden_out, const __half* __restrict__ x,
                                                                  const __half* __restrict__ delta, const __half* __restrict__ gamma,
                                                                  __half* __restrict__ input_sum, __half* __restrict__ scaling, float eps, int H,
                                                                  int ref_block, const PeerArgs peer) {
  extern __shared__ __align__(16) uint8_t sm[];
  __half* sy = reinterpret_cast<__half*>(sm);  // half(y) row, only for the fused sum
  __shared__ float red[2][32];
  __shared__ long long red_ll[32];
  const int row = blockIdx.x;
  const int nvec = H / 8;
  qs_trace(ADD ? QS_K_ADDNORM : QS_K_NORM, 0);
  if (threadIdx.x == 0) pdl_launch_dependents();
  uint4 g[CH];  // gamma is a static weight: fetched before waiting for the producer of x / delta
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    g[c] = (i < nvec) ? __ldg(reinterpret_cast<const uint4*>(gamma) + i) : make_uint4(0u, 0u, 0u, 0u);
  }
  pdl_wait();
  qs_trace(ADD ? QS_K_ADDNORM : QS_K_NORM, 1);
  uint32_t epoch = 0;
  if constexpr (PEER) {
    epoch = *reinterpret_cast<volatile uint32_t*>(peer.state + peer.phase) + 1u;
    if (blockIdx.x == 0 && threadIdx.x < peer.world) st_release_sys(peer.flags[threadIdx.x] + peer.phase * 8 + peer.rank, epoch);
    if (threadIdx.x < peer.world) {
      const uint32_t* mine = peer.flags[peer.rank] + peer.phase * 8 + threadIdx.x;
      unsigned spins = 0;
      while (static_cast<int32_t>(ld_acquire_sys(mine) - epoch) < 0) {
        __nanosleep(40);
        if (++spins > (1u << 27)) {
          printf("qserve_b200: peer all-reduce timed out (rank %d waits for rank %d, phase %d, epoch %u)\n", peer.rank, threadIdx.x, peer.phase, epoch);
          __trap();
        }
      }
    }
    __syncthreads();
  }
  // ---- the row: this thread's chunks i = tid, tid + 512 (8 halves each), kept as packed fp16 in registers ----
  uint4 xv[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    xv[c] = make_uint4(0u, 0u, 0u, 0u);
    if (i < nvec) {
      const uint4 va = __ldg(reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * H) + i);
      if constexpr (ADD) {
        uint4 vb;
        if constexpr (PEER) {
          uint4 pv[8];
#pragma unroll
          for (int r = 0; r < 8; ++r)
            if (r < peer.world) pv[r] = ld_peer_v4(reinterpret_cast<const uint4*>(peer.delta[r] + static_cast<size_t>(row) * H) + i);
          float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            if (r < peer.world) {
              const __half2* hp = reinterpret_cast<const __half2*>(&pv[r]);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(hp[j]);
                acc[2 * j] = __fadd_rn(acc[2 * j], f.x);
                acc[2 * j + 1] = __fadd_rn(acc[2 * j + 1], f.y);
              }
            }
          }
          __half2* hb2 = reinterpret_cast<__half2*>(&vb);
#pragma unroll
          for (int j = 0; j < 4; ++j) hb2[j] = __floats2half2_rn(acc[2 * j], acc[2 * j + 1]);
        } else {
          vb = __ldg(reinterpret_cast<const uint4*>(delta + static_cast<size_t>(row) * H) + i);
        }
        uint4 vo;
        const __half2* ha = reinterpret_cast<const __half2*>(&va);
        const __half2* hb = reinterpret_cast<const __half2*>(&vb);
        __half2* ho2 = reinterpret_cast<__half2*>(&vo);
#pragma unroll
        for (int j = 0; j < 4; ++j) {  // torch half add: float(a) + float(b), rounded once to fp16
          const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
          ho2[j] = __floats2half2_rn(__fadd_rn(fa.x, fb.x), __fadd_rn(fa.y, fb.y));
        }
        xv[c] = vo;
        reinterpret_cast<uint4*>(hidden_out + static_cast<size_t>(row) * H)[i] = vo;
      } else {
        xv[c] = va;
      }
    }
  }
  // ---- mean, variance (two passes over registers; same per-thread order and reduction tree as the shared-memory kernels) ----
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (threadIdx.x + c * kThreads < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&xv[c]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        s += f.x + f.y;
      }
    }
  }
  const float mean = __fdiv_rn(block_reduce_1sync(s, red[0], OpSum(), 0.f), static_cast<float>(H));
  float vs = 0.f;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (threadIdx.x + c * kThreads < nvec) {
      const __half2* h = reinterpret_cast<const __half2*>(&xv[c]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        const float a = f.x - mean, b = f.y - mean;
        vs += a * a + b * b;
      }
    }
  }
  const float var = block_reduce_1sync(vs, red[1], OpSum(), 0.f);
  const float rstd = __frsqrt_rn(__fadd_rn(__fdiv_rn(var, static_cast<float>(H)), eps));
  // ---- y, amax of half(y) (init 1e-6 in fp16), optional half(y) row for the reference-ordered fp16 sum ----
  float amax = __half2float(__float2half_rn(1e-6f));
  float y[CH][8];
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    if (i < nvec) {
      const __half* h = reinterpret_cast<const __half*>(&xv[c]);
      const __half* gh = reinterpret_cast<const __half*>(&g[c]);
      uint4 yv;
      __half* yh = reinterpret_cast<__half*>(&yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        y[c][j] = __fmul_rn(__fmul_rn(__fsub_rn(__half2float(h[j]), mean), rstd), __half2float(gh[j]));
        yh[j] = __float2half_rn(y[c][j]);
        amax = fmaxf(amax, fabsf(__half2float(yh[j])));
      }
      if (input_sum) reinterpret_cast<uint4*>(sy)[i] = yv;
    }
  }
  amax = block_reduce_1sync(amax, red[0], OpMax(), 0.f);  // its barrier also publishes sy
  if (input_sum) {
    // reference thread t (of ref_block threads) accumulates y_h[t], y_h[t+B], ... sequentially IN FP16 (layernorm_kernels.cu:275,286)
    long long part = 0;
    for (int t = threadIdx.x; t < ref_block; t += kThreads) {
      __half acc = __float2half_rn(0.f);
      for (int i = t; i < H; i += ref_block) acc = __hadd(acc, sy[i]);
      part += fx_of_half(__half2float(acc));
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) part += __shfl_xor_sync(0xffffffffu, part, m);
    if ((threadIdx.x & 31) == 0) red_ll[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x < 32) {
      long long r = (threadIdx.x < (kThreads >> 5)) ? red_ll[threadIdx.x] : 0ll;
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) r += __shfl_xor_sync(0xffffffffu, r, m);
      if (threadIdx.x == 0) input_sum[row] = __float2half_rn(fx_to_float(r));
    }
  }
  if (threadIdx.x == 0) scaling[row] = __float2half_rn(__fdiv_rn(amax, 127.f));
  const float qs_ = __fdiv_rn(127.f, amax);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int i = threadIdx.x + c * kThreads;
    if (i < nvec) store_q8(out + static_cast<size_t>(row) * H, i, y[c], qs_);  // quantises the UN-rounded fp32 y (:307-318)
  }
  if constexpr (PEER) {
    if (threadIdx.x == 0) {
      const uint32_t old = atomicAdd(peer.state + 2 + peer.phase, 1u);
      if (old == gridDim.x - 1) {
        peer.state[2 + peer.phase] = 0u;
        *reinterpret_cast<volatile uint32_t*>(peer.state + peer.phase) = epoch;
      }
    }
  }
}

template <typename Kern>
int ensure_smem(Kern kern, size_t bytes, const char* what) {
  if (bytes <= 40 * 1024) return QS_OK;  // static shared memory of the kernel comes on top of the dynamic row
  QS_REQUIRE(bytes <= 200 * 1024, "%s: row of %zu bytes does not fit in shared memory", what, bytes);
  return raise_smem_limit(kern, 200 * 1024, what);
}

// fast path of the norm family: returns 1 if the shape is not eligible (caller falls back to the shared-memory kernels)
template <bool ADD, bool PEER>
int launch_norm_fast(void* out_q, void* hidden_out, const void* x, const void* delta, const void* gamma, void* input_sum, void* scaling, float eps,
                     int tokens, int hidden, const PeerArgs& pa, void* stream, const char* what) {
  const int nvec = hidden / 8;
  if (nvec > 2 * kThreads) return 1;
  int ref_block = hidden < 1024 ? hidden : 1024;
  ref_block = 32 * ((ref_block + 31) / 32);  // layernorm_kernels.cu:433-436
  const size_t smem = input_sum ? static_cast<size_t>(hidden) * 2 : 0;
  auto go = [&](auto kern) {
    return launch(kern, dim3(tokens), dim3(kThreads), smem, 0, stream, what, static_cast<int8_t*>(out_q), static_cast<__half*>(hidden_out),
                  static_cast<const __half*>(x), static_cast<const __half*>(delta), static_cast<const __half*>(gamma), static_cast<__half*>(input_sum),
                  static_cast<__half*>(scaling), eps, hidden, ref_block, pa);
  };
  return nvec <= kThreads ? go(norm_quant_fast_kernel<ADD, PEER, 1>) : go(norm_quant_fast_kernel<ADD, PEER, 2>);
}

}  // namespace

int elementwise_trace_install(void* buf, unsigned cap) { return qs_trace_install(buf, cap); }

int rms_norm(void* out, const void* in, const void* weight, float eps, int use_quant, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "rms_norm: hidden=%d must be a positive multiple of 8", hidden);
  const size_t smem = static_cast<size_t>(hidden) * 2;
  int rc = ensure_smem(rms_norm_kernel, smem, "rms_norm");
  if (rc) return rc;
  return launch(rms_norm_kernel, dim3(tokens), dim3(kThreads), smem, 0, stream, "rms_norm", out, static_cast<const __half*>(in),
                static_cast<const __half*>(weight), eps, hidden, use_quant != 0);
}

int layernorm_general_quant(void* out_q, const void* in, const void* gamma, void* input_sum, void* scaling, float eps, int tokens, int hidden,
                            int per_token, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "rms_norm_general: hidden=%d must be a positive multiple of 8", hidden);
  QS_REQUIRE(per_token || input_sum == nullptr, "rms_norm_general_fuse_sum: per-tensor scaling with input_sum is not implemented by the reference either (layernorm_kernels.cu:490-494)");
  if (per_token) {
    const int fast = launch_norm_fast<false, false>(out_q, nullptr, in, nullptr, gamma, input_sum, scaling, eps, tokens, hidden, PeerArgs{}, stream, "rms_norm_general");
    if (fast != 1) return fast;
  }
  const size_t smem = static_cast<size_t>(hidden) * 2 * (input_sum ? 2 : 1);
  int rc = ensure_smem(layernorm_quant_kernel, smem, "rms_norm_general");
  if (rc) return rc;
  int ref_block = hidden < 1024 ? hidden : 1024;
  ref_block = 32 * ((ref_block + 31) / 32);  // layernorm_kernels.cu:433-436
  return launch(layernorm_quant_kernel, dim3(tokens), dim3(kThreads), smem, 0, stream, "rms_norm_general", static_cast<int8_t*>(out_q),
                static_cast<const __half*>(in), static_cast<const __half*>(gamma), static_cast<__half*>(input_sum),
                static_cast<__half*>(scaling), eps, hidden, ref_block, per_token != 0);
}

int quant_per_token(void* out_q, const void* in, void* input_sum, void* scale, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "invoke_quant: hidden=%d must be a positive multiple of 8", hidden);
  {
    const int nvec = hidden / 8;
    auto go = [&](auto kern) {
      return launch(kern, dim3(tokens), dim3(kThreads), 0, 0, stream, "invoke_quant", static_cast<int8_t*>(out_q), static_cast<const __half*>(in),
                    static_cast<__half*>(input_sum), static_cast<__half*>(scale), hidden);
    };
    if (nvec <= kThreads) return go(quant_per_token_fast_kernel<1>);
    if (nvec <= 2 * kThreads) return go(quant_per_token_fast_kernel<2>);
    if (nvec <= 4 * kThreads) return go(quant_per_token_fast_kernel<4>);
  }
  const size_t smem = static_cast<size_t>(hidden) * 2;
  int rc = ensure_smem(quant_per_token_kernel, smem, "invoke_quant");
  if (rc) return rc;
  return launch(quant_per_token_kernel, dim3(tokens), dim3(kThreads), smem, 0, stream, "invoke_quant", static_cast<int8_t*>(out_q),
                static_cast<const __half*>(in), static_cast<__half*>(input_sum), static_cast<__half*>(scale), hidden);
}

int row_absmax(void* amax_f32, const void* in, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "row_absmax: hidden=%d must be a positive multiple of 8", hidden);
  return launch(row_absmax_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "row_absmax", static_cast<float*>(amax_f32), static_cast<const __half*>(in), hidden);
}

int quant_given_amax(void* out_q, const void* in, const void* amax_f32, void* input_sum, void* scale, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "quant_given_amax: hidden=%d must be a positive multiple of 8", hidden);
  return launch(quant_given_amax_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "quant_given_amax", static_cast<int8_t*>(out_q),
                static_cast<const __half*>(in), static_cast<const float*>(amax_f32), static_cast<__half*>(input_sum), static_cast<__half*>(scale), hidden);
}

int quant_scalar(void* out_q, const void* in, float scale, int tokens, int hidden, void* stream) {
  const size_t n = static_cast<size_t>(tokens) * hidden;
  if (n == 0) return QS_OK;
  const int grid = static_cast<int>((n + 1023) / 1024 < 2048 ? (n + 1023) / 1024 : 2048);
  return launch(quant_scalar_kernel, dim3(grid), dim3(256), 0, 0, stream, "invoke_quant(scalar)", static_cast<int8_t*>(out_q),
                static_cast<const __half*>(in), scale, n);
}

int silu_and_mul(void* out, const void* in, int tokens, int d, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(d > 0 && d % 8 == 0, "silu_and_mul: d=%d must be a positive multiple of 8", d);
  const long long n_vec = static_cast<long long>(tokens) * (d / 8);
  const long long want = (n_vec + 255) / 256;  // one vector per thread up to 8 CTAs per SM (decode sizes), then two per thread and loop iteration
  const long long cap = static_cast<long long>(num_sms()) * 8;
  return launch(silu_and_mul_kernel, dim3(static_cast<unsigned>(want < cap ? want : cap)), dim3(256), 0, 0, stream, "silu_and_mul", static_cast<__half*>(out),
                static_cast<const __half*>(in), d, n_vec);
}

int gelu(void* out, const void* in, int tokens, int d, int fast, void* stream) {
  const size_t n = static_cast<size_t>(tokens) * d;
  if (n == 0) return QS_OK;
  const int grid = static_cast<int>((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  return launch(gelu_kernel, dim3(grid), dim3(256), 0, 0, stream, "gelu", static_cast<__half*>(out), static_cast<const __half*>(in), n, fast != 0);
}

int dequant_add_residual(void* out, const void* in_i32, const void* residual, const void* scale_vec, float scale, int tokens, int hidden,
                         void* stream) {
  if (tokens == 0) return QS_OK;
  return launch(dequant_add_residual_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "invoke_dequant_add_residual", static_cast<__half*>(out),
                static_cast<const int32_t*>(in_i32), static_cast<const __half*>(residual), static_cast<const __half*>(scale_vec), scale, hidden);
}

int dequant(void* out, const void* in_i32, float scale, int tokens, int hidden, int in_stride, int out_stride, void* stream) {
  if (tokens == 0) return QS_OK;
  return launch(dequant_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "invoke_dequant", static_cast<__half*>(out),
                static_cast<const int32_t*>(in_i32), scale, hidden, in_stride, out_stride);
}

int dequant_add_residual_rms_norm_quant(void* out_q, const void* in_i32, void* residual, const void* gamma, const void* scale_vec, float scale,
                                        float eps, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  return launch(dequant_add_residual_rms_norm_quant_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "invoke_dequant_add_residual_rms_norm_quant",
                static_cast<int8_t*>(out_q), static_cast<const int32_t*>(in_i32), static_cast<__half*>(residual),
                static_cast<const __half*>(gamma), static_cast<const __half*>(scale_vec), scale, eps, hidden);
}

int dequant_silu_and_mul_quant(void* out_q, const void* in_i32, float scale_gate, float scale_up, float scale_out, void* scale_out_vec, void* tmp,
                               int tokens, int d, void* stream) {
  if (tokens == 0) return QS_OK;
  return launch(dequant_silu_and_mul_quant_kernel, dim3(tokens), dim3(kThreads), 0, 0, stream, "invoke_dequant_silu_and_mul_quant",
                static_cast<int8_t*>(out_q), static_cast<const int32_t*>(in_i32), d, scale_gate, scale_up, scale_out,
                static_cast<float*>(scale_out_vec), static_cast<float*>(tmp));
}

int silu_and_mul_quant(void* out_q, const void* in, void* input_sum, void* scale, int tokens, int d, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(d > 0 && d % 8 == 0, "silu_and_mul_quant: d=%d must be a positive multiple of 8", d);
  // split a row over a cluster so that tokens * csize CTAs fill the machine (each CTA keeps >= 512 columns)
  int csize = 1;
  while (csize < 8 && tokens * csize < 2 * num_sms() && d % (csize * 2 * 8) == 0 && d / (csize * 2) >= 512) csize *= 2;
  const int nvec = d / csize / 8;
  const bool fast = nvec <= 2 * kSiluQuantThreads;  // register-resident kernel (no dynamic shared memory)
  const size_t smem = fast ? 0 : static_cast<size_t>(d / csize) * 2;
  if (!fast) {
    int rc = ensure_smem(silu_mul_quant_kernel, smem, "silu_and_mul_quant");
    if (rc) return rc;
  }
  auto kern = !fast ? silu_mul_quant_kernel : (nvec <= kSiluQuantThreads ? silu_mul_quant_fast_kernel<1> : silu_mul_quant_fast_kernel<2>);
  return launch(kern, dim3(tokens * csize), dim3(kSiluQuantThreads), smem, csize, stream, "silu_and_mul_quant", static_cast<int8_t*>(out_q),
                static_cast<const __half*>(in), static_cast<__half*>(input_sum), static_cast<__half*>(scale), d, csize);
}

int add_layernorm_quant(void* out_q, void* hidden_out, const void* x, const void* delta, const void* gamma, void* input_sum, void* scaling,
                        float eps, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "add_rms_norm_general: hidden=%d must be a positive multiple of 8", hidden);
  {
    const int fast = launch_norm_fast<true, false>(out_q, hidden_out, x, delta, gamma, input_sum, scaling, eps, tokens, hidden, PeerArgs{}, stream, "add_rms_norm_general");
    if (fast != 1) return fast;
  }
  const size_t smem = static_cast<size_t>(hidden) * 2 * (input_sum ? 2 : 1);
  int rc = ensure_smem(add_layernorm_quant_kernel<false>, smem, "add_rms_norm_general");
  if (rc) return rc;
  int ref_block = hidden < 1024 ? hidden : 1024;
  ref_block = 32 * ((ref_block + 31) / 32);
  return launch(add_layernorm_quant_kernel<false>, dim3(tokens), dim3(kFusedThreads), smem, 0, stream, "add_rms_norm_general", static_cast<int8_t*>(out_q),
                static_cast<__half*>(hidden_out), static_cast<const __half*>(x), static_cast<const __half*>(delta),
                static_cast<const __half*>(gamma), static_cast<__half*>(input_sum), static_cast<__half*>(scaling), eps, hidden, ref_block, PeerArgs{});
}

int add_layernorm_quant_peer(void* out_q, void* hidden_out, const void* x, const void* const* delta_ptrs, void* const* flag_ptrs, void* state, int world,
                             int rank, int phase, const void* gamma, void* input_sum, void* scaling, float eps, int tokens, int hidden, void* stream) {
  if (tokens == 0) return QS_OK;
  QS_REQUIRE(hidden > 0 && hidden % 8 == 0, "add_rms_norm_general_peer: hidden=%d must be a positive multiple of 8", hidden);
  QS_REQUIRE(world >= 1 && world <= 8 && rank >= 0 && rank < world && (phase == 0 || phase == 1), "add_rms_norm_general_peer: world=%d rank=%d phase=%d", world, rank, phase);
  PeerArgs pa{};
  for (int r = 0; r < world; ++r) {
    QS_REQUIRE(delta_ptrs[r] && flag_ptrs[r] && (reinterpret_cast<uintptr_t>(delta_ptrs[r]) & 15) == 0, "add_rms_norm_general_peer: bad peer pointer of rank %d", r);
    pa.delta[r] = static_cast<const __half*>(delta_ptrs[r]);
    pa.flags[r] = static_cast<uint32_t*>(flag_ptrs[r]);
  }
  pa.state = static_cast<uint32_t*>(state);
  pa.world = world; pa.rank = rank; pa.phase = phase;
  {
    const int fast = launch_norm_fast<true, true>(out_q, hidden_out, x, nullptr, gamma, input_sum, scaling, eps, tokens, hidden, pa, stream, "add_rms_norm_general_peer");
    if (fast != 1) return fast;
  }
  const size_t smem = static_cast<size_t>(hidden) * 2 * (input_sum ? 2 : 1);
  int rc = ensure_smem(add_layernorm_quant_kernel<true>, smem, "add_rms_norm_general_peer");
  if (rc) return rc;
  int ref_block = hidden < 1024 ? hidden : 1024;
  ref_block = 32 * ((ref_block + 31) / 32);
  return launch(add_layernorm_quant_kernel<true>, dim3(tokens), dim3(kFusedThreads), smem, 0, stream, "add_rms_norm_general_peer", static_cast<int8_t*>(out_q),
                static_cast<__half*>(hidden_out), static_cast<const __half*>(x), static_cast<const __half*>(nullptr),
                static_cast<const __half*>(gamma), static_cast<__half*>(input_sum), static_cast<__half*>(scaling), eps, hidden, ref_block, pa);
}

int argmax_rows(void* out, const void* logits, int rows, int vocab, void* stream) {
  if (rows == 0) return QS_OK;
  QS_REQUIRE(vocab > 0 && vocab % 8 == 0, "argmax_rows: vocab=%d must be a positive multiple of 8", vocab);
  return launch(argmax_rows_kernel, dim3(rows * kArgmaxCluster), dim3(kThreads), 0, kArgmaxCluster, stream, "argmax_rows", static_cast<long long*>(out),
                static_cast<const __half*>(logits), vocab);
}

}  // namespace qs
