// qserve_b200 -- temperature / top-p / top-k sampling of fp16 logits and lossless sampled acceptance of draft trees, sm_90a.
//
// sample_rows_kernel: one token per row of fp16 logits [rows, V].  One cluster of 8 CTAs per row (the argmax_rows pattern); each CTA copies
// its V / 8 slice into shared memory once and every later pass reads it there.
//   * greedy rows (T < 1e-5 or top_p < 1e-8) and rows without a finite logit return what argmax_rows returns;
//   * otherwise z = x / T (IEEE fp32), w = exp(z - max z), NaN and -inf logits have weight 0.  The kept set is {key >= max(tau_p, tau_k)}
//     on the order-preserving 16-bit key of the fp16 logit: tau_k is the k-th largest key (radix select: a 256-bin count histogram of the
//     high byte, then of the low byte inside the selected bin, summed through distributed shared memory), tau_p the smallest key whose
//     strictly-larger weight is < top_p * sum w (the same two-level histogram over weights, restricted to keys >= tau_k);
//   * the token is drawn by inverse CDF in index order: an ordered prefix of the per-CTA kept sums selects the CTA that holds u * S, and
//     a block scan over contiguous per-thread ranges selects the token inside it.
// Every weight sum is accumulated in 64-bit fixed point (40 fractional bits, w <= 1): integer addition is associative, so histograms built
// with shared-memory atomics are exact and a call is bitwise deterministic.  Quantising each weight to 2^-41 moves a CDF by at most
// V * 2^-41 <= 1e-7 of the largest weight, far below the fp32 exp error the tests allow for.
//
// Random numbers: Philox4x32-10, counter (lo(off), hi(off), row, j), key (lo(seed), hi(seed)), u = (x0 >> 8) * 2^-24; off = offsets[row],
// which the call advances by one.  Counter-based and per row: a CUDA-graph replay draws fresh numbers and no cross-CTA atomics are needed.
//
// tree_accept_sampling_kernel: the sampled counterpart of tree_accept_greedy (SpecInfer multi-step speculative sampling; Leviathan / Chen
// rejection sampling for a chain).  One cluster per sequence keeps the current target distribution p (unnormalised fp32, one V / 8 slice per
// CTA) in shared memory.  At each node the children are tried in index order: child c with token d is accepted iff u_c * q_c(d) < p(d)
// (u_c: draw j = c); on rejection p <- max(p - q_c, 0) (one pass over p and q_c plus a cluster reduction; for one-hot q_c only p(d) is
// zeroed).  With no child accepted the bonus token is drawn from p with draw j = 0.  Greedy rows keep p one-hot at the argmax, which makes
// the result exactly tree_accept_greedy(draft, mask, argmax_rows(logits)).
//
// apply_penalties_kernel: repetition / presence / frequency penalties on the logits before the sampler, one CTA per row over its history
// only (sorted keys, one writer per distinct token).  apply_penalties_tree_kernel: the same penalties on every node row of a draft tree, each
// node's history extended by its path (the history sorted once per sequence).  logprobs_rows_kernel: the log-probability of a chosen token
// and the top-n tokens of the T = 1 softmax, on the sample_rows cluster structure (fixed-point sums, radix select of the n-th largest key).
// logprobs_accepted_kernel: the same arithmetic for the tokens a speculative step emits, written at their history columns.
//
// All kernels read everything a preceding kernel may write (logits, drafts, mask, history, parameters, offsets) after griddepcontrol.wait,
// need no host synchronisation and can be captured in a CUDA graph.
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

using u64 = unsigned long long;

constexpr int kCluster = 8;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxVocab = 196608;  // 24576 logits per CTA: 48 KB of fp16 (+ 96 KB of fp32 p in the tree kernel)
constexpr int kMaxNodes = 16;
constexpr float kFix = 1099511627776.f;  // 2^40: fixed-point scale of the weight sums

// ------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
template <typename T>
__device__ __forceinline__ T* peer(T* p, int rank) {  // the same shared-memory variable in CTA `rank` of the cluster (generic address)
  uint64_t out;
  asm volatile("mapa.u64 %0, %1, %2;" : "=l"(out) : "l"(reinterpret_cast<uint64_t>(p)), "r"(rank));
  return reinterpret_cast<T*>(out);
}

// Philox4x32-10, first output word
__device__ __forceinline__ uint32_t philox_x0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}
// u in [0, 1 - 2^-24], exact in fp32
__device__ __forceinline__ float uniform(u64 seed, long long off, int row, int j) {
  const u64 o = static_cast<u64>(off);
  const uint32_t x = philox_x0(static_cast<uint32_t>(o), static_cast<uint32_t>(o >> 32), static_cast<uint32_t>(row), static_cast<uint32_t>(j),
                               static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  return __uint2float_rn(x >> 8) * 5.9604644775390625e-8f;
}

// order-preserving 16-bit key of an fp16 logit, and its inverse
__device__ __forceinline__ uint32_t okey(uint32_t b) { return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u); }
__device__ __forceinline__ uint32_t key_bits(uint32_t k) { return (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu); }
__device__ __forceinline__ bool valid_bits(uint32_t b) { return (b & 0x7fffu) <= 0x7c00u && b != 0xfc00u; }  // neither NaN nor -inf

__device__ __forceinline__ float weight(uint32_t b, float T, float mz) {
  const float z = __fdiv_rn(__half2float(__ushort_as_half(static_cast<unsigned short>(b))), T);
  return z == mz ? 1.f : expf(__fsub_rn(z, mz));
}
__device__ __forceinline__ u64 fix(float w) { return __float2ull_rn(__fmul_rn(w, kFix)); }

struct Smem {
  u64 hist[256];
  u64 red[kWarps];
  u64 part[2];      // this CTA's published value (alternating slots: one cluster barrier per gather)
  int sel;
  u64 sel_above;
  int tok;
  int2 arg[kWarps];
};

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, T* red, Op op) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, m));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = red[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) r = op(r, red[w]);  // fixed order
  __syncthreads();
  return r;
}
struct OpAdd { __device__ u64 operator()(u64 a, u64 b) const { return a + b; } };
struct OpMax { __device__ u64 operator()(u64 a, u64 b) const { return a > b ? a : b; } };

// exclusive prefix over the threads of the block in thread order
__device__ __forceinline__ u64 block_excl_scan(u64 v, u64* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  u64 inc = v;
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {
    const u64 o = __shfl_up_sync(0xffffffffu, inc, m);
    if (lane >= m) inc += o;
  }
  if (lane == 31) red[w] = inc;
  __syncthreads();
  u64 off = 0;
  for (int i = 0; i < w; ++i) off += red[i];
  __syncthreads();
  return off + inc - v;
}

// publish one value per CTA and read all of them, in rank order, in every thread
__device__ __forceinline__ void gather(Smem& s, int& phase, u64 mine, u64 (&all)[kCluster]) {
  if (threadIdx.x == 0) s.part[phase] = mine;
  cluster_sync();
#pragma unroll
  for (int r = 0; r < kCluster; ++r) all[r] = *peer(&s.part[phase], r);
  phase ^= 1;
}

// Sum the 256-bin histograms of the cluster and select a bin, scanning from the top: COUNT: the bin holding the k-th largest key;
// WEIGHT: the lowest non-empty bin whose strictly-higher weight plus `base` is < thr.  Returns the bin and the total above it.
template <bool COUNT>
__device__ __forceinline__ int hist_select(Smem& s, u64 k, u64 base, double thr, u64& above_out) {
  cluster_sync();  // every CTA's histogram is complete
  const int t = threadIdx.x, bin = 255 - t;  // thread order = descending bins
  u64 tot = 0;
#pragma unroll
  for (int r = 0; r < kCluster; ++r) tot += peer(s.hist, r)[bin];
  if (t == 0) s.sel = -1;
  const u64 above = block_excl_scan(tot, s.red);  // has a __syncthreads after the write of s.sel
  bool hit;
  if (COUNT)
    hit = above < k && k <= above + tot;
  else
    hit = tot > 0 && static_cast<double>(base + above) < thr;
  if (hit) atomicMax(&s.sel, t);  // COUNT: exactly one thread; WEIGHT: the hits are a prefix of the threads, take the lowest bin
  __syncthreads();
  if (t == s.sel) s.sel_above = above;
  __syncthreads();
  const int sel = s.sel;
  above_out = s.sel_above;
  cluster_sync();  // the peers are done reading this histogram
  return 255 - sel;
}

__device__ __forceinline__ void zero_hist(Smem& s) {
  s.hist[threadIdx.x] = 0;
  __syncthreads();
}

// argmax_rows over the cluster (the same (value, index) order), result in every thread
__device__ __forceinline__ int cluster_argmax(Smem& s, int& phase, const __half* xs, int n_loc, int g0) {
  float best = __int_as_float(0xff800000);
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < n_loc; i += kThreads) {
    const float f = __half2float(xs[i]);
    if (argmax_better(f, g0 + i, best, bi)) { best = f; bi = g0 + i; }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, m);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, m);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) s.arg[threadIdx.x >> 5] = make_int2(__float_as_int(best), bi);
  __syncthreads();
  best = __int_as_float(s.arg[0].x);
  bi = s.arg[0].y;
  for (int w = 1; w < kWarps; ++w)
    if (argmax_better(__int_as_float(s.arg[w].x), s.arg[w].y, best, bi)) { best = __int_as_float(s.arg[w].x); bi = s.arg[w].y; }
  __syncthreads();
  u64 all[kCluster];
  gather(s, phase, (static_cast<u64>(static_cast<uint32_t>(__float_as_int(best))) << 32) | static_cast<uint32_t>(bi), all);
  best = __int_as_float(static_cast<int>(all[0] >> 32));
  bi = static_cast<int>(all[0] & 0xffffffffu);
#pragma unroll
  for (int r = 1; r < kCluster; ++r) {
    const float v = __int_as_float(static_cast<int>(all[r] >> 32));
    const int i = static_cast<int>(all[r] & 0xffffffffu);
    if (argmax_better(v, i, best, bi)) { best = v; bi = i; }
  }
  return bi;
}

struct Warped {
  bool greedy;   // greedy row or no finite logit: the answer is `argmax`
  int argmax;
  uint32_t tau;  // kept: valid keys >= tau
  float T, mz;   // weights: weight(bits, T, mz)
};

// Steps 1-5 of the sampling contract for the row slice xs[0 .. n_loc) (global index g0 + i); uniform over the cluster.
__device__ __forceinline__ Warped warp_row(Smem& s, int& phase, const __half* xs, int n_loc, int g0, float T, int top_k, float top_p) {
  Warped r;
  r.T = T;
  r.tau = 0;
  r.mz = 0.f;
  r.argmax = 0;
  const uint16_t* xb = reinterpret_cast<const uint16_t*>(xs);
  u64 mk = 0, cnt = 0;
  for (int i = threadIdx.x; i < n_loc; i += kThreads) {
    const uint32_t b = xb[i];
    if (valid_bits(b)) {
      mk = max(mk, static_cast<u64>(okey(b)));
      ++cnt;
    }
  }
  mk = block_reduce(mk, s.red, OpMax());
  cnt = block_reduce(cnt, s.red, OpAdd());
  u64 all[kCluster];
  gather(s, phase, (mk << 40) | cnt, all);
  mk = 0;
  cnt = 0;
#pragma unroll
  for (int q = 0; q < kCluster; ++q) {
    mk = max(mk, all[q] >> 40);
    cnt += all[q] & ((1ull << 40) - 1);
  }
  r.greedy = T < 1e-5f || top_p < 1e-8f || cnt == 0;
  if (r.greedy) {
    r.argmax = cluster_argmax(s, phase, xs, n_loc, g0);
    return r;
  }
  const uint32_t kmax = static_cast<uint32_t>(mk);
  r.mz = __fdiv_rn(__half2float(__ushort_as_half(static_cast<unsigned short>(key_bits(kmax)))), T);
  if (top_k == 1) {
    r.tau = kmax;
  } else if (top_k > 1 && static_cast<u64>(top_k) < cnt) {  // radix select of the k-th largest key
    u64 above;
    zero_hist(s);
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (valid_bits(b)) atomicAdd(&s.hist[okey(b) >> 8], 1ull);
    }
    const int hi = hist_select<true>(s, static_cast<u64>(top_k), 0, 0.0, above);
    zero_hist(s);
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (valid_bits(b) && static_cast<int>(okey(b) >> 8) == hi) atomicAdd(&s.hist[okey(b) & 255u], 1ull);
    }
    const int lo = hist_select<true>(s, static_cast<u64>(top_k) - above, 0, 0.0, above);
    r.tau = static_cast<uint32_t>(hi << 8 | lo);
  }
  if (top_p < 1.f) {  // the two-level histogram of fixed-point weights over the keys >= tau_k; every valid weight counts towards the total
    zero_hist(s);
    u64 tot = 0;
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (valid_bits(b)) {
        const u64 f = fix(weight(b, T, r.mz));
        tot += f;
        const uint32_t k = okey(b);
        if (k >= r.tau && f) atomicAdd(&s.hist[k >> 8], f);
      }
    }
    tot = block_reduce(tot, s.red, OpAdd());
    gather(s, phase, tot, all);
    tot = 0;
#pragma unroll
    for (int q = 0; q < kCluster; ++q) tot += all[q];
    const double thr = static_cast<double>(top_p) * static_cast<double>(tot);
    u64 above_hi, above_lo;
    const int hi = hist_select<false>(s, 0, 0, thr, above_hi);
    zero_hist(s);
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (!valid_bits(b)) continue;
      const uint32_t k = okey(b);
      if (static_cast<int>(k >> 8) == hi && k >= r.tau) {
        const u64 f = fix(weight(b, T, r.mz));
        if (f) atomicAdd(&s.hist[k & 255u], f);
      }
    }
    const int lo = hist_select<false>(s, 0, above_hi, thr, above_lo);
    r.tau = max(r.tau, static_cast<uint32_t>(hi << 8 | lo));
  }
  return r;
}

__device__ __forceinline__ u64 kept_fix(uint32_t b, const Warped& w) {
  return (valid_bits(b) && okey(b) >= w.tau) ? fix(weight(b, w.T, w.mz)) : 0ull;
}

// Step 6: the smallest index t with sum_{j <= t} val(j) > u * S.  `mine` is this CTA's sum of val; returns the token in the CTA that
// holds it and -1 in the others.
template <typename Val>
__device__ __forceinline__ int cluster_draw(Smem& s, int& phase, Val val, int n_loc, int g0, u64 mine, float u, int rank) {
  u64 all[kCluster];
  gather(s, phase, mine, all);
  u64 pre = 0, S = 0;
#pragma unroll
  for (int q = 0; q < kCluster; ++q) {
    if (q < rank) pre += all[q];
    S += all[q];
  }
  const u64 target = static_cast<u64>(static_cast<double>(u) * static_cast<double>(S));  // < S: u <= 1 - 2^-24 and S >= 2^40
  if (!(pre <= target && target < pre + mine)) return -1;  // uniform over the CTA; true in exactly one CTA
  const u64 t = target - pre;
  const int per = (n_loc + kThreads - 1) / kThreads;
  const int i0 = min(static_cast<int>(threadIdx.x) * per, n_loc), i1 = min(i0 + per, n_loc);
  u64 sum = 0;
  for (int i = i0; i < i1; ++i) sum += val(i);
  const u64 ex = block_excl_scan(sum, s.red);
  if (ex <= t && t < ex + sum) {
    u64 c = ex;
    for (int i = i0; i < i1; ++i) {
      c += val(i);
      if (c > t) {
        s.tok = g0 + i;
        break;
      }
    }
  }
  __syncthreads();
  return s.tok;
}

// copy this CTA's slice of an fp16 row into shared memory (128-bit loads)
__device__ __forceinline__ void load_slice(__half* xs, const __half* row, int v0, int v1) {
  const uint4* src = reinterpret_cast<const uint4*>(row) + v0;
  uint4* dst = reinterpret_cast<uint4*>(xs);
  for (int i = threadIdx.x; i < v1 - v0; i += kThreads) dst[i] = __ldg(src + i);
  __syncthreads();
}

__device__ __forceinline__ void slice_of(int V, int rank, int& v0, int& v1) {
  const int nvec = V / 8;  // V % 8 == 0 (checked on the host)
  v0 = static_cast<int>((static_cast<long long>(nvec) * rank) / kCluster);
  v1 = static_cast<int>((static_cast<long long>(nvec) * (rank + 1)) / kCluster);
}

__global__ void __launch_bounds__(kThreads, 1) sample_rows_kernel(long long* __restrict__ out, const __half* __restrict__ logits,
                                                               const float* __restrict__ temperature, const int* __restrict__ top_k,
                                                               const float* __restrict__ top_p, u64 seed, long long* __restrict__ offsets, int V) {
  extern __shared__ uint4 dyn[];
  __shared__ Smem s;
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits, parameters and offsets may come from the preceding kernels
  const int row = blockIdx.x / kCluster, rank = blockIdx.x % kCluster;
  int v0, v1;
  slice_of(V, rank, v0, v1);
  const int n_loc = (v1 - v0) * 8, g0 = v0 * 8;
  __half* xs = reinterpret_cast<__half*>(dyn);
  const long long off = offsets[row];
  const float T = temperature[row], tp = top_p[row];
  const int tk = top_k[row];
  load_slice(xs, logits + static_cast<size_t>(row) * V, v0, v1);
  int phase = 0;
  const Warped w = warp_row(s, phase, xs, n_loc, g0, T, tk, tp);
  if (w.greedy) {
    if (rank == 0 && threadIdx.x == 0) out[row] = w.argmax;
  } else {
    const uint16_t* xb = reinterpret_cast<const uint16_t*>(xs);
    u64 mine = 0;
    for (int i = threadIdx.x; i < n_loc; i += kThreads) mine += kept_fix(xb[i], w);
    mine = block_reduce(mine, s.red, OpAdd());
    const int tok = cluster_draw(s, phase, [&](int i) { return kept_fix(xb[i], w); }, n_loc, g0, mine, uniform(seed, off, row, 0), rank);
    if (tok >= 0 && threadIdx.x == 0) out[row] = tok;
  }
  cluster_sync();  // every CTA has read `off` and is done with its peers' shared memory
  if (rank == 0 && threadIdx.x == 0) offsets[row] = off + 1;
}

__global__ void __launch_bounds__(kThreads, 1) tree_accept_sampling_kernel(
    const long long* __restrict__ draft, const int* __restrict__ tree_mask, const __half* __restrict__ logits, const float* __restrict__ draft_probs,
    const float* __restrict__ temperature, const int* __restrict__ top_k, const float* __restrict__ top_p, u64 seed, long long* __restrict__ offsets,
    int* __restrict__ accept_len, int* __restrict__ path, long long* __restrict__ bonus, int n, int V, int slice_cap) {
  extern __shared__ uint4 dyn[];
  __shared__ Smem s;
  __shared__ long long s_draft[kMaxNodes];
  __shared__ int s_parent[kMaxNodes], s_path[kMaxNodes];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits, drafts, mask, q, parameters and offsets may come from the preceding kernels
  const int b = blockIdx.x / kCluster, rank = blockIdx.x % kCluster;
  int v0, v1;
  slice_of(V, rank, v0, v1);
  const int n_loc = (v1 - v0) * 8, g0 = v0 * 8;
  __half* xs = reinterpret_cast<__half*>(dyn);
  float* ps = reinterpret_cast<float*>(xs + slice_cap);
  const long long off = offsets[b];
  const float T = temperature[b], tp = top_p[b];
  const int tk = top_k[b];
  const size_t row0 = static_cast<size_t>(b) * n;
  if (threadIdx.x < kMaxNodes) {
    const int c = threadIdx.x;
    const uint32_t anc = (c < n && c > 0) ? static_cast<uint32_t>(tree_mask[row0 + c]) & ((1u << c) - 1u) : 0u;
    s_draft[c] = c < n ? draft[row0 + c] : -1;
    s_parent[c] = anc ? 31 - __clz(anc) : -1;  // the root and parentless nodes are never a child
  }
  int phase = 0;
  Warped w;
  u64 mine = 0, S = 0;
  auto enter = [&](int node) {  // p <- warp(logits[b, node])
    load_slice(xs, logits + (row0 + node) * V, v0, v1);
    w = warp_row(s, phase, xs, n_loc, g0, T, tk, tp);
    if (w.greedy) return;
    const uint16_t* xb = reinterpret_cast<const uint16_t*>(xs);
    u64 m = 0;
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t bb = xb[i];
      const float p = (valid_bits(bb) && okey(bb) >= w.tau) ? weight(bb, w.T, w.mz) : 0.f;
      ps[i] = p;
      m += fix(p);
    }
    mine = block_reduce(m, s.red, OpAdd());
    u64 all[kCluster];
    gather(s, phase, mine, all);  // also publishes ps to the peers
    S = 0;
#pragma unroll
    for (int q = 0; q < kCluster; ++q) S += all[q];
  };
  enter(0);
  int cur = 0, len = 1;
  if (threadIdx.x == 0) s_path[0] = 0;
  for (;;) {
    int next = -1;
    for (int c = cur + 1; c < n; ++c) {
      if (s_parent[c] != cur) continue;
      const long long d = s_draft[c];
      if (d < 0 || d >= V) continue;  // padding / out of range: never accepted, p unchanged
      const int di = static_cast<int>(d);
      if (w.greedy) {
        if (di == w.argmax) { next = c; break; }
        continue;
      }
      const float u = uniform(seed, off, b, c);
      const float* qrow = draft_probs ? draft_probs + (row0 + c) * V : nullptr;
      const float qd = qrow ? qrow[di] : 1.f;
      int owner = kCluster - 1, ov0, ov1;
      for (int q = 0; q < kCluster - 1; ++q) {
        slice_of(V, q, ov0, ov1);
        if (di < ov1 * 8) {
          owner = q;
          break;
        }
      }
      slice_of(V, owner, ov0, ov1);
      const float pd = *peer(ps + (di - ov0 * 8), owner);
      // p(d) = pd / (S 2^-40): accept iff u q(d) < p(d)
      if (static_cast<double>(u) * static_cast<double>(qd) * (static_cast<double>(S) * 9.094947017729282e-13) < static_cast<double>(pd)) {
        next = c;
        break;
      }
      cluster_sync();  // every CTA has read pd: p may change
      if (!qrow) {     // one-hot q: p - q only loses p(d)
        if (rank == owner) {
          if (threadIdx.x == 0) ps[di - g0] = 0.f;
          mine -= fix(pd);
        }
        u64 all[kCluster];
        gather(s, phase, mine, all);
        S = 0;
#pragma unroll
    for (int q = 0; q < kCluster; ++q) S += all[q];
      } else {  // p <- max(p / R - q, 0); kept as is when the residual mass is 0
        const float inv = static_cast<float>(1099511627776.0 / static_cast<double>(S));
        const float* qs = qrow + g0;
        u64 m = 0;
        for (int i = threadIdx.x; i < n_loc; i += kThreads) m += fix(fmaxf(__fsub_rn(__fmul_rn(ps[i], inv), __ldg(qs + i)), 0.f));
        m = block_reduce(m, s.red, OpAdd());
        u64 all[kCluster];
        gather(s, phase, m, all);
        u64 M = 0;
#pragma unroll
    for (int q = 0; q < kCluster; ++q) M += all[q];
        if (M > 0) {
          for (int i = threadIdx.x; i < n_loc; i += kThreads) ps[i] = fmaxf(__fsub_rn(__fmul_rn(ps[i], inv), __ldg(qs + i)), 0.f);
          mine = m;
          S = M;
          cluster_sync();  // the new p is visible to the peers
        }
      }
    }
    if (next < 0) break;
    cur = next;
    if (threadIdx.x == 0) s_path[len] = cur;
    ++len;
    cluster_sync();  // the peers are done reading this CTA's p
    enter(cur);
  }
  if (w.greedy) {
    if (rank == 0 && threadIdx.x == 0) bonus[b] = w.argmax;
  } else {
    const int tok = cluster_draw(s, phase, [&](int i) { return fix(ps[i]); }, n_loc, g0, mine, uniform(seed, off, b, 0), rank);
    if (tok >= 0 && threadIdx.x == 0) bonus[b] = tok;
  }
  __syncthreads();
  if (rank == 0 && threadIdx.x < n) path[row0 + threadIdx.x] = static_cast<int>(threadIdx.x) < len ? s_path[threadIdx.x] : -1;
  if (rank == 0 && threadIdx.x == 0) accept_len[b] = len;
  cluster_sync();  // every CTA has read `off` and is done with its peers' shared memory
  if (rank == 0 && threadIdx.x == 0) offsets[b] = off + 1;
}

// ------------------------------------------------------------------------------------------------
// repetition / presence / frequency penalties
// ------------------------------------------------------------------------------------------------
constexpr int kPenThreads = 1024;
constexpr int kMaxHistory = 32768;  // 128 KB of sort keys per row
constexpr uint32_t kNoKey = 0xffffffffu;

// first index in [lo, hi) of the ascending keys with keys[i] >= v
__device__ __forceinline__ int lower_bound(const uint32_t* keys, int lo, int hi, uint32_t v) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The row's history h[0 .. hl) as keys (token << 1) | is_output (position >= pl) in shared memory (padding, out-of-range ids and the tail
// past hl: kNoKey), sorted ascending (bitonic over the next power of two of hl).  Returns that power of two.
__device__ __forceinline__ int sorted_history_keys(uint32_t* keys, const long long* hrow, int hl, int pl, int V) {
  int n = 1;
  while (n < hl) n <<= 1;
  for (int i = threadIdx.x; i < n; i += kPenThreads) {
    uint32_t k = kNoKey;
    if (i < hl) {
      const long long t = hrow[i];
      if (t >= 0 && t < V) k = (static_cast<uint32_t>(t) << 1) | (i >= pl ? 1u : 0u);
    }
    keys[i] = k;
  }
  __syncthreads();
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += kPenThreads) {
        const int p = i ^ j;
        if (p > i) {
          const uint32_t a = keys[i], b = keys[p];
          if ((a > b) == ((i & k) == 0)) {
            keys[i] = b;
            keys[p] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  return n;
}

// the penalties of a token that occurs in the history, c_out times at an output position, on lrow[t]; written only when the bits change
__device__ __forceinline__ void penalise(__half* lrow, uint32_t t, float rep, float pres, float freq, int c_out) {
  const __half old = lrow[t];
  float x = __half2float(old);
  if (x != x) return;  // NaN logits are not written
  if (rep != 1.f) x = x > 0.f ? __fdiv_rn(x, rep) : __fmul_rn(x, rep);
  if (c_out > 0) {
    x = __fsub_rn(x, __fmul_rn(freq, static_cast<float>(c_out)));
    x = __fsub_rn(x, pres);
  }
  const __half nw = __float2half_rn(x);
  if (__half_as_ushort(nw) != __half_as_ushort(old)) lrow[t] = nw;
}

// One CTA per row.  The history becomes sorted keys (sorted_history_keys).  The first key of each run of one token applies the penalties to
// that token's logit: the run's output keys are its upper part, found by binary search.  Every distinct token is written by exactly one
// thread, and only when its fp16 bits change.
__global__ void __launch_bounds__(kPenThreads, 1) apply_penalties_kernel(__half* __restrict__ logits, const long long* __restrict__ history,
                                                                       const int* __restrict__ prompt_lens, const int* __restrict__ seq_lens,
                                                                       const float* __restrict__ repetition, const float* __restrict__ presence,
                                                                       const float* __restrict__ frequency, int V, int H) {
  extern __shared__ uint32_t keys[];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits, history, lengths and parameters may come from the preceding kernels
  const int row = blockIdx.x;
  const float rep = repetition[row], pres = presence[row], freq = frequency[row];
  if (rep == 1.f && pres == 0.f && freq == 0.f) return;  // neutral row: nothing is written
  const int hl = min(max(seq_lens[row], 0), H);
  const int pl = min(max(prompt_lens[row], 0), hl);
  const int n = sorted_history_keys(keys, history + static_cast<size_t>(row) * H, hl, pl, V);
  __half* lrow = logits + static_cast<size_t>(row) * V;
  for (int i = threadIdx.x; i < n; i += kPenThreads) {
    const uint32_t k = keys[i];
    if (k == kNoKey || (i > 0 && (keys[i - 1] >> 1) == (k >> 1))) continue;
    const uint32_t t = k >> 1;
    penalise(lrow, t, rep, pres, freq, lower_bound(keys, i, n, (t + 1) << 1) - lower_bound(keys, i, n, (t << 1) | 1u));
  }
}

// The penalties of every node of a draft tree, one CTA per sequence over its `nodes` verify rows.  Node i's expanded history is the row's
// history h[0 .. hl), then the tokens of its ancestors j >= 1 in index order, then its own token (i >= 1); path position k sits at hl + k
// and is an output position iff hl + k >= prompt_len.  The history is sorted once (sorted_history_keys); the <= 16 node tokens, path words
// and output words are staged beside it.  Pass 1: the first key of each distinct history token applies, for every node, the penalties with
// the history's output count plus that token's output occurrences on the node's path.  Pass 2: for each (node, path node j) whose token is
// absent from the history (binary search) and does not occur earlier on the path, the penalties with its output occurrences on the path.
// Each (node, token) is written by one thread at most, and only when its bits change.
__global__ void __launch_bounds__(kPenThreads, 1) apply_penalties_tree_kernel(__half* __restrict__ logits, const long long* __restrict__ draft,
                                                                            const int* __restrict__ tree_mask, const long long* __restrict__ history,
                                                                            const int* __restrict__ prompt_lens, const int* __restrict__ seq_lens,
                                                                            const float* __restrict__ repetition, const float* __restrict__ presence,
                                                                            const float* __restrict__ frequency, int nodes, int V, int H) {
  extern __shared__ uint32_t keys[];
  __shared__ uint32_t s_tok[kMaxNodes];   // node tokens, kNoKey outside [0, V)
  __shared__ uint32_t s_path[kMaxNodes];  // node i: the nodes whose tokens its expanded history appends
  __shared__ uint32_t s_out[kMaxNodes];   // node i: the path nodes at an output position
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits, drafts, masks, history, lengths and parameters may come from the preceding kernels
  const int b = blockIdx.x;
  const float rep = repetition[b], pres = presence[b], freq = frequency[b];
  if (rep == 1.f && pres == 0.f && freq == 0.f) return;  // neutral row: nothing is written
  const int hl = min(max(seq_lens[b], 0), H);
  const int p0 = max(prompt_lens[b], 0);
  const size_t row0 = static_cast<size_t>(b) * nodes;
  if (threadIdx.x < kMaxNodes) {
    const int i = threadIdx.x;
    uint32_t tok = kNoKey, path = 0, out = 0;
    if (i < nodes) {
      const long long t = draft[row0 + i];
      if (t >= 0 && t < V) tok = static_cast<uint32_t>(t);
      if (i > 0) path = (static_cast<uint32_t>(tree_mask[row0 + i]) & ((1u << i) - 1u) & ~1u) | (1u << i);
      for (uint32_t m = path; m; m &= m - 1) {
        const int j = __ffs(m) - 1;
        if (hl + __popc(path & ((1u << j) - 1u)) >= p0) out |= 1u << j;
      }
    }
    s_tok[i] = tok;
    s_path[i] = path;
    s_out[i] = out;
  }
  // (sorted_history_keys synchronises the block before any key, and so any s_* entry, is read)
  const int n = sorted_history_keys(keys, history + static_cast<size_t>(b) * H, hl, min(p0, hl), V);
  auto same = [&](uint32_t t) {  // the nodes whose token is t
    uint32_t m = 0;
#pragma unroll
    for (int j = 0; j < kMaxNodes; ++j) m |= (s_tok[j] == t ? 1u : 0u) << j;
    return m;
  };
  __half* lb = logits + row0 * V;
  for (int i = threadIdx.x; i < n; i += kPenThreads) {  // pass 1: the history's tokens
    const uint32_t k = keys[i];
    if (k == kNoKey || (i > 0 && (keys[i - 1] >> 1) == (k >> 1))) continue;
    const uint32_t t = k >> 1;
    const int c_hist = lower_bound(keys, i, n, (t + 1) << 1) - lower_bound(keys, i, n, (t << 1) | 1u);
    const uint32_t on = same(t);
    for (int node = 0; node < nodes; ++node) penalise(lb + static_cast<size_t>(node) * V, t, rep, pres, freq, c_hist + __popc(on & s_out[node]));
  }
  for (int p = threadIdx.x; p < nodes * kMaxNodes; p += kPenThreads) {  // pass 2: path tokens absent from the history
    const int node = p / kMaxNodes, j = p % kMaxNodes;
    const uint32_t path = s_path[node], t = s_tok[j];
    if (!((path >> j) & 1u) || t == kNoKey) continue;
    const uint32_t on = same(t);
    if (on & path & ((1u << j) - 1u)) continue;  // an earlier path node has the same token
    const int at = lower_bound(keys, 0, n, t << 1);
    if (at < n && (keys[at] >> 1) == t) continue;  // in the history: pass 1
    penalise(lb + static_cast<size_t>(node) * V, t, rep, pres, freq, __popc(on & s_out[node]));
  }
}

// ------------------------------------------------------------------------------------------------
// log-probabilities of a chosen token and the top-n tokens
// ------------------------------------------------------------------------------------------------
constexpr int kMaxTop = 20;

struct TopSmem {
  int n_above, n_eq;
  uint32_t above_key[kMaxTop];  // this CTA's keys > tau (fewer than n in the whole cluster)
  int above_idx[kMaxTop];
  int eq_idx[kMaxTop];          // this CTA's first keys == tau, in index order
  uint32_t top_key[kMaxTop];    // rank 0: the merged, ordered list
  int top_idx[kMaxTop];
  uint32_t wmax[kWarps];        // this CTA's per-warp maximum keys (0: no non-NaN logit)
  uint32_t allw[kCluster * kWarps];
  uint32_t tau0;
};

__device__ __forceinline__ bool not_nan_bits(uint32_t b) { return (b & 0x7fffu) <= 0x7c00u; }
// the order key of the top-n list: -0 ties with +0
__device__ __forceinline__ uint32_t top_key(uint32_t b) { return okey(b == 0x8000u ? 0u : b); }

// One cluster of 8 CTAs per row (the sample_rows structure).  The softmax is the sampler's at T = 1: NaN and -inf weigh 0, w = exp(x - max)
// with w = 1 at the maximum, S = sum w in 64-bit fixed point; a logit's log-probability is (x - max) - log S in fp64 (-log S at the
// maximum).  Top-n: tau = the n-th largest non-NaN key by the two-level radix select over the keys above a lower bound (the n-th largest
// per-warp maximum); the keys > tau (fewer than n) and the first keys == tau in index order are merged by rank 0.
//
// logprob_row: that arithmetic for the fp16 row lrow, called by every thread of the cluster; rank 0 reads the scored token with token() at
// the end and writes logprob[out] and top_ids / top_logprobs[out * n .. + n).
template <typename Tok>
__device__ __forceinline__ void logprob_row(Smem& s, TopSmem& ts, __half* xs, const __half* lrow, int rank, int n, int V, Tok token, int out,
                                            float* __restrict__ logprob, long long* __restrict__ top_ids, float* __restrict__ top_logprobs) {
  int v0, v1;
  slice_of(V, rank, v0, v1);
  const int n_loc = (v1 - v0) * 8, g0 = v0 * 8;
  load_slice(xs, lrow, v0, v1);
  const uint16_t* xb = reinterpret_cast<const uint16_t*>(xs);
  int phase = 0;
  u64 all[kCluster];

  // max key and count of the weighted logits, count of the non-NaN ones
  u64 mk = 0, cv = 0, cn = 0;
  for (int i = threadIdx.x; i < n_loc; i += kThreads) {
    const uint32_t b = xb[i];
    if (valid_bits(b)) {
      mk = max(mk, static_cast<u64>(okey(b)));
      ++cv;
    }
    cn += not_nan_bits(b) ? 1 : 0;
  }
  mk = block_reduce(mk, s.red, OpMax());
  cv = block_reduce(cv, s.red, OpAdd());
  cn = block_reduce(cn, s.red, OpAdd());
  gather(s, phase, (mk << 48) | (cv << 24) | cn, all);  // counts < 2^24 (V <= 196608)
  mk = cv = cn = 0;
#pragma unroll
  for (int q = 0; q < kCluster; ++q) {
    mk = max(mk, all[q] >> 48);
    cv += (all[q] >> 24) & 0xffffffu;
    cn += all[q] & 0xffffffu;
  }
  const bool none = cv == 0;  // no weight: NaN log-probabilities, no top tokens
  float mz = 0.f;
  double log_s = 0.0;
  if (!none) {
    mz = __half2float(__ushort_as_half(static_cast<unsigned short>(key_bits(static_cast<uint32_t>(mk)))));
    u64 m = 0;
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (valid_bits(b)) m += fix(weight(b, 1.f, mz));
    }
    m = block_reduce(m, s.red, OpAdd());
    gather(s, phase, m, all);
    u64 S = 0;
#pragma unroll
    for (int q = 0; q < kCluster; ++q) S += all[q];
    log_s = log(static_cast<double>(S) * 9.094947017729282e-13);  // S 2^-40 >= 1
  }
  const float kNan = __int_as_float(0x7fc00000);
  auto lp_of = [&](float x) -> float {
    if (none || x != x) return kNan;
    if (x == mz) return static_cast<float>(-log_s);
    return static_cast<float>(static_cast<double>(x) - static_cast<double>(mz) - log_s);
  };

  const int ne = none ? 0 : static_cast<int>(min(static_cast<u64>(n), cn));  // listed tokens; the slots past ne get -1 / -inf
  if (ne > 0) {
    // tau0 = the ne-th largest of the cluster's 64 per-warp maximum keys: ne warps hold a key >= tau0 each, so the ne-th largest key is
    // >= tau0 and the histograms count only the keys >= tau0 (a handful for most rows, instead of the whole row on a few bins)
    uint32_t wm = 0;
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (not_nan_bits(b)) wm = max(wm, top_key(b));
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) wm = max(wm, __shfl_xor_sync(0xffffffffu, wm, m));
    if ((threadIdx.x & 31) == 0) ts.wmax[threadIdx.x >> 5] = wm;
    cluster_sync();
    if (threadIdx.x < kCluster * kWarps) ts.allw[threadIdx.x] = peer(ts.wmax, threadIdx.x / kWarps)[threadIdx.x % kWarps];
    __syncthreads();
    if (threadIdx.x < kCluster * kWarps) {
      const int t = threadIdx.x;
      const uint32_t v = ts.allw[t];
      int below = 0;  // the warp maxima ordered before this one (larger, or equal with a smaller position)
      for (int j = 0; j < kCluster * kWarps; ++j) below += (ts.allw[j] > v || (ts.allw[j] == v && j < t)) ? 1 : 0;
      if (below == ne - 1) ts.tau0 = v;
    }
    __syncthreads();
    const uint32_t tau0 = ts.tau0;
    u64 above;
    zero_hist(s);
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (not_nan_bits(b) && top_key(b) >= tau0) atomicAdd(&s.hist[top_key(b) >> 8], 1ull);
    }
    const int hi = hist_select<true>(s, static_cast<u64>(ne), 0, 0.0, above);
    zero_hist(s);
    for (int i = threadIdx.x; i < n_loc; i += kThreads) {
      const uint32_t b = xb[i];
      if (not_nan_bits(b) && top_key(b) >= tau0 && static_cast<int>(top_key(b) >> 8) == hi) atomicAdd(&s.hist[top_key(b) & 255u], 1ull);
    }
    const int lo = hist_select<true>(s, static_cast<u64>(ne) - above, 0, 0.0, above);
    const uint32_t tau = static_cast<uint32_t>(hi << 8 | lo);
    if (threadIdx.x == 0) ts.n_above = 0;
    __syncthreads();
    const int per = (n_loc + kThreads - 1) / kThreads;
    const int i0 = min(static_cast<int>(threadIdx.x) * per, n_loc), i1 = min(i0 + per, n_loc);
    u64 ce = 0;
    for (int i = i0; i < i1; ++i) {
      const uint32_t b = xb[i];
      if (!not_nan_bits(b)) continue;
      const uint32_t k = top_key(b);
      if (k > tau) {
        const int slot = atomicAdd(&ts.n_above, 1);
        ts.above_key[slot] = k;
        ts.above_idx[slot] = g0 + i;
      } else if (k == tau) {
        ++ce;
      }
    }
    const u64 ex = block_excl_scan(ce, s.red);
    if (ce > 0 && ex < static_cast<u64>(ne)) {
      int j = static_cast<int>(ex);
      for (int i = i0; i < i1 && j < ne; ++i) {
        const uint32_t b = xb[i];
        if (not_nan_bits(b) && top_key(b) == tau) ts.eq_idx[j++] = g0 + i;
      }
    }
    if (threadIdx.x == kThreads - 1) ts.n_eq = static_cast<int>(min(ex + ce, static_cast<u64>(ne)));
    cluster_sync();  // every CTA's lists are complete
    if (rank == 0 && threadIdx.x == 0) {
      int m = 0;
      for (int r = 0; r < kCluster; ++r) {  // the keys > tau, insertion-sorted by (key descending, index ascending)
        const TopSmem* p = peer(&ts, r);
        for (int a = 0; a < p->n_above; ++a) {
          const uint32_t k = p->above_key[a];
          const int idx = p->above_idx[a];
          int j = m++;
          while (j > 0 && (ts.top_key[j - 1] < k || (ts.top_key[j - 1] == k && ts.top_idx[j - 1] > idx))) {
            ts.top_key[j] = ts.top_key[j - 1];
            ts.top_idx[j] = ts.top_idx[j - 1];
            --j;
          }
          ts.top_key[j] = k;
          ts.top_idx[j] = idx;
        }
      }
      for (int r = 0; r < kCluster && m < ne; ++r) {  // then the ties at tau, lowest indices first
        const TopSmem* p = peer(&ts, r);
        for (int a = 0; a < p->n_eq && m < ne; ++a) {
          ts.top_key[m] = tau;
          ts.top_idx[m++] = p->eq_idx[a];
        }
      }
    }
  }
  if (rank == 0 && threadIdx.x == 0) {
    const long long t = token();
    logprob[out] = (t >= 0 && t < V) ? lp_of(__half2float(lrow[t])) : kNan;
    for (int j = 0; j < n; ++j) {
      const bool listed = j < ne;
      top_ids[static_cast<size_t>(out) * n + j] = listed ? ts.top_idx[j] : -1;
      top_logprobs[static_cast<size_t>(out) * n + j] =
          listed ? lp_of(__half2float(__ushort_as_half(static_cast<unsigned short>(key_bits(ts.top_key[j]))))) : (none ? kNan : -INFINITY);
    }
  }
  cluster_sync();  // the peers' lists stay alive until rank 0 has read them
}

__global__ void __launch_bounds__(kThreads, 1) logprobs_rows_kernel(float* __restrict__ logprob, long long* __restrict__ top_ids,
                                                                  float* __restrict__ top_logprobs, const __half* __restrict__ logits,
                                                                  const long long* __restrict__ tokens, int n, int V) {
  extern __shared__ uint4 dyn[];
  __shared__ Smem s;
  __shared__ TopSmem ts;
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits and tokens may come from the preceding kernels
  const int row = blockIdx.x / kCluster, rank = blockIdx.x % kCluster;
  logprob_row(s, ts, reinterpret_cast<__half*>(dyn), logits + static_cast<size_t>(row) * V, rank, n, V, [&] { return tokens[row]; }, row, logprob,
              top_ids, top_logprobs);
}

// The log-probabilities of the tokens a speculative step emits, one cluster per (sequence b, emitted token k).  With acc = accept_len[b]
// clamped to [1, nodes] and path entries to [0, nodes - 1] (as spec_commit clamps them), token k < acc is draft[path[k + 1]] for k < acc - 1
// and bonus[b] for k = acc - 1; it is scored by node row path[k] with the logprobs_rows arithmetic and written at history column
// min(max(seq_lens[b], 0), W) + k, where spec_commit puts it.  Finished rows, tokens past acc and columns >= W exit after the dependency wait.
__global__ void __launch_bounds__(kThreads, 1) logprobs_accepted_kernel(float* __restrict__ logprob, long long* __restrict__ top_ids,
                                                                      float* __restrict__ top_logprobs, const __half* __restrict__ logits,
                                                                      const long long* __restrict__ draft, const int* __restrict__ path,
                                                                      const int* __restrict__ accept_len, const long long* __restrict__ bonus,
                                                                      const int* __restrict__ seq_lens, const int* __restrict__ finished, int nodes,
                                                                      int n, int V, int W) {
  extern __shared__ uint4 dyn[];
  __shared__ Smem s;
  __shared__ TopSmem ts;
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // logits and the acceptance outputs come from the preceding kernels, the lengths from the previous step
  const int c = blockIdx.x / kCluster, rank = blockIdx.x % kCluster;
  const int b = c / nodes, k = c % nodes;
  if (finished[b]) return;  // uniform over the cluster: every CTA reads the same values
  const int acc = min(max(accept_len[b], 1), nodes);
  const int col = min(max(seq_lens[b], 0), W) + k;
  if (k >= acc || col >= W) return;
  const size_t row0 = static_cast<size_t>(b) * nodes;
  const int node = min(max(path[row0 + k], 0), nodes - 1);
  logprob_row(s, ts, reinterpret_cast<__half*>(dyn), logits + (row0 + node) * V, rank, n, V,
              [&] { return k + 1 < acc ? draft[row0 + min(max(path[row0 + k + 1], 0), nodes - 1)] : bonus[b]; }, b * W + col, logprob, top_ids,
              top_logprobs);
}

int slice_cap_of(int V) { return ((V / 8 + kCluster - 1) / kCluster) * 8; }

}  // namespace

int sample_rows(const SampleArgs& a) {
  QS_REQUIRE(a.rows >= 0 && a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "sample_rows: rows=%d vocab=%d (a multiple of 8, 8 .. %d)",
             a.rows, a.vocab, kMaxVocab);
  QS_REQUIRE(a.rows <= 0x7fffffff / kCluster, "sample_rows: too many rows");
  if (a.rows == 0) return QS_OK;
  QS_REQUIRE(a.out && a.logits && a.temperature && a.top_k && a.top_p && a.offsets, "sample_rows: null pointer");
  const int cap = slice_cap_of(a.vocab);
  const size_t smem = static_cast<size_t>(cap) * 2;
  const int rc = raise_smem_limit(sample_rows_kernel, smem, "sample_rows");
  if (rc) return rc;
  return launch(sample_rows_kernel, dim3(static_cast<unsigned>(a.rows) * kCluster), dim3(kThreads), smem, kCluster, a.stream, "sample_rows", a.out,
                static_cast<const __half*>(a.logits), a.temperature, a.top_k, a.top_p, static_cast<u64>(a.seed), a.offsets, a.vocab);
}

int tree_accept_sampling(const TreeAcceptSamplingArgs& a) {
  QS_REQUIRE(a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "tree_accept_sampling: batch=%d, num_nodes=%d (1 .. 16)", a.batch,
             a.num_nodes);
  QS_REQUIRE(a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "tree_accept_sampling: vocab=%d (a multiple of 8, 8 .. %d)", a.vocab,
             kMaxVocab);
  QS_REQUIRE(a.batch <= 0x7fffffff / kCluster, "tree_accept_sampling: batch too large");
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.draft && a.tree_mask && a.logits && a.temperature && a.top_k && a.top_p && a.offsets && a.accept_len && a.path && a.bonus,
             "tree_accept_sampling: null pointer");
  const int cap = slice_cap_of(a.vocab);
  const size_t smem = static_cast<size_t>(cap) * 6;  // above the default 48 KB for V > 65536
  const int rc = raise_smem_limit(tree_accept_sampling_kernel, smem, "tree_accept_sampling");
  if (rc) return rc;
  return launch(tree_accept_sampling_kernel, dim3(static_cast<unsigned>(a.batch) * kCluster), dim3(kThreads), smem, kCluster, a.stream,
                "tree_accept_sampling", a.draft, a.tree_mask, static_cast<const __half*>(a.logits), a.draft_probs, a.temperature, a.top_k, a.top_p,
                static_cast<u64>(a.seed), a.offsets, a.accept_len, a.path, a.bonus, a.num_nodes, a.vocab, cap);
}

int apply_penalties(const PenaltyArgs& a) {
  QS_REQUIRE(a.rows >= 0 && a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "apply_penalties: rows=%d vocab=%d (a multiple of 8, 8 .. %d)",
             a.rows, a.vocab, kMaxVocab);
  QS_REQUIRE(a.history_len >= 0 && a.history_len <= kMaxHistory, "apply_penalties: history_len=%d (0 .. %d)", a.history_len, kMaxHistory);
  if (a.rows == 0 || a.history_len == 0) return QS_OK;
  QS_REQUIRE(a.logits && a.history && a.prompt_lens && a.seq_lens && a.repetition && a.presence && a.frequency, "apply_penalties: null pointer");
  int n = 1;
  while (n < a.history_len) n <<= 1;
  const size_t smem = static_cast<size_t>(n) * sizeof(uint32_t);
  const int rc = raise_smem_limit(apply_penalties_kernel, smem, "apply_penalties");
  if (rc) return rc;
  return launch(apply_penalties_kernel, dim3(static_cast<unsigned>(a.rows)), dim3(kPenThreads), smem, 0, a.stream, "apply_penalties",
                static_cast<__half*>(a.logits), a.history, a.prompt_lens, a.seq_lens, a.repetition, a.presence, a.frequency, a.vocab,
                a.history_len);
}

int logprobs_rows(const LogprobArgs& a) {
  QS_REQUIRE(a.rows >= 0 && a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "logprobs_rows: rows=%d vocab=%d (a multiple of 8, 8 .. %d)",
             a.rows, a.vocab, kMaxVocab);
  QS_REQUIRE(a.n >= 0 && a.n <= kMaxTop, "logprobs_rows: n=%d (0 .. %d)", a.n, kMaxTop);
  QS_REQUIRE(a.rows <= 0x7fffffff / kCluster, "logprobs_rows: too many rows");
  if (a.rows == 0) return QS_OK;
  QS_REQUIRE(a.logprob && a.logits && a.tokens && (a.n == 0 || (a.top_ids && a.top_logprobs)), "logprobs_rows: null pointer");
  const size_t smem = static_cast<size_t>(slice_cap_of(a.vocab)) * 2;
  const int rc = raise_smem_limit(logprobs_rows_kernel, smem, "logprobs_rows");
  if (rc) return rc;
  return launch(logprobs_rows_kernel, dim3(static_cast<unsigned>(a.rows) * kCluster), dim3(kThreads), smem, kCluster, a.stream, "logprobs_rows",
                a.logprob, a.top_ids, a.top_logprobs, static_cast<const __half*>(a.logits), a.tokens, a.n, a.vocab);
}

int apply_penalties_tree(const PenaltyTreeArgs& a) {
  QS_REQUIRE(a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "apply_penalties_tree: batch=%d num_nodes=%d (1 .. %d)", a.batch,
             a.num_nodes, kMaxNodes);
  QS_REQUIRE(a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "apply_penalties_tree: vocab=%d (a multiple of 8, 8 .. %d)", a.vocab,
             kMaxVocab);
  QS_REQUIRE(a.history_len >= 0 && a.history_len <= kMaxHistory, "apply_penalties_tree: history_len=%d (0 .. %d)", a.history_len, kMaxHistory);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.logits && a.draft && a.tree_mask && (a.history || a.history_len == 0) && a.prompt_lens && a.seq_lens && a.repetition && a.presence &&
                 a.frequency,
             "apply_penalties_tree: null pointer");
  int n = 1;
  while (n < a.history_len) n <<= 1;
  const size_t smem = static_cast<size_t>(n) * sizeof(uint32_t);
  const int rc = raise_smem_limit(apply_penalties_tree_kernel, smem, "apply_penalties_tree");
  if (rc) return rc;
  return launch(apply_penalties_tree_kernel, dim3(static_cast<unsigned>(a.batch)), dim3(kPenThreads), smem, 0, a.stream, "apply_penalties_tree",
                static_cast<__half*>(a.logits), a.draft, a.tree_mask, a.history, a.prompt_lens, a.seq_lens, a.repetition, a.presence, a.frequency,
                a.num_nodes, a.vocab, a.history_len);
}

int logprobs_accepted(const LogprobAcceptedArgs& a) {
  QS_REQUIRE(a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "logprobs_accepted: batch=%d num_nodes=%d (1 .. %d)", a.batch,
             a.num_nodes, kMaxNodes);
  QS_REQUIRE(a.vocab >= 8 && a.vocab % 8 == 0 && a.vocab <= kMaxVocab, "logprobs_accepted: vocab=%d (a multiple of 8, 8 .. %d)", a.vocab, kMaxVocab);
  QS_REQUIRE(a.n >= 0 && a.n <= kMaxTop, "logprobs_accepted: n=%d (0 .. %d)", a.n, kMaxTop);
  QS_REQUIRE(a.width >= 1, "logprobs_accepted: width=%d", a.width);
  QS_REQUIRE(static_cast<long long>(a.batch) * a.num_nodes <= 0x7fffffff / kCluster &&
                 static_cast<long long>(a.batch) * a.width * (a.n > 0 ? a.n : 1) <= 0x7fffffffLL,
             "logprobs_accepted: batch too large");
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.logprob && a.logits && a.draft && a.path && a.accept_len && a.bonus && a.seq_lens && a.finished &&
                 (a.n == 0 || (a.top_ids && a.top_logprobs)),
             "logprobs_accepted: null pointer");
  const size_t smem = static_cast<size_t>(slice_cap_of(a.vocab)) * 2;
  const int rc = raise_smem_limit(logprobs_accepted_kernel, smem, "logprobs_accepted");
  if (rc) return rc;
  return launch(logprobs_accepted_kernel, dim3(static_cast<unsigned>(a.batch * a.num_nodes) * kCluster), dim3(kThreads), smem, kCluster, a.stream,
                "logprobs_accepted", a.logprob, a.top_ids, a.top_logprobs, static_cast<const __half*>(a.logits), a.draft, a.path, a.accept_len,
                a.bonus, a.seq_lens, a.finished, a.num_nodes, a.n, a.vocab, a.width);
}

}  // namespace qs
