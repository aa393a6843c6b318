// qserve_b200 -- beam search inside the captured decode step (SamplingParams.use_beam_search), sm_90a.
//
// R requests of W <= 8 beams each; request r owns rows r W .. r W + W - 1.  Every step the decode runner scores each live beam's 2 W best
// next tokens with logprobs_rows, then:
//   beam_select_kernel   one CTA per request: merges the W x 2 W candidates, keeps the finished hypotheses in a pool of W, decides when the
//                        request stops and assigns the running children to the request's slots (the contract is tests/beam_oracle.py).
//   beam_reorder_kernel  re-parents every slot whose parent is another slot: page-table entries, the filled slots of the partial tail page
//                        and the generated token history, for every layer in one launch.
//
// The parents of one step are a permutation with repeats inside a request: a slot can be a parent and a child at once, which kv_fork_kernel
// does not allow.  The reorder therefore stages every copy through shared memory: a CTA owns one (request, layer, K / V, KV head) slice (or
// the request's table entries / history) and reads the slices of all W parents before it writes any child.  Requests never share rows, so
// no ordering between CTAs is needed.
//
// Two conditions make the in-place reorder sound; the decode runner keeps both.
//   * Pages are never written while shared.  A row writes only its own page, at block (context_len - 1) / 64.  After the reorder a child's
//     entries below P / 64 (P = the cached tokens after this step's decode) are its parent's and entry P / 64 stays the child's own page, so
//     no other row's table references a row's own page at or above that row's tail block.  beam_select gives every slot of a request it
//     ran, dead or alive, context_len = P + 1; a dead slot and every slot of a done request keep being computed at fixed shapes but are not
//     advanced, and write only position P of their own page, which no table shares.
//   * Table writes finish before they are read.  The attention kernels read page tables and context lengths before their dependency wait.
//     The reorder's table writes (and beam_select's context lengths) reach them only because the next step begins with the embedding
//     gather, a launch without programmatic dependent launch.  Keep the reorder before that boundary.
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kMaxBeam = 8;
constexpr int kMaxCand = 2 * kMaxBeam;
constexpr int kSelectThreads = kMaxBeam * kMaxCand;  // one thread per candidate
constexpr int kTokensPerPage = 64;
constexpr int kReorderThreads = 256;
constexpr int kStageBytes = 16384;

// The hypothesis score of vLLM's get_beam_search_score: cum / len ** length_penalty, a correctly rounded division.
__device__ __forceinline__ float beam_score(float cum, int len, float length_penalty) {
  return __fdiv_rn(cum, powf(static_cast<float>(len), length_penalty));
}

__global__ void __launch_bounds__(kSelectThreads) beam_select_kernel(BeamSelectArgs a) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int W = a.beam_width, C = 2 * W, r = blockIdx.x, base = r * W;
  const int k = threadIdx.x;
  if (a.done[r]) {
    if (k < W) a.parents[base + k] = -1;
    return;
  }
  __shared__ float s_s[kSelectThreads];
  __shared__ long long s_id[kSelectThreads];
  __shared__ int s_ok[kSelectThreads];
  __shared__ int s_child[kMaxCand];  // candidate index of child c (children ordered by score)
  __shared__ int s_run[kMaxBeam];    // running children, in child order
  __shared__ int s_src[kMaxBeam];    // new pool entry q: old entry s_src[q] >= 0, or child -s_src[q] - 1
  __shared__ float s_pcum[kMaxBeam], s_pscore[kMaxBeam];
  __shared__ int s_plen[kMaxBeam];
  __shared__ int s_count, s_nrun, s_done;
  const int L = a.seq_lens[base], P0 = a.prompt_lens[base];  // every live beam of the request has this length
  const int out_len = L - P0;
  // 1. candidates: s = cum_j + lp, ids < 0 and dead slots skipped
  bool ok = false;
  float s = 0.f;
  long long id = -1;
  if (k < W * C) {
    const int j = k / C;
    if (a.live[base + j]) {
      id = a.top_ids[static_cast<size_t>(base + j) * C + (k - j * C)];
      if (id >= 0) {
        ok = true;
        s = __fadd_rn(a.cum[base + j], a.top_logprobs[static_cast<size_t>(base + j) * C + (k - j * C)]);
      }
    }
  }
  s_s[k] = s;
  s_id[k] = id;
  s_ok[k] = ok;
  __syncthreads();
  // 2. selection: rank by (s descending, candidate index ascending); the index orders (slot, rank) lexicographically
  if (ok) {
    int pos = 0;
    for (int q = 0; q < W * C; ++q) pos += s_ok[q] && (s_s[q] > s || (s_s[q] == s && q < k));
    if (pos < C) s_child[pos] = k;
  }
  const int nvalid = __syncthreads_count(ok);
  const int nchild = min(C, nvalid);
  const int budget = min(max(a.budget[r], 1), a.max_tokens);
  // 3 - 7: finishing, the pool merge and the stopping rule (at most W + 2 W items: one thread)
  if (k == 0) {
    const float lp = a.length_penalty[r];
    const long long eos = a.eos[r];
    const int clen = L + 1;  // prompt plus generated tokens of a child
    float it_score[kMaxBeam + kMaxCand];
    int it_src[kMaxBeam + kMaxCand];
    int n = a.pool_count[r];
    n = min(max(n, 0), W);
    for (int q = 0; q < n; ++q) {
      it_score[q] = a.pool_score[base + q];
      it_src[q] = q;
    }
    int nrun = 0;
    for (int c = 0; c < nchild; ++c) {
      const long long tok = s_id[s_child[c]];
      bool fin = (eos >= 0 && tok == eos) || out_len + 1 >= budget;
      for (int i = 0; i < a.num_stops; ++i) fin |= a.stop_ids[static_cast<size_t>(r) * a.num_stops + i] >= 0 && tok == a.stop_ids[static_cast<size_t>(r) * a.num_stops + i];
      if (!fin) {
        if (nrun < W) s_run[nrun] = c;
        ++nrun;
        continue;
      }
      // stable insertion by score descending: after every item with score >= this one
      const float sc = beam_score(s_s[s_child[c]], clen - (eos >= 0 && tok == eos ? 1 : 0), lp);
      int at = n;
      while (at > 0 && !(it_score[at - 1] >= sc)) {
        it_score[at] = it_score[at - 1];
        it_src[at] = it_src[at - 1];
        --at;
      }
      it_score[at] = sc;
      it_src[at] = -c - 1;
      ++n;
    }
    const int count = min(n, W);
    for (int q = 0; q < count; ++q) {
      s_src[q] = it_src[q];
      s_pscore[q] = it_score[q];
      if (it_src[q] >= 0) {
        s_pcum[q] = a.pool_cum[base + it_src[q]];
        s_plen[q] = a.pool_len[base + it_src[q]];
      } else {
        s_pcum[q] = s_s[s_child[-it_src[q] - 1]];
        s_plen[q] = min(max(out_len + 1, 0), a.max_tokens);
      }
    }
    bool done = nrun == 0;
    if (!done && count == W) {
      const int es = a.early_stopping[r];
      if (es == 1) {
        done = true;
      } else {
        const float best = s_s[s_child[s_run[0]]];
        const int len = (es == 2 && lp > 0.f) ? max(P0 + budget, a.max_model_len) : clen;
        done = s_pscore[W - 1] >= beam_score(best, len, lp);
      }
    }
    s_count = count;
    s_nrun = min(nrun, W);
    s_done = done;
  }
  __syncthreads();
  const int count = s_count;
  long long* pool = a.pool_tokens + static_cast<size_t>(base) * a.max_tokens;
  // kept old hypotheses move to the same or a later entry: move them last entry first
  for (int q = count - 1; q >= 0; --q) {
    const int o = s_src[q];
    if (o >= 0 && o != q) {
      for (int i = k; i < s_plen[q]; i += kSelectThreads) pool[static_cast<size_t>(q) * a.max_tokens + i] = pool[static_cast<size_t>(o) * a.max_tokens + i];
    }
    __syncthreads();
  }
  // new hypotheses: the parent's generated tokens, then the child's token
  for (int q = 0; q < count; ++q) {
    if (s_src[q] >= 0) continue;
    const int kk = s_child[-s_src[q] - 1];
    const long long* h = a.history + static_cast<size_t>(base + kk / C) * a.history_len;
    long long* dst = pool + static_cast<size_t>(q) * a.max_tokens;
    for (int i = k; i < min(out_len, a.max_tokens); i += kSelectThreads) dst[i] = P0 + i < a.history_len ? h[P0 + i] : -1;
    if (k == 0 && out_len >= 0 && out_len < a.max_tokens) dst[out_len] = s_id[kk];
  }
  if (k < count) {
    a.pool_len[base + k] = s_plen[k];
    a.pool_cum[base + k] = s_pcum[k];
    a.pool_score[base + k] = s_pscore[k];
  }
  // 8. the new beams
  if (k < W) {
    const int slot = base + k;
    if (!s_done && k < s_nrun) {
      const int kk = s_child[s_run[k]];
      a.parents[slot] = base + kk / C;
      a.tokens[slot] = s_id[kk];
      a.cum[slot] = s_s[kk];
      a.live[slot] = 1;
    } else {
      a.parents[slot] = -1;
      a.live[slot] = 0;
    }
    a.seq_lens[slot] = L + 1;
    a.context_lens[slot] = L + 1;
  }
  if (k == 0) {
    a.pool_count[r] = count;
    a.done[r] = s_done;
  }
}

// dst[i][0 .. n[i]) = src[i][0 .. n[i]) for every slot i < w with src[i] != null, through `stage`: every chunk is read from all sources before
// it is written to any destination.  Sources and destinations sit at the same offset of their slot's slice, so a chunk's writes never reach
// what a later chunk reads, and a slot may be a source and a destination at once.
template <typename E>
__device__ void move_slices(unsigned char* stage, int w, const void* const* src, void* const* dst, const int* n, int n_max) {
  E* buf = reinterpret_cast<E*>(stage);
  const int cap = kStageBytes / static_cast<int>(sizeof(E)) / w;
  for (int c0 = 0; c0 < n_max; c0 += cap) {
    const int m = min(cap, n_max - c0);
    for (int e = threadIdx.x; e < w * m; e += kReorderThreads) {
      const int i = e / m, x = c0 + e - i * m;
      if (src[i] && x < n[i]) buf[i * cap + x - c0] = static_cast<const E*>(src[i])[x];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < w * m; e += kReorderThreads) {
      const int i = e / m, x = c0 + e - i * m;
      if (src[i] && x < n[i]) static_cast<E*>(dst[i])[x] = buf[i * cap + x - c0];
    }
    __syncthreads();
  }
}

template <int BITS>
__global__ void __launch_bounds__(kReorderThreads) beam_reorder_kernel(long long* kv_pointers, const int* __restrict__ parents,
                                                                       const int* __restrict__ context_lens, const int* __restrict__ prompt_lens,
                                                                       const long long* __restrict__ tokens, long long* history, int batch,
                                                                       int beam_width, int max_blocks, int num_kv_heads, int code_bytes,
                                                                       int history_len) {
  constexpr int kRow = 128 * BITS / 8;  // code bytes of one (token, KV head)
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  __shared__ __align__(16) unsigned char stage[kStageBytes];
  __shared__ const void* s_src[kMaxBeam];
  __shared__ void* s_dst[kMaxBeam];
  __shared__ int s_n[kMaxBeam], s_p[kMaxBeam], s_P[kMaxBeam];
  const int W = beam_width, base = blockIdx.x * W;
  const int layer = blockIdx.y >> 1, kv = blockIdx.y & 1, head = blockIdx.z;
  long long* table = kv_pointers + static_cast<size_t>(layer) * batch * 2 * max_blocks;
  if (threadIdx.x < W) {
    const int s = base + threadIdx.x;
    const int p = parents[s];
    s_p[threadIdx.x] = p >= base && p < base + W ? p : -1;  // parents outside the request are ignored
    // one P per request, the first slot's: every entry the table CTA writes (< P / 64) differs from every entry the head CTAs read (P / 64)
    s_P[threadIdx.x] = context_lens[base] - 1;
  }
  __syncthreads();
  // slot i moves when its parent is another slot
  auto moving = [&](int i) { return s_p[i] >= 0 && s_p[i] != base + i && s_P[i] > 0; };
  if (head < num_kv_heads) {  // the filled slots 0 .. P % 64 - 1 of the parent's tail page, codes then scale and zero rows of this head
    int n_max = 0;
    if (threadIdx.x < W) {
      const int i = threadIdx.x, P = s_P[i], t = P % kTokensPerPage, blk = P / kTokensPerPage;
      const bool go = moving(i) && t > 0 && blk < max_blocks;
      s_src[i] = go ? reinterpret_cast<const void*>(table[(static_cast<size_t>(s_p[i]) * 2 + kv) * max_blocks + blk]) : nullptr;
      s_dst[i] = go ? reinterpret_cast<void*>(table[(static_cast<size_t>(base + i) * 2 + kv) * max_blocks + blk]) : nullptr;
      s_n[i] = go ? t : 0;
    }
    __syncthreads();
    for (int i = 0; i < W; ++i) n_max = max(n_max, s_n[i]);
    if (n_max == 0) return;
    __shared__ const void* c_src[kMaxBeam];
    __shared__ void* c_dst[kMaxBeam];
    __shared__ int c_n[kMaxBeam];
    constexpr int kVec = kRow / 16;  // 16-byte vectors per token
    if (threadIdx.x < W) {
      const int i = threadIdx.x;
      const size_t off = static_cast<size_t>(head) * kTokensPerPage * kRow;
      c_src[i] = s_src[i] ? static_cast<const uint8_t*>(s_src[i]) + off : nullptr;
      c_dst[i] = s_dst[i] ? static_cast<uint8_t*>(s_dst[i]) + off : nullptr;
      c_n[i] = s_n[i] * kVec;
    }
    __syncthreads();
    move_slices<uint4>(stage, W, c_src, c_dst, c_n, n_max * kVec);
    for (int row = 0; row < 2; ++row) {  // [2][Hkv][64] fp16: scale rows, then zero rows
      if (threadIdx.x < W) {
        const int i = threadIdx.x;
        const size_t off = code_bytes + (static_cast<size_t>(row) * num_kv_heads + head) * kTokensPerPage * sizeof(__half);
        c_src[i] = s_src[i] ? static_cast<const uint8_t*>(s_src[i]) + off : nullptr;
        c_dst[i] = s_dst[i] ? static_cast<uint8_t*>(s_dst[i]) + off : nullptr;
        c_n[i] = s_n[i];
      }
      __syncthreads();
      move_slices<__half>(stage, W, c_src, c_dst, c_n, n_max);
    }
    return;
  }
  // head == num_kv_heads: the table entries of this (layer, K / V) below P / 64, and for blockIdx.y == 0 the token history
  int n_max = 0;
  if (threadIdx.x < W) {
    const int i = threadIdx.x;
    const bool go = moving(i);
    s_src[i] = go ? table + (static_cast<size_t>(s_p[i]) * 2 + kv) * max_blocks : nullptr;
    s_dst[i] = go ? table + (static_cast<size_t>(base + i) * 2 + kv) * max_blocks : nullptr;
    s_n[i] = go ? min(s_P[i] / kTokensPerPage, max_blocks) : 0;
  }
  __syncthreads();
  for (int i = 0; i < W; ++i) n_max = max(n_max, s_n[i]);
  move_slices<long long>(stage, W, s_src, s_dst, s_n, n_max);
  if (blockIdx.y != 0) return;
  n_max = 0;
  if (threadIdx.x < W) {  // generated columns [P0, P) from the parent
    const int i = threadIdx.x, P0 = max(prompt_lens[base + i], 0), P = min(s_P[i], history_len);
    const bool go = moving(i) && P > P0;
    s_src[i] = go ? history + static_cast<size_t>(s_p[i]) * history_len + P0 : nullptr;
    s_dst[i] = go ? history + static_cast<size_t>(base + i) * history_len + P0 : nullptr;
    s_n[i] = go ? P - P0 : 0;
  }
  __syncthreads();
  for (int i = 0; i < W; ++i) n_max = max(n_max, s_n[i]);
  move_slices<long long>(stage, W, s_src, s_dst, s_n, n_max);
  if (threadIdx.x < W) {  // every live child appends its token at column P
    const int i = threadIdx.x, P = s_P[i];
    if (s_p[i] >= 0 && P >= 0 && P < history_len) history[static_cast<size_t>(base + i) * history_len + P] = tokens[base + i];
  }
}

}  // namespace

int beam_select(const BeamSelectArgs& a) {
  QS_REQUIRE(a.num_requests >= 0 && a.beam_width >= 1 && a.beam_width <= kMaxBeam, "beam_select: num_requests=%d beam_width=%d (1 .. %d)",
             a.num_requests, a.beam_width, kMaxBeam);
  QS_REQUIRE(a.max_tokens >= 1 && a.history_len >= 1 && a.num_stops >= 0 && a.num_stops <= 8,
             "beam_select: max_tokens=%d history_len=%d num_stops=%d (0 .. 8)", a.max_tokens, a.history_len, a.num_stops);
  if (a.num_requests == 0) return QS_OK;
  QS_REQUIRE(a.top_ids && a.top_logprobs && a.live && a.cum && a.seq_lens && a.context_lens && a.tokens && a.parents && a.prompt_lens &&
                 a.history && a.length_penalty && a.early_stopping && a.eos && (a.stop_ids || a.num_stops == 0) && a.budget && a.done &&
                 a.pool_tokens && a.pool_len && a.pool_cum && a.pool_score && a.pool_count,
             "beam_select: null pointer");
  return launch(beam_select_kernel, dim3(a.num_requests), dim3(kSelectThreads), 0, 0, a.stream, "beam_select", a);
}

int beam_reorder(const BeamReorderArgs& a) {
  QS_REQUIRE(a.layers >= 1 && a.layers <= 32767 && a.batch >= 0 && a.beam_width >= 1 && a.beam_width <= kMaxBeam && a.max_blocks >= 1 &&
                 a.num_kv_heads >= 1 && a.num_kv_heads < 65535 && a.history_len >= 1,
             "beam_reorder: layers=%d (1 .. 32767) batch=%d beam_width=%d (1 .. %d) max_blocks=%d kv_heads=%d history_len=%d", a.layers, a.batch,
             a.beam_width, kMaxBeam, a.max_blocks, a.num_kv_heads, a.history_len);
  QS_REQUIRE(a.batch % a.beam_width == 0, "beam_reorder: batch=%d is not a multiple of beam_width=%d", a.batch, a.beam_width);
  QS_REQUIRE(a.tokens_per_block == kTokensPerPage, "beam_reorder: tokens_per_block=%d, only 64 is supported", a.tokens_per_block);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * 128 * bits / 8, "beam_reorder: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.kv_pointers && a.parents && a.context_lens && a.prompt_lens && a.tokens && a.history, "beam_reorder: null pointer");
  const int code_bytes = kTokensPerPage * a.size_per_token;
  return launch(a.int4_kv ? beam_reorder_kernel<4> : beam_reorder_kernel<8>,
                dim3(static_cast<unsigned>(a.batch / a.beam_width), static_cast<unsigned>(a.layers) * 2u, static_cast<unsigned>(a.num_kv_heads) + 1u),
                dim3(kReorderThreads), 0, 0, a.stream, "beam_reorder", a.kv_pointers, a.parents, a.context_lens, a.prompt_lens, a.tokens,
                a.history, a.batch, a.beam_width, a.max_blocks, a.num_kv_heads, code_bytes, a.history_len);
}

}  // namespace qs
