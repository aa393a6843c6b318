// qserve_b200 -- the schedule of the decode runner's in-flight batching step, sm_90a (DESIGN.md 3.12).
//
// inflight_schedule_kernel runs first in every in-flight step, as one CTA: it retires the rows whose request the previous step finished,
// admits queued requests into free rows first-come-first-served, plans the step's chunk segment (the next prompt tokens of the prefilling rows
// in admission order, laid out in row order) and its decode segment (the decoding rows; every other row idle), and sets the tail masks the
// unchanged sampler and commit read.  The rules are those of include/qserve_b200.h (qs_inflight_schedule), restated in tests/inflight_oracle.py.
//
// The decisions that depend on other rows (the retire ring order, which row takes which request, the admission-order scan of the chunk
// budget, the row-order offsets) are made by thread 0 over shared-memory copies of the row state: B <= 512 rows, a few cycles each.  The
// bulk copies (histories of retiring and admitted rows, the chunk's token ids) are spread over the whole block.  Every input is read after
// the PDL dependency wait: the previous step's commit writes the lengths, the histories and `finished`, and the host writes the queue and
// the tail counter between steps.
//
// inflight_schedule_kernel<true, false> adds the shared KV page pool of qs_inflight_schedule_pool: thread 0 also keeps the free stack (retire
// and preemption push, decode growth and starts pop, in the header's order), and the block then writes the new table entries of every layer.
// <false, false> is the same body with no page step: every PREFILL row counts as started and its target is its prompt length.
//
// inflight_schedule_kernel<true, true> adds the prefix cache of qs_inflight_schedule_pool_cache: per-page refs, states, epochs and keys, an LRU
// list of the evictable pages and an open-addressing index of the registered ones, all in device memory.  The two scans that touch the 64
// token ids of a page run block-parallel, a warp per page or row, so thread 0 only makes the serial decisions: the token hashes of the pages
// rule 0 may register (written with the ids into the pages' key slots; a private page's key slot is scratch), and the longest match of every
// waiting row, searched after the decode growth.  Registrations happen only in rule 0, so during the starts a match can only shrink, when a
// start evicts one of its pages: thread 0 cuts it at the first page that is no longer registered, which gives the sequential rule exactly.
#include <math_constants.h>

#include <climits>

#include "../../include/qserve_b200.h"
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxRows = 512;
constexpr int kStops = 8;  // stop ids per request (MAX_STOP_TOKENS)
constexpr int kWarps = kThreads / 32;
constexpr int kPageTokens = 64;
enum : int { kFree = 0, kPrefill = 1, kDecode = 2 };
enum : int { kPageFree = 0, kPagePrivate = 1, kPageRegistered = 2 };
// qs_prefix_cache_args.counters
enum : int { kLruHead = 0, kLruTail = 1, kEvictable = 2, kRegistered = 3, kHitPages = 4, kRegistrations = 5, kEvictions = 6, kDuplicates = 7,
             kCacheCounters = 8 };
enum : int { kHead = 0, kTail = 1, kRetired = 2, kAdmitted = 3 };
enum : int { kReasonEos = 1, kReasonStop = 2, kReasonBudget = 3 };

// Pushes row b's pages [0, count) onto the free stack in page order (thread 0).
__device__ __forceinline__ void push_pages(const qs_kv_pool_args& p, int b, int count, int& top) {
  const int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
  for (int j = 0; j < count; ++j) p.free_pages[top++] = pg[j];
}

// ---- prefix cache (qs_inflight_schedule_pool_cache); tests/prefix_cache_oracle.py computes the same hashes ----
__device__ __forceinline__ uint32_t fmix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

// The token hash of a page: the sum of every id's mix with its slot, summed over a warp (lane i holds ids i and i + 32).
__device__ __forceinline__ uint32_t token_hash(int t0, int t1, int lane) {
  uint32_t s = fmix32(static_cast<uint32_t>(t0) + static_cast<uint32_t>(lane) * 0x9E3779B9u) +
               fmix32(static_cast<uint32_t>(t1) + static_cast<uint32_t>(lane + 32) * 0x9E3779B9u);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__device__ __forceinline__ int key_hash(uint32_t tokens, int parent, int parent_epoch) {
  return static_cast<int>(fmix32(tokens ^ fmix32(static_cast<uint32_t>(parent) * 0x27D4EB2Fu + static_cast<uint32_t>(parent_epoch))));
}

// Index lookup by thread 0: the registered page whose key is (parent, parent_epoch, tok[0 .. 64)) and whose hash is h, else -1.
__device__ int cache_find(const qs_prefix_cache_args& c, int h, int parent, int parent_epoch, const int32_t* tok) {
  const int mask = c.index_size - 1;
  for (int i = h & mask;; i = (i + 1) & mask) {
    const int q = c.index[i];
    if (q < 0) return -1;
    if (c.hash[q] != h || c.key_parent[q] != parent || c.key_epoch[q] != parent_epoch) continue;
    const int4* x = reinterpret_cast<const int4*>(c.key_tokens + static_cast<size_t>(q) * kPageTokens);
    const int4* y = reinterpret_cast<const int4*>(tok);
    bool same = true;
    for (int k = 0; k < kPageTokens / 4 && same; ++k) {
      const int4 u = x[k], v = y[k];
      same = u.x == v.x && u.y == v.y && u.z == v.z && u.w == v.w;
    }
    if (same) return q;
  }
}

__device__ void cache_insert(const qs_prefix_cache_args& c, int q) {
  const int mask = c.index_size - 1;
  int i = c.hash[q] & mask;
  while (c.index[i] >= 0) i = (i + 1) & mask;
  c.index[i] = q;
}

// Backward-shift deletion: every later entry of the probe run that may fill the hole moves into it, so the index never holds tombstones.
__device__ void cache_erase(const qs_prefix_cache_args& c, int q) {
  const int mask = c.index_size - 1;
  int i = c.hash[q] & mask;
  while (c.index[i] != q) i = (i + 1) & mask;
  for (int j = (i + 1) & mask;; j = (j + 1) & mask) {
    const int r = c.index[j];
    if (r < 0) break;
    const int k = c.hash[r] & mask;  // r's home slot: r may move to i unless k lies cyclically in (i, j]
    if (i <= j ? (i < k && k <= j) : (i < k || k <= j)) continue;
    c.index[i] = r;
    i = j;
  }
  c.index[i] = -1;
}

__device__ void lru_push(const qs_prefix_cache_args& c, int* cc, int q) {
  const int t = cc[kLruTail];
  c.lru_prev[q] = t;
  c.lru_next[q] = -1;
  if (t >= 0) c.lru_next[t] = q;
  else cc[kLruHead] = q;
  cc[kLruTail] = q;
  ++cc[kEvictable];
}

__device__ void lru_remove(const qs_prefix_cache_args& c, int* cc, int q) {
  const int pr = c.lru_prev[q], nx = c.lru_next[q];
  if (pr >= 0) c.lru_next[pr] = nx;
  else cc[kLruHead] = nx;
  if (nx >= 0) c.lru_prev[nx] = pr;
  else cc[kLruTail] = pr;
  --cc[kEvictable];
}

// Rule 1 (thread 0): row b's private pages [reg, count) onto the free stack in page order, then its registered pages from the last to the
// first lose a ref, and those at ref 0 join the LRU tail.
__device__ void cache_release(const qs_kv_pool_args& p, const qs_prefix_cache_args& c, int* cc, int b, int count, int* s_reg, int* s_stop,
                              int& top) {
  const int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
  for (int j = s_reg[b]; j < count; ++j) {
    const int q = pg[j];
    p.free_pages[top++] = q;
    c.ref[q] = 0;
    c.state[q] = kPageFree;
  }
  for (int j = s_reg[b] - 1; j >= 0; --j)
    if (--c.ref[pg[j]] == 0) lru_push(c, cc, pg[j]);
  s_reg[b] = s_stop[b] = 0;
}

// Rule 3's page (thread 0): the top of the free stack, else the evicted LRU head; the caller has checked that one exists.
__device__ int cache_take(const qs_kv_pool_args& p, const qs_prefix_cache_args& c, int* cc, int& top) {
  int q;
  if (top > 0) {
    q = p.free_pages[--top];
  } else {
    q = cc[kLruHead];
    lru_remove(c, cc, q);
    cache_erase(c, q);
    ++c.epoch[q];
    --cc[kRegistered];
    ++cc[kEvictions];
  }
  c.ref[q] = 1;
  c.state[q] = kPagePrivate;
  return q;
}

// The youngest row that holds pages and is younger than the requester b of admission rank r, else b (thread 0).
__device__ __forceinline__ int youngest_holder(int r, int b, int n_live, const int* s_order, const int* s_cnt) {
  for (int q = n_live - 1; q > r; --q)
    if (s_cnt[s_order[q]] > 0) return s_order[q];
  return b;
}

// One body for the three schedules: `if constexpr` guards only the state a mode adds, pages and tables (kPool), registration, LRU and match
// (kCache), never a second copy of a rule.
template <bool kPool, bool kCache>
__global__ void __launch_bounds__(kThreads) inflight_schedule_kernel(const qs_inflight_args a, const qs_kv_pool_args p, const qs_prefix_cache_args c) {
  __shared__ int s_phase[kMaxRows];  // phase before this call (after the retire: FREE)
  __shared__ int s_ring[kMaxRows];   // retire: index in the retired ring + 1, else 0
  __shared__ int s_gone[kMaxRows];   // retire: the request the row hands back (row_req is cleared while the block still copies its outputs)
  __shared__ int s_req[kMaxRows];    // admit: the request taken in this call, else -1
  __shared__ int s_adm[kMaxRows];    // admission numbers of the live rows
  __shared__ int s_rem[kMaxRows];    // prompt tokens taken, by admission rank
  __shared__ int s_rank[kMaxRows];
  __shared__ int s_order[kMaxRows];  // the live rows by admission rank
  __shared__ int s_done[kMaxRows];   // prompt tokens cached before this call
  __shared__ int s_tgt[kMaxRows];    // prefill target
  __shared__ int s_cu[kMaxRows + 1];
  constexpr int kPoolRows = kPool ? kMaxRows : 1;
  __shared__ int s_cnt[kPoolRows];   // pool: pages held
  __shared__ int s_keep[kPoolRows];  // pool: leading page-list entries this call leaves as they were
  __shared__ int s_len[kPoolRows];   // pool: seq_lens after the admissions
  constexpr int kCacheRows = kCache ? kMaxRows : 1;
  __shared__ int s_reg[kCacheRows];   // cache: registered leading pages
  __shared__ int s_stop[kCacheRows];  // cache: registration stopped by a duplicate
  __shared__ int s_m[kCacheRows];     // cache: rule 0's end page, then a waiting row's longest match
  __shared__ int s_cc[kCacheCounters];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int B = a.batch, Q = a.queue, H = a.history_len, T = a.max_tokens, C = a.chunk;
  const int tid = threadIdx.x;
  for (int b = tid; b < B; b += kThreads) {
    s_tgt[b] = kPool ? p.target[b] : a.prompt_lens[b];
    if constexpr (kPool) s_cnt[b] = s_keep[b] = p.row_count[b];
    if constexpr (kCache) {
      s_reg[b] = c.reg[b];
      s_stop[b] = c.stop[b];
      const int ph = a.phase[b], cached = ph == kPrefill ? a.done[b] : ph == kDecode ? a.seq_lens[b] - 1 : 0;
      s_m[b] = s_cnt[b] > 0 && !s_stop[b] ? cached / kPageTokens : 0;
    }
  }
  if constexpr (kCache) {
    if (tid < kCacheCounters) s_cc[tid] = c.counters[tid];
  }
  __syncthreads();

  // Thread 0's page steps, in the header's order.  The free-stack top and the pool counters stay in its registers from the retire to the
  // starts.  A page is taken from the free stack, else (cache) from the evicted LRU head; a released row's pages go back to the free stack,
  // or (cache, registered pages) lose a ref and join the LRU at ref 0.
  int top = 0, peak = 0, preempted = 0, started = 0, n_live = 0;
  auto takeable = [&] { return top + (kCache ? s_cc[kEvictable] : 0); };
  auto take = [&](int b) {
    int q;
    if constexpr (kCache) q = cache_take(p, c, s_cc, top);
    else q = p.free_pages[--top];
    p.row_pages[static_cast<size_t>(b) * p.blocks + s_cnt[b]++] = q;
    peak = max(peak, p.pages - takeable());
  };
  auto release = [&](int b) {
    if constexpr (kCache) cache_release(p, c, s_cc, b, s_cnt[b], s_reg, s_stop, top);
    else push_pages(p, b, s_cnt[b], top);
    s_cnt[b] = s_keep[b] = 0;
  };

  if constexpr (kCache) {
    // ---- cache 0, in parallel: the token hashes and key ids of the pages the registration may take, a warp per page ----
    const int warp = tid >> 5, lane = tid & 31;
    for (int b = 0; b < B; ++b) {
      for (int j = s_reg[b] + warp; j < s_m[b]; j += kWarps) {
        const int q = p.row_pages[static_cast<size_t>(b) * p.blocks + j];
        const int64_t* h = a.history + static_cast<size_t>(b) * H + j * kPageTokens;
        const int t0 = static_cast<int>(h[lane]), t1 = static_cast<int>(h[lane + 32]);
        int32_t* kt = c.key_tokens + static_cast<size_t>(q) * kPageTokens;
        kt[lane] = t0;
        kt[lane + 32] = t1;
        const uint32_t th = token_hash(t0, t1, lane);
        if (lane == 0) c.hash[q] = static_cast<int>(th);
      }
    }
    __syncthreads();
  }

  // ---- 1 + 2: retire and admission decisions (thread 0, row order) ----
  if (tid == 0) {
    int retired = a.counters[kRetired];
    int head = a.counters[kHead];
    const int tail = a.counters[kTail];
    int admitted = a.counters[kAdmitted];
    if constexpr (kPool) {
      top = p.counters[0];
      peak = p.counters[1];
      preempted = p.counters[2];
      started = p.counters[3];
    }
    if constexpr (kCache) {
      // 0: register, in row order, the full cached pages past each row's registered ones, until a key is already cached
      for (int b = 0; b < B; ++b) {
        const int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
        for (int j = s_reg[b]; j < s_m[b]; ++j) {
          const int q = pg[j], parent = j > 0 ? pg[j - 1] : -1, pe = j > 0 ? c.epoch[parent] : 0;
          const int key = key_hash(static_cast<uint32_t>(c.hash[q]), parent, pe);
          if (cache_find(c, key, parent, pe, c.key_tokens + static_cast<size_t>(q) * kPageTokens) >= 0) {
            s_stop[b] = 1;
            ++s_cc[kDuplicates];
            break;
          }
          c.state[q] = kPageRegistered;
          ++c.epoch[q];
          c.key_parent[q] = parent;
          c.key_epoch[q] = pe;
          c.hash[q] = key;
          cache_insert(c, q);
          s_reg[b] = j + 1;
          ++s_cc[kRegistrations];
          ++s_cc[kRegistered];
        }
      }
    }
    for (int b = 0; b < B; ++b) {
      int ph = a.phase[b];
      s_ring[b] = 0;
      if (ph == kDecode && a.finished[b]) {
        s_ring[b] = ++retired;
        s_gone[b] = a.row_req[b];
        ph = kFree;
        if constexpr (kPool) release(b);
      }
      s_phase[b] = ph;
      s_req[b] = -1;
      if (a.chunk_budget > 0 && ph == kFree && head < tail) {
        s_req[b] = head++;
        a.adm[b] = admitted++;
      }
    }
    a.counters[kRetired] = retired;
    a.counters[kHead] = head;
    a.counters[kAdmitted] = admitted;
  }
  __syncthreads();

  // ---- 1: retire copies (reads the histories before an admission overwrites them) ----
  for (int b = 0; b < B; ++b) {
    if (s_ring[b] == 0) continue;  // uniform
    const int req = s_gone[b], slot = req % Q;  // not a.row_req[b]: thread 0 clears it below while other warps may still be reading
    const int p = a.prompt_lens[b], L = a.seq_lens[b];
    const int n = min(max(L - p, 0), T);
    const int64_t* h = a.history + static_cast<size_t>(b) * H;
    for (int c = tid; c < n; c += kThreads) {
      a.out_tokens[static_cast<size_t>(slot) * T + c] = h[p + c];
      if (a.out_logprob) a.out_logprob[static_cast<size_t>(slot) * T + c] = a.logprob[static_cast<size_t>(b) * H + p + c];
    }
    if (tid == 0) {
      const int64_t last = L > 0 ? h[L - 1] : -1;
      int reason = kReasonBudget;
      if (last >= 0 && last == a.eos[b]) {
        reason = kReasonEos;
      } else {
        for (int s = 0; s < kStops; ++s)
          if (last >= 0 && last == a.stop[static_cast<size_t>(b) * kStops + s]) reason = kReasonStop;
      }
      a.out_len[slot] = n;
      a.out_reason[slot] = reason;
      a.out_ids[(s_ring[b] - 1) % Q] = req;
      a.phase[b] = kFree;
      a.row_req[b] = -1;
    }
  }
  __syncthreads();

  // ---- 2: admitted rows take their request's prompt and parameters ----
  for (int b = 0; b < B; ++b) {
    const int req = s_req[b];
    if (req < 0) continue;  // uniform
    const int slot = req % Q;
    const int len = a.q_lens[slot];
    const int64_t* src = a.q_prompts + static_cast<size_t>(slot) * a.prompt_cols;
    int64_t* h = a.history + static_cast<size_t>(b) * H;
    for (int c = tid; c < H; c += kThreads) {
      h[c] = c < len ? src[c] : -1;
      if (a.logprob) a.logprob[static_cast<size_t>(b) * H + c] = CUDART_NAN_F;
    }
    if (tid < kStops) a.stop[static_cast<size_t>(b) * kStops + tid] = a.q_stop[static_cast<size_t>(slot) * kStops + tid];
    if (tid == 0) {
      a.prompt_lens[b] = len;
      a.seq_lens[b] = len;
      a.temperature[b] = a.q_temperature[slot];
      a.top_k[b] = a.q_top_k[slot];
      a.top_p[b] = a.q_top_p[slot];
      a.repetition[b] = a.q_repetition[slot];
      a.presence[b] = a.q_presence[slot];
      a.frequency[b] = a.q_frequency[slot];
      a.eos[b] = a.q_eos[slot];
      a.budget[b] = a.q_max_tokens[slot];
      a.offsets[b] = 0;
      a.done[b] = 0;
      a.row_req[b] = req;
      a.phase[b] = kPrefill;
      s_phase[b] = kPrefill;
      s_tgt[b] = len;
    }
  }
  __syncthreads();

  // ---- admission ranks of the live rows and shared copies of done / seq_lens (parallel) ----
  for (int b = tid; b < B; b += kThreads) {
    s_adm[b] = s_phase[b] != kFree ? a.adm[b] : INT_MAX;
    if constexpr (kPool) s_len[b] = a.seq_lens[b];
  }
  __syncthreads();
  for (int b = tid; b < B; b += kThreads) {
    if (s_phase[b] == kFree) continue;
    int r = 0;
    for (int o = 0; o < B; ++o) r += s_adm[o] < s_adm[b];  // admission numbers are distinct
    s_rank[b] = r;
    s_order[r] = b;
    s_done[b] = a.done[b];
  }
  __syncthreads();
  // ---- pool 3: decode growth (thread 0); the victim is the youngest page holder, never older than the requester (which holds pages).  With
  // the cache a victim whose pages are all shared frees none, so the preemptions go on until a page can be taken or the requester was the victim ----
  if (tid == 0) {
    for (int b = 0; b < B; ++b) n_live += s_phase[b] != kFree;
    if constexpr (kPool) {
      for (int r = 0; r < n_live; ++r) {
        const int b = s_order[r];
        if (s_phase[b] != kDecode || s_cnt[b] > (s_len[b] - 1) / kPageTokens) continue;
        bool self = false;
        while (!self && takeable() == 0) {
          const int v = youngest_holder(r, b, n_live, s_order, s_cnt);
          release(v);
          s_done[v] = 0;
          s_tgt[v] = s_len[v];
          s_phase[v] = kPrefill;
          a.phase[v] = kPrefill;
          ++preempted;
          self = v == b;
        }
        if (!self) take(b);
      }
    }
  }
  if constexpr (kCache) {
    __syncthreads();
    // 4, in parallel: every waiting row's longest chain of registered pages matching its history, a warp per row, with full key checks;
    // the pages go to the row's (empty) page list, their number to s_m
    const int warp = tid >> 5, lane = tid & 31, mask = c.index_size - 1;
    for (int b = warp; b < B; b += kWarps) {
      if (s_phase[b] != kPrefill || s_cnt[b] > 0) continue;  // warp-uniform
      const int64_t* h = a.history + static_cast<size_t>(b) * a.history_len;
      int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
      const int most = (s_tgt[b] - 1) / kPageTokens;  // at least one token is computed, so the completing step has a logit
      int parent = -1, pe = 0, m = 0;
      for (; m < most; ++m) {
        const int t0 = static_cast<int>(h[m * kPageTokens + lane]), t1 = static_cast<int>(h[m * kPageTokens + 32 + lane]);
        const int key = key_hash(token_hash(t0, t1, lane), parent, pe);
        int q = -1;
        for (int i = key & mask;; i = (i + 1) & mask) {
          const int r = c.index[i];
          if (r < 0) break;
          const int32_t* kt = c.key_tokens + static_cast<size_t>(r) * kPageTokens;
          if (c.hash[r] == key && c.key_parent[r] == parent && c.key_epoch[r] == pe && __all_sync(0xffffffffu, kt[lane] == t0 && kt[lane + 32] == t1)) {
            q = r;
            break;
          }
        }
        if (q < 0) break;
        if (lane == 0) pg[m] = q;
        parent = q;
        pe = c.epoch[q];
      }
      if (lane == 0) s_m[b] = m;
    }
    __syncthreads();
  }
  if (tid == 0) {
    if constexpr (kPool) {
      // 4: starts, strict first-come-first-served.  With the cache a row reuses its match, cut at the first page an earlier start evicted,
      // and needs e pages fewer to reach: the evictable pages of its match are its own
      for (int r = 0; r < n_live; ++r) {
        const int b = s_order[r];
        if (s_phase[b] != kPrefill || s_cnt[b] > 0) continue;
        const int need = (s_tgt[b] + kPageTokens - 1) / kPageTokens;
        const int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
        int m = 0, e = 0;
        if constexpr (kCache)
          for (; m < s_m[b] && c.state[pg[m]] == kPageRegistered; ++m) e += c.ref[pg[m]] == 0;
        if (takeable() - e < need - m) break;
        if constexpr (kCache) {
          for (int j = 0; j < m; ++j)
            if (c.ref[pg[j]]++ == 0) lru_remove(c, s_cc, pg[j]);
          s_reg[b] = m;
          s_cc[kHitPages] += m;
        }
        s_cnt[b] = m;
        s_done[b] = m * kPageTokens;
        while (s_cnt[b] < need) take(b);  // need > m: the takes also count the matched pages in the peak
        ++started;
      }
      p.counters[0] = top;
      p.counters[1] = peak;
      p.counters[2] = preempted;
      p.counters[3] = started;
    }
    // 5: the chunk budget over the started PREFILL rows in admission order, then the row-order offsets
    int used = 0;
    for (int r = 0; r < n_live; ++r) {
      const int b = s_order[r];
      const int n = s_phase[b] == kPrefill && (!kPool || s_cnt[b] > 0) ? min(s_tgt[b] - s_done[b], a.chunk_budget - used) : 0;
      s_rem[r] = n;
      used += n;
    }
    s_cu[0] = 0;
    for (int b = 0; b < B; ++b) s_cu[b + 1] = s_cu[b] + (s_phase[b] == kPrefill ? s_rem[s_rank[b]] : 0);
  }
  __syncthreads();

  // ---- 3 + 4: the plan and the tail masks, one thread per row ----
  if (tid == 0) a.cu_seqlens[0] = 0;
  for (int b = tid; b < B; b += kThreads) {
    const int ph = s_phase[b];
    const int c = s_cu[b + 1] - s_cu[b];
    a.cu_seqlens[b + 1] = s_cu[b + 1];
    a.chunk_lens[b] = c;
    a.context_lens[b] = ph == kDecode ? a.seq_lens[b] : 0;
    a.tokens[b] = ph == kDecode ? a.tokens_in[b] : 0;
    long long logit = b;
    int fin = ph == kDecode ? 0 : 1;
    if (ph == kPrefill) {
      const int d = s_done[b], len = s_tgt[b];
      a.prefix_lens[b] = d;
      a.done[b] = d + c;
      if (d + c == len) {
        a.phase[b] = kDecode;
        a.start_pos[b] = len;
        logit = B + s_cu[b + 1] - 1;
        fin = 0;
      }
    } else {
      a.prefix_lens[b] = 0;
    }
    a.logit_rows[b] = logit;
    a.finished[b] = fin;
  }
  // chunk token ids in row order (only PREFILL rows take tokens), then the padding slots
  for (int b = 0; b < B; ++b) {
    const int c = s_cu[b + 1] - s_cu[b];
    if (c == 0) continue;  // uniform
    const int d = s_done[b];
    const int64_t* h = a.history + static_cast<size_t>(b) * H;
    for (int j = tid; j < c; j += kThreads) {
      a.tokens[B + s_cu[b] + j] = h[d + j];
      a.padding_offset[s_cu[b] + j] = b * C - s_cu[b];
    }
  }
  for (int t = s_cu[B] + tid; t < C; t += kThreads) {
    a.tokens[B + t] = 0;
    a.padding_offset[t] = C - 1 - t;
  }
  if constexpr (kPool) {
    // ---- pool 6: the new table entries [keep, count) of every row, all layers, K and V (the page lists are visible after the barrier) ----
    const int L = p.layers, nb = p.blocks;
    for (int b = 0; b < B; ++b) {
      const int k0 = s_keep[b], n = (s_cnt[b] - k0) * L * 2;
      if (n <= 0) continue;  // uniform
      const int32_t* pg = p.row_pages + static_cast<size_t>(b) * nb;
      for (int i = tid; i < n; i += kThreads) {
        const int j = k0 + i / (2 * L), l = (i >> 1) % L, kv = i & 1;
        p.tables[((static_cast<size_t>(l) * B + b) * 2 + kv) * nb + j] = p.layer_base[2 * l + kv] + static_cast<long long>(pg[j]) * p.page_bytes;
      }
    }
    for (int b = tid; b < B; b += kThreads) {
      p.row_count[b] = s_cnt[b];
      p.target[b] = s_tgt[b];
      if constexpr (kCache) {
        c.reg[b] = s_reg[b];
        c.stop[b] = s_stop[b];
      }
    }
  }
  if constexpr (kCache) {
    if (tid < kCacheCounters) c.counters[tid] = s_cc[tid];
  }
}

// The argument checks both schedules share.
int check_inflight_args(const qs_inflight_args& a) {
  QS_REQUIRE(a.batch >= 1 && a.batch <= kMaxRows, "inflight_schedule: batch=%d (1 .. %d)", a.batch, kMaxRows);
  QS_REQUIRE(a.queue >= 1 && a.chunk >= 1 && a.max_tokens >= 1 && a.prompt_cols >= 1, "inflight_schedule: queue=%d chunk=%d max_tokens=%d prompt_cols=%d",
             a.queue, a.chunk, a.max_tokens, a.prompt_cols);
  QS_REQUIRE(a.chunk_budget == 0 || a.chunk_budget == a.chunk, "inflight_schedule: chunk_budget=%d must be 0 or the chunk segment (%d)", a.chunk_budget,
             a.chunk);
  QS_REQUIRE(a.history_len >= a.prompt_cols + a.max_tokens, "inflight_schedule: history_len=%d < prompt_cols %d + max_tokens %d", a.history_len,
             a.prompt_cols, a.max_tokens);
  QS_REQUIRE(a.q_prompts && a.q_lens && a.q_max_tokens && a.q_eos && a.q_stop && a.q_temperature && a.q_top_k && a.q_top_p && a.q_repetition &&
                 a.q_presence && a.q_frequency && a.counters && a.phase && a.row_req && a.done && a.adm && a.history && a.prompt_lens &&
                 a.seq_lens && a.temperature && a.top_k && a.top_p && a.repetition && a.presence && a.frequency && a.eos && a.stop && a.budget &&
                 a.offsets && a.finished && a.start_pos && a.tokens_in && a.cu_seqlens && a.prefix_lens && a.chunk_lens && a.padding_offset &&
                 a.context_lens && a.tokens && a.logit_rows && a.out_tokens && a.out_len && a.out_reason && a.out_ids,
             "inflight_schedule: null pointer");
  QS_REQUIRE((a.logprob == nullptr) == (a.out_logprob == nullptr), "inflight_schedule: logprob and out_logprob must both be given or both NULL");
  return 0;
}

// The argument checks of both pool schedules.
int check_pool_args(const qs_inflight_args& a, const qs_kv_pool_args& p) {
  const long long need = (static_cast<long long>(a.prompt_cols) + a.max_tokens + 1 + kPageTokens - 1) / kPageTokens;
  QS_REQUIRE(p.pages >= need && p.blocks >= need, "inflight_schedule_pool: pages=%d blocks=%d (each at least ceil((prompt_cols %d + max_tokens %d + 1) / 64) = %lld)",
             p.pages, p.blocks, a.prompt_cols, a.max_tokens, need);
  QS_REQUIRE(p.layers >= 1 && p.page_bytes >= 1, "inflight_schedule_pool: layers=%d page_bytes=%lld", p.layers, p.page_bytes);
  QS_REQUIRE(p.free_pages && p.counters && p.row_pages && p.row_count && p.target && p.tables && p.layer_base, "inflight_schedule_pool: null pointer");
  return check_inflight_args(a);
}

}  // namespace

int inflight_schedule(const qs_inflight_args& a, void* stream) {
  const int rc = check_inflight_args(a);
  if (rc) return rc;
  return launch(inflight_schedule_kernel<false, false>, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule", a, qs_kv_pool_args{},
                qs_prefix_cache_args{});
}

int inflight_schedule_pool(const qs_inflight_args& a, const qs_kv_pool_args& p, void* stream) {
  const int rc = check_pool_args(a, p);
  if (rc) return rc;
  return launch(inflight_schedule_kernel<true, false>, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule_pool", a, p, qs_prefix_cache_args{});
}

int inflight_schedule_pool_cache(const qs_inflight_args& a, const qs_kv_pool_args& p, const qs_prefix_cache_args& c, void* stream) {
  QS_REQUIRE(c.index_size >= 2 * p.pages && (c.index_size & (c.index_size - 1)) == 0,
             "inflight_schedule_pool_cache: index_size=%d must be a power of two >= 2 pages (%d)", c.index_size, p.pages);
  QS_REQUIRE(c.ref && c.state && c.epoch && c.key_parent && c.key_epoch && c.hash && c.key_tokens && c.lru_prev && c.lru_next && c.index && c.reg &&
                 c.stop && c.counters,
             "inflight_schedule_pool_cache: null pointer");
  const int rc = check_pool_args(a, p);
  if (rc) return rc;
  return launch(inflight_schedule_kernel<true, true>, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule_pool_cache", a, p, c);
}

}  // namespace qs
