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
// inflight_schedule_kernel<true> adds the shared KV page pool of qs_inflight_schedule_pool: thread 0 also keeps the free stack (retire and
// preemption push, decode growth and starts pop, in the header's order), and the block then writes the new table entries of every layer.
// <false> is the own-pages schedule above, unchanged.
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
constexpr int kPageTokens = 64;
enum : int { kFree = 0, kPrefill = 1, kDecode = 2 };
enum : int { kHead = 0, kTail = 1, kRetired = 2, kAdmitted = 3 };
enum : int { kReasonEos = 1, kReasonStop = 2, kReasonBudget = 3 };

// Pushes row b's pages [0, count) onto the free stack in page order (thread 0).
__device__ __forceinline__ void push_pages(const qs_kv_pool_args& p, int b, int count, int& top) {
  const int32_t* pg = p.row_pages + static_cast<size_t>(b) * p.blocks;
  for (int j = 0; j < count; ++j) p.free_pages[top++] = pg[j];
}

// Pool rules 3-5 (qs_inflight_schedule_pool), called by the whole block after the admissions: admission ranks of every live row and the
// shared copies of seq_lens / done (parallel), then thread 0 runs the decode growth (with preemption), the starts and the chunk budget scan
// over the started rows in admission order, and the row-order offsets.  Ends with a barrier.
__device__ void pool_plan(const qs_inflight_args& a, const qs_kv_pool_args& p, int* s_phase, int* s_adm, int* s_rem, int* s_rank, int* s_done,
                          int* s_cu, int* s_cnt, int* s_keep, int* s_tgt, int* s_len, int* s_order) {
  const int B = a.batch, tid = threadIdx.x;
  for (int b = tid; b < B; b += kThreads) {
    s_adm[b] = s_phase[b] != kFree ? a.adm[b] : INT_MAX;
    s_len[b] = a.seq_lens[b];
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
  if (tid == 0) {
    int n_live = 0;
    for (int b = 0; b < B; ++b) n_live += s_phase[b] != kFree;
    int top = p.counters[0], peak = p.counters[1], preempted = p.counters[2], started = p.counters[3];
    auto pop = [&](int b) {
      p.row_pages[static_cast<size_t>(b) * p.blocks + s_cnt[b]++] = p.free_pages[--top];
      peak = max(peak, p.pages - top);
    };
    // 3: decode growth; the victim is the youngest page holder, never older than the requester (which holds pages)
    for (int r = 0; r < n_live; ++r) {
      const int b = s_order[r];
      if (s_phase[b] != kDecode || s_cnt[b] > (s_len[b] - 1) / kPageTokens) continue;
      if (top == 0) {
        int v = b;
        for (int q = n_live - 1; q > r; --q)
          if (s_cnt[s_order[q]] > 0) {
            v = s_order[q];
            break;
          }
        push_pages(p, v, s_cnt[v], top);
        s_cnt[v] = s_keep[v] = s_done[v] = 0;
        s_tgt[v] = s_len[v];
        s_phase[v] = kPrefill;
        a.phase[v] = kPrefill;
        ++preempted;
        if (v == b) continue;
      }
      pop(b);
    }
    // 4: starts, strict first-come-first-served
    for (int r = 0; r < n_live; ++r) {
      const int b = s_order[r];
      if (s_phase[b] != kPrefill || s_cnt[b] > 0) continue;
      const int need = (s_tgt[b] + kPageTokens - 1) / kPageTokens;
      if (need > top) break;
      while (s_cnt[b] < need) pop(b);
      ++started;
    }
    // 5: the chunk budget over the started rows in admission order, then the row-order offsets
    int used = 0;
    for (int r = 0; r < n_live; ++r) {
      const int b = s_order[r];
      const int take = s_phase[b] == kPrefill && s_cnt[b] > 0 ? min(s_tgt[b] - s_done[b], a.chunk_budget - used) : 0;
      s_rem[r] = take;
      used += take;
    }
    s_cu[0] = 0;
    for (int b = 0; b < B; ++b) s_cu[b + 1] = s_cu[b] + (s_phase[b] == kPrefill ? s_rem[s_rank[b]] : 0);
    p.counters[0] = top;
    p.counters[1] = peak;
    p.counters[2] = preempted;
    p.counters[3] = started;
  }
  __syncthreads();
}

template <bool kPool>
__global__ void __launch_bounds__(kThreads) inflight_schedule_kernel(const qs_inflight_args a, const qs_kv_pool_args p) {
  __shared__ int s_phase[kMaxRows];  // phase before this call (after the retire: FREE)
  __shared__ int s_ring[kMaxRows];   // retire: index in the retired ring + 1, else 0
  __shared__ int s_gone[kMaxRows];   // retire: the request the row hands back (row_req is cleared while the block still copies its outputs)
  __shared__ int s_req[kMaxRows];    // admit: the request taken in this call, else -1
  __shared__ int s_adm[kMaxRows];    // admission numbers of the PREFILL rows (pool: of every live row)
  __shared__ int s_rem[kMaxRows];    // prompt tokens still to cache, by admission rank, then the tokens taken, by rank
  __shared__ int s_rank[kMaxRows];
  __shared__ int s_done[kMaxRows];   // prompt tokens cached before this call
  __shared__ int s_cu[kMaxRows + 1];
  constexpr int kPoolRows = kPool ? kMaxRows : 1;
  __shared__ int s_cnt[kPoolRows];    // pool: pages held
  __shared__ int s_keep[kPoolRows];   // pool: leading page-list entries this call leaves as they were
  __shared__ int s_tgt[kPoolRows];    // pool: prefill target
  __shared__ int s_len[kPoolRows];    // pool: seq_lens after the admissions
  __shared__ int s_order[kPoolRows];  // pool: the live rows by admission rank
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int B = a.batch, Q = a.queue, H = a.history_len, T = a.max_tokens, C = a.chunk;
  const int tid = threadIdx.x;
  if constexpr (kPool) {
    for (int b = tid; b < B; b += kThreads) {
      s_cnt[b] = s_keep[b] = p.row_count[b];
      s_tgt[b] = p.target[b];
    }
    __syncthreads();
  }

  // ---- 1 + 2: retire and admission decisions (thread 0, row order) ----
  if (tid == 0) {
    int retired = a.counters[kRetired];
    int head = a.counters[kHead];
    const int tail = a.counters[kTail];
    int admitted = a.counters[kAdmitted];
    int top = kPool ? p.counters[0] : 0;
    for (int b = 0; b < B; ++b) {
      int ph = a.phase[b];
      s_ring[b] = 0;
      if (ph == kDecode && a.finished[b]) {
        s_ring[b] = ++retired;
        s_gone[b] = a.row_req[b];
        ph = kFree;
        if constexpr (kPool) {
          push_pages(p, b, s_cnt[b], top);
          s_cnt[b] = s_keep[b] = 0;
        }
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
    if constexpr (kPool) p.counters[0] = top;
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
      if constexpr (kPool) s_tgt[b] = len;
    }
  }
  __syncthreads();

  if constexpr (kPool) {
    pool_plan(a, p, s_phase, s_adm, s_rem, s_rank, s_done, s_cu, s_cnt, s_keep, s_tgt, s_len, s_order);
  } else {
    // ---- 3: admission ranks of the PREFILL rows (parallel), the budget scan in admission order and the row-order offsets (thread 0) ----
    for (int b = tid; b < B; b += kThreads) s_adm[b] = s_phase[b] == kPrefill ? a.adm[b] : INT_MAX;
    __syncthreads();
    for (int b = tid; b < B; b += kThreads) {
      if (s_phase[b] != kPrefill) continue;
      int r = 0;
      for (int o = 0; o < B; ++o) r += s_adm[o] < s_adm[b];  // admission numbers are distinct
      s_rank[b] = r;
      s_done[b] = a.done[b];
      s_rem[r] = a.prompt_lens[b] - s_done[b];
    }
    __syncthreads();
    if (tid == 0) {
      int n_pre = 0;
      for (int b = 0; b < B; ++b) n_pre += s_phase[b] == kPrefill;
      int used = 0;
      for (int r = 0; r < n_pre; ++r) {
        const int take = min(s_rem[r], a.chunk_budget - used);
        s_rem[r] = take;
        used += take;
      }
      s_cu[0] = 0;
      for (int b = 0; b < B; ++b) s_cu[b + 1] = s_cu[b] + (s_phase[b] == kPrefill ? s_rem[s_rank[b]] : 0);
    }
    __syncthreads();
  }

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
      const int d = s_done[b], len = kPool ? s_tgt[b] : a.prompt_lens[b];
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
    // ---- pool 6: the new table entries [keep, count) of every row, all layers, K and V (pool_plan's page lists are visible after its barrier) ----
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
    }
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

}  // namespace

int inflight_schedule(const qs_inflight_args& a, void* stream) {
  const int rc = check_inflight_args(a);
  if (rc) return rc;
  return launch(inflight_schedule_kernel<false>, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule", a, qs_kv_pool_args{});
}

int inflight_schedule_pool(const qs_inflight_args& a, const qs_kv_pool_args& p, void* stream) {
  const long long need = (static_cast<long long>(a.prompt_cols) + a.max_tokens + 1 + kPageTokens - 1) / kPageTokens;
  QS_REQUIRE(p.pages >= need && p.blocks >= need, "inflight_schedule_pool: pages=%d blocks=%d (each at least ceil((prompt_cols %d + max_tokens %d + 1) / 64) = %lld)",
             p.pages, p.blocks, a.prompt_cols, a.max_tokens, need);
  QS_REQUIRE(p.layers >= 1 && p.page_bytes >= 1, "inflight_schedule_pool: layers=%d page_bytes=%lld", p.layers, p.page_bytes);
  QS_REQUIRE(p.free_pages && p.counters && p.row_pages && p.row_count && p.target && p.tables && p.layer_base, "inflight_schedule_pool: null pointer");
  const int rc = check_inflight_args(a);
  if (rc) return rc;
  return launch(inflight_schedule_kernel<true>, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule_pool", a, p);
}

}  // namespace qs
