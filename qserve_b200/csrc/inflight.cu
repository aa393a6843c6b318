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
enum : int { kFree = 0, kPrefill = 1, kDecode = 2 };
enum : int { kHead = 0, kTail = 1, kRetired = 2, kAdmitted = 3 };
enum : int { kReasonEos = 1, kReasonStop = 2, kReasonBudget = 3 };

__global__ void __launch_bounds__(kThreads) inflight_schedule_kernel(const qs_inflight_args a) {
  __shared__ int s_phase[kMaxRows];  // phase before this call (after the retire: FREE)
  __shared__ int s_ring[kMaxRows];   // retire: index in the retired ring + 1, else 0
  __shared__ int s_gone[kMaxRows];   // retire: the request the row hands back (row_req is cleared while the block still copies its outputs)
  __shared__ int s_req[kMaxRows];    // admit: the request taken in this call, else -1
  __shared__ int s_adm[kMaxRows];    // admission numbers of the PREFILL rows
  __shared__ int s_rem[kMaxRows];    // prompt tokens still to cache, by admission rank, then the tokens taken, by rank
  __shared__ int s_rank[kMaxRows];
  __shared__ int s_done[kMaxRows];   // prompt tokens cached before this call
  __shared__ int s_cu[kMaxRows + 1];
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int B = a.batch, Q = a.queue, H = a.history_len, T = a.max_tokens, C = a.chunk;
  const int tid = threadIdx.x;

  // ---- 1 + 2: retire and admission decisions (thread 0, row order) ----
  if (tid == 0) {
    int retired = a.counters[kRetired];
    int head = a.counters[kHead];
    const int tail = a.counters[kTail];
    int admitted = a.counters[kAdmitted];
    for (int b = 0; b < B; ++b) {
      int ph = a.phase[b];
      s_ring[b] = 0;
      if (ph == kDecode && a.finished[b]) {
        s_ring[b] = ++retired;
        s_gone[b] = a.row_req[b];
        ph = kFree;
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
    }
  }
  __syncthreads();

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
      const int d = s_done[b], len = a.prompt_lens[b];
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
}

}  // namespace

int inflight_schedule(const qs_inflight_args& a, void* stream) {
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
  return launch(inflight_schedule_kernel, dim3(1), dim3(kThreads), 0, 0, stream, "inflight_schedule", a);
}

}  // namespace qs
