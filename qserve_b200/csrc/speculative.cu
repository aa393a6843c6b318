// qserve_b200 -- the two ends of a speculative-decoding step, sm_90a: the prompt-lookup drafter and the commit of what was accepted.
//
// ngram_propose_kernel: prompt lookup (n-gram drafting).  One CTA per sequence.  The key is the last n_max ids of the row's history; every
// earlier position j whose backward window matches the key's last m >= n_min ids is a candidate, ranked by (m descending, j descending).
// Each thread scans the positions tid, tid + kThreads, ... (coalesced int64 loads; most positions fail on the first compare), keeps its best
// kMaxBranches candidates as packed keys (m << 16 | j) in registers, and `branches` rounds of a block-wide max merge them in rank order
// (keys are distinct, so the merge is exact and needs no atomics).  Warp 0 then inserts the candidates' continuations into a trie below the
// root: lane i holds node i, a ballot finds an existing child, and the lane with the next free index takes a new node.  The same warp writes
// the tokens and the ancestor words; uncreated nodes are padding (token -1, mask 1).  The output is bitwise deterministic.
//
// spec_commit_kernel: one thread per sequence appends draft[path[1 .. acc - 1]] and the bonus token to the history, cut after the first eos
// and at the row's budget, and writes the positions the next step reads (start_pos, context_lens, roots).  spec_commit_stops_kernel cuts
// after the first token of {eos} and the row's stop set instead.  Every kernel reads every input after the PDL dependency wait: the previous
// step's commit writes the history and the lengths.  All are CUDA-graph capturable.
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxNodes = 16;
constexpr int kMaxBranches = 8;
constexpr int kMaxNgram = 8;
constexpr int kMaxHistory = 32768;  // j < 2^15: a candidate packs into (m << 16) | j
constexpr int kCommitThreads = 128;
constexpr int kMaxStops = 8;  // stop tokens per row besides eos

__device__ __forceinline__ int block_max(int v, int* red) {  // every thread calls; returns the block-wide maximum to all
  v = __reduce_max_sync(0xffffffffu, v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < kWarps ? red[lane] : 0;
  v = __reduce_max_sync(0xffffffffu, v);
  __syncthreads();  // red is reused by the next call
  return v;
}

__global__ void __launch_bounds__(kThreads) ngram_propose_kernel(const long long* __restrict__ history, const int* __restrict__ seq_lens,
                                                                 long long* __restrict__ tokens, int* __restrict__ tree_mask, int hist_len,
                                                                 int n, int n_min, int n_max, int branches) {
  __shared__ long long key[kMaxNgram];  // key[i] = h[L - 1 - i], -1 past the history's start
  __shared__ int red[kWarps];
  __shared__ int cand[kMaxBranches];  // packed (m << 16) | j in rank order, 0: none
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // the previous step's commit writes the history and the lengths
  const int b = blockIdx.x;
  const long long* h = history + static_cast<size_t>(b) * hist_len;
  const int L = min(max(seq_lens[b], 0), hist_len);
  if (threadIdx.x < kMaxNgram) key[threadIdx.x] = threadIdx.x < L ? h[L - 1 - threadIdx.x] : -1;
  __syncthreads();

  // ---- scan: the best kMaxBranches candidates of this thread, sorted descending ----
  int best[kMaxBranches];
#pragma unroll
  for (int s = 0; s < kMaxBranches; ++s) best[s] = 0;
  const long long k0 = key[0];
  if (n > 1 && k0 >= 0) {
    for (int j = threadIdx.x; j <= L - 2; j += kThreads) {
      if (h[j] != k0) continue;
      const int gmax = min(n_max, j + 1);
      int m = 1;
      while (m < gmax) {
        const long long kk = key[m];
        if (kk < 0 || h[j - m] != kk) break;
        ++m;
      }
      if (m < n_min) continue;
      int c = (m << 16) | j;
#pragma unroll
      for (int s = 0; s < kMaxBranches; ++s) {  // branch-free insertion keeps best[] in registers
        const int hi = max(best[s], c);
        c = min(best[s], c);
        best[s] = hi;
      }
    }
  }

  // ---- merge: `branches` rounds of a block max; the owner of the winner pops it ----
  for (int r = 0; r < branches; ++r) {
    const int w = block_max(best[0], red);
    if (threadIdx.x == 0) cand[r] = w;
    if (w != 0 && best[0] == w) {
#pragma unroll
      for (int s = 0; s + 1 < kMaxBranches; ++s) best[s] = best[s + 1];
      best[kMaxBranches - 1] = 0;
    }
  }
  __syncthreads();
  if (threadIdx.x >= 32) return;

  // ---- trie: warp 0, lane i holds node i ----
  const int lane = threadIdx.x;
  long long tok = lane == 0 ? k0 : -1;
  int parent = -1, mask = lane == 0 ? 0 : 1;
  int cnt = 1;  // nodes created, root included
  for (int r = 0; r < branches && cnt < n; ++r) {
    const int c = cand[r];
    if (c == 0) break;
    const int j = c & 0xffff;
    const int clen = min(n - 1, L - 1 - j);
    const long long cont = lane < clen ? h[j + 1 + lane] : -1;  // the continuation, one token per lane
    int cur = 0;
    for (int k = 0; k < clen; ++k) {
      const long long t = __shfl_sync(0xffffffffu, cont, k);
      const uint32_t hit = __ballot_sync(0xffffffffu, lane > 0 && lane < cnt && parent == cur && tok == t);
      if (hit) {
        cur = __ffs(hit) - 1;
        continue;
      }
      if (cnt == n) break;  // the node budget is spent: no later candidate can add a node either
      const int pmask = __shfl_sync(0xffffffffu, mask, cur);
      if (lane == cnt) {
        tok = t;
        parent = cur;
        mask = pmask | (1 << cur);
      }
      cur = cnt++;
    }
  }
  if (lane < n) {
    tokens[static_cast<size_t>(b) * n + lane] = tok;
    tree_mask[static_cast<size_t>(b) * n + lane] = mask;
  }
}

__global__ void __launch_bounds__(kCommitThreads) spec_commit_kernel(const long long* __restrict__ draft, const int* __restrict__ path,
                                                                     const int* __restrict__ accept_len, const long long* __restrict__ bonus,
                                                                     long long* __restrict__ history, int* __restrict__ seq_lens,
                                                                     const int* __restrict__ prompt_lens, const int* __restrict__ budget,
                                                                     const long long* __restrict__ eos, int* __restrict__ finished,
                                                                     int* __restrict__ start_pos, int* __restrict__ context_lens,
                                                                     long long* __restrict__ roots, int batch, int n, int hist_len) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // the acceptance outputs come from the kernels before; the lengths from the previous step
  const int b = blockIdx.x * kCommitThreads + threadIdx.x;
  if (b >= batch || finished[b]) return;
  long long* h = history + static_cast<size_t>(b) * hist_len;
  const int L = min(max(seq_lens[b], 0), hist_len);
  const int acc = min(max(accept_len[b], 1), n);
  const long long e = eos[b];
  const size_t row = static_cast<size_t>(b) * n;
  long long app[kMaxNodes];  // the accepted drafts after the root, then the bonus token
  int count = acc;
  bool hit_eos = false;
#pragma unroll
  for (int k = 0; k < kMaxNodes; ++k) {
    if (k < acc) {
      app[k] = k + 1 < acc ? draft[row + min(max(path[row + k + 1], 0), n - 1)] : bonus[b];
      if (!hit_eos && e >= 0 && app[k] == e) {
        hit_eos = true;
        count = k + 1;
      }
    }
  }
  const int room = max(budget[b] - (L - prompt_lens[b]), 0);
  if (count > room) {
    count = room;
    hit_eos = false;  // the eos fell behind the budget cut
  }
  long long last = L > 0 ? h[L - 1] : -1;
#pragma unroll
  for (int k = 0; k < kMaxNodes; ++k) {
    if (k < count) {
      if (L + k < hist_len) h[L + k] = app[k];
      last = app[k];
    }
  }
  const int L2 = L + count;
  seq_lens[b] = L2;
  start_pos[b] = L2 - 1;
  if (context_lens) context_lens[b] = L2;
  if (roots) roots[b] = last;
  if (hit_eos || L2 - prompt_lens[b] >= budget[b]) finished[b] = 1;
}

// spec_commit_kernel with a per-row stop-token set stop_ids [batch, num_stops] (num_stops <= kMaxStops, -1 pads): the first emitted token
// in {eos} and the set ends the row as eos does
__global__ void __launch_bounds__(kCommitThreads) spec_commit_stops_kernel(const long long* __restrict__ draft, const int* __restrict__ path,
                                                                           const int* __restrict__ accept_len, const long long* __restrict__ bonus,
                                                                           long long* __restrict__ history, int* __restrict__ seq_lens,
                                                                           const int* __restrict__ prompt_lens, const int* __restrict__ budget,
                                                                           const long long* __restrict__ eos, const long long* __restrict__ stop_ids,
                                                                           int* __restrict__ finished, int* __restrict__ start_pos,
                                                                           int* __restrict__ context_lens, long long* __restrict__ roots, int batch, int n,
                                                                           int hist_len, int num_stops) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // the acceptance outputs come from the kernels before; the lengths from the previous step
  const int b = blockIdx.x * kCommitThreads + threadIdx.x;
  if (b >= batch || finished[b]) return;
  long long stops[kMaxStops];
#pragma unroll
  for (int s = 0; s < kMaxStops; ++s) stops[s] = s < num_stops ? stop_ids[static_cast<size_t>(b) * num_stops + s] : -1;
  long long* h = history + static_cast<size_t>(b) * hist_len;
  const int L = min(max(seq_lens[b], 0), hist_len);
  const int acc = min(max(accept_len[b], 1), n);
  const long long e = eos[b];
  const size_t row = static_cast<size_t>(b) * n;
  long long app[kMaxNodes];  // the accepted drafts after the root, then the bonus token
  int count = acc;
  bool hit_stop = false;
#pragma unroll
  for (int k = 0; k < kMaxNodes; ++k) {
    if (k < acc) {
      app[k] = k + 1 < acc ? draft[row + min(max(path[row + k + 1], 0), n - 1)] : bonus[b];
      bool stop = e >= 0 && app[k] == e;
#pragma unroll
      for (int s = 0; s < kMaxStops; ++s) stop |= stops[s] >= 0 && app[k] == stops[s];
      if (!hit_stop && stop) {
        hit_stop = true;
        count = k + 1;
      }
    }
  }
  const int room = max(budget[b] - (L - prompt_lens[b]), 0);
  if (count > room) {
    count = room;
    hit_stop = false;  // the stop token fell behind the budget cut
  }
  long long last = L > 0 ? h[L - 1] : -1;
#pragma unroll
  for (int k = 0; k < kMaxNodes; ++k) {
    if (k < count) {
      if (L + k < hist_len) h[L + k] = app[k];
      last = app[k];
    }
  }
  const int L2 = L + count;
  seq_lens[b] = L2;
  start_pos[b] = L2 - 1;
  if (context_lens) context_lens[b] = L2;
  if (roots) roots[b] = last;
  if (hit_stop || L2 - prompt_lens[b] >= budget[b]) finished[b] = 1;
}

}  // namespace

int ngram_propose(const NgramProposeArgs& a) {
  QS_REQUIRE(a.batch >= 0 && a.history_len >= 1 && a.history_len <= kMaxHistory, "ngram_propose: batch=%d history_len=%d (1 .. %d)", a.batch,
             a.history_len, kMaxHistory);
  QS_REQUIRE(a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "ngram_propose: num_nodes=%d (1 .. %d)", a.num_nodes, kMaxNodes);
  QS_REQUIRE(a.n_min >= 1 && a.n_min <= a.n_max && a.n_max <= kMaxNgram, "ngram_propose: n_min=%d n_max=%d (1 <= n_min <= n_max <= %d)", a.n_min,
             a.n_max, kMaxNgram);
  QS_REQUIRE(a.branches >= 1 && a.branches <= kMaxBranches, "ngram_propose: branches=%d (1 .. %d)", a.branches, kMaxBranches);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.history && a.seq_lens && a.tokens && a.tree_mask, "ngram_propose: null pointer");
  return launch(ngram_propose_kernel, dim3(a.batch), dim3(kThreads), 0, 0, a.stream, "ngram_propose", a.history, a.seq_lens, a.tokens, a.tree_mask,
                a.history_len, a.num_nodes, a.n_min, a.n_max, a.branches);
}

int spec_commit(const SpecCommitArgs& a) {
  QS_REQUIRE(a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "spec_commit: batch=%d num_nodes=%d (1 .. %d)", a.batch, a.num_nodes,
             kMaxNodes);
  QS_REQUIRE(a.history_len >= 1, "spec_commit: history_len=%d", a.history_len);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.draft && a.path && a.accept_len && a.bonus && a.history && a.seq_lens && a.prompt_lens && a.budget && a.eos && a.finished && a.start_pos,
             "spec_commit: null pointer");
  return launch(spec_commit_kernel, dim3((a.batch + kCommitThreads - 1) / kCommitThreads), dim3(kCommitThreads), 0, 0, a.stream, "spec_commit", a.draft,
                a.path, a.accept_len, a.bonus, a.history, a.seq_lens, a.prompt_lens, a.budget, a.eos, a.finished, a.start_pos, a.context_lens, a.roots,
                a.batch, a.num_nodes, a.history_len);
}

int spec_commit_stops(const SpecCommitArgs& a, const long long* stop_ids, int num_stops) {
  QS_REQUIRE(a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes, "spec_commit_stops: batch=%d num_nodes=%d (1 .. %d)", a.batch,
             a.num_nodes, kMaxNodes);
  QS_REQUIRE(a.history_len >= 1, "spec_commit_stops: history_len=%d", a.history_len);
  QS_REQUIRE(num_stops >= 0 && num_stops <= kMaxStops, "spec_commit_stops: num_stops=%d (0 .. %d)", num_stops, kMaxStops);
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.draft && a.path && a.accept_len && a.bonus && a.history && a.seq_lens && a.prompt_lens && a.budget && a.eos && a.finished && a.start_pos &&
                 (stop_ids || num_stops == 0),
             "spec_commit_stops: null pointer");
  return launch(spec_commit_stops_kernel, dim3((a.batch + kCommitThreads - 1) / kCommitThreads), dim3(kCommitThreads), 0, 0, a.stream,
                "spec_commit_stops", a.draft, a.path, a.accept_len, a.bonus, a.history, a.seq_lens, a.prompt_lens, a.budget, a.eos, stop_ids,
                a.finished, a.start_pos, a.context_lens, a.roots, a.batch, a.num_nodes, a.history_len, num_stops);
}

}  // namespace qs
