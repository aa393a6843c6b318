// qserve_b200 -- the two small steps that follow the verify of a tree of draft tokens (speculative decoding with token trees), sm_90a.
//
// tree_accept_kernel: greedy acceptance.  One warp per sequence, lane j holds draft node j.  Starting at the root (node 0), the walk moves to
// the lowest-index child c of the current node with draft[c] == target[current] until no child matches; the parent of c is the highest set
// bit of its ancestor word below c.  Output: the path length (root included), the path's node indices and the bonus token target[last].
//
// kv_compact_kernel: after acceptance the accepted nodes' K / V sit in the scattered slots P + path[k]; node path[k] has depth k and was
// therefore rotated at position P + k (apply_bias_rope_update_kv_cache_tree).  Copying slot P + path[k] to slot P + k (codes, scale and zero)
// leaves slots P .. P + accept_len - 1 byte-identical to sequential decoding of the accepted tokens.  One warp per (layer, sequence, K / V,
// KV head): it loads every accepted slot into registers first and stores after a __syncwarp, so overlapping moves (path [0, 2, 3]: 2 -> 1,
// 3 -> 2) are safe.  Both kernels are graph-capturable and need no host synchronisation.
#include <type_traits>

#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kMaxNodes = 16;
constexpr int kTokensPerPage = 64;
constexpr int kWarpsPerCta = 4;

__global__ void __launch_bounds__(kWarpsPerCta * 32) tree_accept_kernel(const long long* __restrict__ draft, const int* __restrict__ tree_mask,
                                                                        const long long* __restrict__ target, int* __restrict__ accept_len,
                                                                        int* __restrict__ path, long long* __restrict__ bonus, int batch, int n) {
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();  // the drafts, the mask and the target tokens are produced by the preceding kernels
  const int b = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= batch) return;  // uniform over the warp
  const size_t row = static_cast<size_t>(b) * n;
  const bool node = lane < n;
  const long long d = node ? draft[row + lane] : -1;
  const long long tg = node ? target[row + lane] : -1;
  const uint32_t anc = (node && lane > 0) ? static_cast<uint32_t>(tree_mask[row + lane]) & ((1u << lane) - 1u) : 0u;
  const int parent = anc ? 31 - __clz(anc) : -1;  // the root and parentless nodes are never a child
  int cur = 0, len = 1, my_path = lane == 0 ? 0 : -1;
  long long want = __shfl_sync(0xffffffffu, tg, 0);
  for (;;) {  // every step moves to a higher node index: at most n - 1 steps
    const uint32_t hit = __ballot_sync(0xffffffffu, parent == cur && d == want);
    if (hit == 0u) break;
    cur = __ffs(hit) - 1;  // the lowest index among matching siblings
    if (lane == len) my_path = cur;
    ++len;
    want = __shfl_sync(0xffffffffu, tg, cur);
  }
  if (node) path[row + lane] = my_path;  // -1 past the accepted path
  if (lane == 0) {
    accept_len[b] = len;
    bonus[b] = want;
  }
}

template <int BITS>
__global__ void __launch_bounds__(kWarpsPerCta * 32) kv_compact_kernel(const long long* __restrict__ kv_pointers, const int* __restrict__ start_pos,
                                                                       const int* __restrict__ path, const int* __restrict__ accept_len, int batch,
                                                                       int n, int max_blocks, int num_kv_heads, int code_bytes, long long n_warps) {
  constexpr int kRow = 128 * BITS / 8;  // code bytes of one (token, KV head)
  using Word = typename std::conditional<BITS == 4, uint16_t, uint32_t>::type;  // each lane moves kRow / 32 bytes per slot
  if (threadIdx.x == 0) pdl_launch_dependents();
  const long long w = static_cast<long long>(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_warps) return;  // uniform over the warp
  const int hk = static_cast<int>(w % num_kv_heads);
  long long r = w / num_kv_heads;
  const int kv = static_cast<int>(r & 1);
  r >>= 1;
  const int b = static_cast<int>(r % batch);
  const long long layer = r / batch;
  // host-prepared before the step: the cached length and the (at most two) pages that hold the slots P .. P + n - 1
  const int P = start_pos[b];
  const int blk0 = P / kTokensPerPage;
  const long long* row = kv_pointers + ((layer * batch + b) * 2 + kv) * max_blocks;
  const long long page_l = (lane < 2 && blk0 + lane < max_blocks) ? row[blk0 + lane] : 0;
  pdl_wait();  // path and accept_len come from the acceptance kernel
  const int in_table = min(n, max_blocks * kTokensPerPage - P);  // slots P + s, s < in_table, have a page (the table is not trusted to cover n)
  const int a = min(max(accept_len[b], 0), in_table);
  const int src_l = lane < a ? path[static_cast<size_t>(b) * n + lane] : -1;
  const int zoff = num_kv_heads * kTokensPerPage * 2;  // bytes from the scale row to the zero row
  auto slot_addr = [&](int s, uint8_t*& page, int& slot) {  // all lanes call (shuffle)
    const int pos = P + s;
    const long long pp = __shfl_sync(0xffffffffu, page_l, pos / kTokensPerPage - blk0);
    page = reinterpret_cast<uint8_t*>(pp);
    slot = pos % kTokensPerPage;
  };
  Word code[kMaxNodes];
  __half sc = __float2half(0.f), zp = sc;
  uint32_t moved = 0;  // bit k: slot P + k receives slot P + path[k]
#pragma unroll
  for (int k = 1; k < kMaxNodes; ++k) {  // path[0] = 0: the root never moves
    const int src = __shfl_sync(0xffffffffu, src_l, k);
    if (k < a && src != k && src >= 0 && src < in_table) {
      uint8_t* page;
      int slot;
      slot_addr(src, page, slot);
      code[k] = reinterpret_cast<const Word*>(page + static_cast<size_t>(hk * kTokensPerPage + slot) * kRow)[lane];
      if (lane == k) {
        const __half* meta = reinterpret_cast<const __half*>(page + code_bytes) + hk * kTokensPerPage + slot;
        sc = meta[0];
        zp = meta[zoff / 2];
      }
      moved |= 1u << k;
    }
  }
  __syncwarp();  // every load of the warp is done before any store: sources and destinations may overlap
#pragma unroll
  for (int k = 1; k < kMaxNodes; ++k) {
    if (moved & (1u << k)) {
      uint8_t* page;
      int slot;
      slot_addr(k, page, slot);
      reinterpret_cast<Word*>(page + static_cast<size_t>(hk * kTokensPerPage + slot) * kRow)[lane] = code[k];
      if (lane == k) {
        __half* meta = reinterpret_cast<__half*>(page + code_bytes) + hk * kTokensPerPage + slot;
        meta[0] = sc;
        meta[zoff / 2] = zp;
      }
    }
  }
}

}  // namespace

int tree_accept_greedy(const long long* draft, const int* tree_mask, const long long* target, int* accept_len, int* path, long long* bonus,
                       int batch, int num_nodes, void* stream) {
  QS_REQUIRE(batch >= 0 && num_nodes >= 1 && num_nodes <= kMaxNodes, "tree_accept_greedy: batch=%d, num_nodes=%d (1 .. 16)", batch, num_nodes);
  if (batch == 0) return QS_OK;
  QS_REQUIRE(draft && tree_mask && target && accept_len && path && bonus, "tree_accept_greedy: null pointer");
  return launch(tree_accept_kernel, dim3((batch + kWarpsPerCta - 1) / kWarpsPerCta), dim3(kWarpsPerCta * 32), 0, 0, stream, "tree_accept_greedy", draft,
                tree_mask, target, accept_len, path, bonus, batch, num_nodes);
}

int kv_cache_compact(const KvCompactArgs& a) {
  QS_REQUIRE(a.layers >= 1 && a.batch >= 0 && a.num_nodes >= 1 && a.num_nodes <= kMaxNodes && a.max_blocks >= 1 && a.num_kv_heads >= 1,
             "kv_cache_compact: layers=%d batch=%d num_nodes=%d (1 .. 16) max_blocks=%d kv_heads=%d", a.layers, a.batch, a.num_nodes, a.max_blocks,
             a.num_kv_heads);
  // page geometry only: these ops have no query heads
  const int rc = check_page_geometry("kv_cache_compact", 128, a.num_kv_heads, a.num_kv_heads, a.tokens_per_block, a.size_per_token, a.int4_kv);
  if (rc) return rc;
  if (a.batch == 0) return QS_OK;
  QS_REQUIRE(a.kv_pointers && a.start_pos && a.path && a.accept_len, "kv_cache_compact: null pointer");
  const long long n_warps = static_cast<long long>(a.layers) * a.batch * 2 * a.num_kv_heads;
  const long long ctas = (n_warps + kWarpsPerCta - 1) / kWarpsPerCta;
  QS_REQUIRE(ctas <= 0x7fffffffLL, "kv_cache_compact: grid too large");
  const int code_bytes = kTokensPerPage * a.size_per_token;
  return launch(a.int4_kv ? kv_compact_kernel<4> : kv_compact_kernel<8>, dim3(static_cast<unsigned>(ctas)), dim3(kWarpsPerCta * 32), 0, 0, a.stream,
                "kv_cache_compact", a.kv_pointers, a.start_pos, a.path, a.accept_len, a.batch, a.num_nodes, a.max_blocks, a.num_kv_heads, code_bytes,
                n_warps);
}

}  // namespace qs
