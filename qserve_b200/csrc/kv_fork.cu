// qserve_b200 -- copy-on-write fork of a cached prompt into other sequences (SamplingParams.n / best_of), sm_90a.
//
// A prompt of P tokens is prefilled once; each of its n rows then shares the parent's full pages 0 .. P / 64 - 1 (the child's block-table
// entries point at them, set by the caller) and gets a private copy of the partial tail page, block P / 64, because the child appends its own
// tokens to that page.  kv_fork_kernel makes those copies: one CTA per (pair, K / V, layer) copies slots 0 .. P % 64 - 1 of the parent's tail
// page into the child's own page at the same block index.  In the page layout ([Hkv][64][128 * bits / 8] codes, then the scale rows [Hkv][64]
// and the zero rows [Hkv][64], fp16) the codes of those slots are one contiguous run of (P % 64) * 128 * bits / 8 bytes per KV head, a
// multiple of 16, moved as 16-byte vectors; the scale and zero of each slot are moved as halves.  Pages and lengths are written by the kernels
// before it, so the kernel reads everything after the dependency wait.
#include "common.cuh"
#include "launch.cuh"

namespace qs {
namespace {

constexpr int kTokensPerPage = 64;
constexpr int kThreads = 256;

template <int BITS>
__global__ void __launch_bounds__(kThreads) kv_fork_kernel(const long long* __restrict__ kv_pointers, const int* __restrict__ parents,
                                                           const int* __restrict__ children, const int* __restrict__ lens, int batch,
                                                           int max_blocks, int num_kv_heads, int code_bytes) {
  constexpr int kRow = 128 * BITS / 8;  // code bytes of one (token, KV head)
  if (threadIdx.x == 0) pdl_launch_dependents();
  pdl_wait();
  const int pair = blockIdx.x >> 1, kv = blockIdx.x & 1;
  const long long layer = blockIdx.y;
  const int pb = parents[pair], cb = children[pair];
  const int P = lens[pb];
  const int t = P % kTokensPerPage, blk = P / kTokensPerPage;
  if (P <= 0 || t == 0 || blk >= max_blocks) return;  // no partial tail page (or none in the table): nothing to copy
  const long long* table = kv_pointers + layer * batch * 2 * max_blocks;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(table[(static_cast<long long>(pb) * 2 + kv) * max_blocks + blk]);
  uint8_t* dst = reinterpret_cast<uint8_t*>(table[(static_cast<long long>(cb) * 2 + kv) * max_blocks + blk]);
  const int run = t * kRow / 16;  // 16-byte vectors of one KV head's slots 0 .. t - 1
  for (int i = threadIdx.x; i < num_kv_heads * run; i += kThreads) {
    const int h = i / run;
    const size_t off = static_cast<size_t>(h) * kTokensPerPage * kRow + static_cast<size_t>(i - h * run) * 16;
    *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(src + off);
  }
  const __half* ms = reinterpret_cast<const __half*>(src + code_bytes);  // [2][Hkv][64]: scale rows, then zero rows
  __half* md = reinterpret_cast<__half*>(dst + code_bytes);
  for (int i = threadIdx.x; i < 2 * num_kv_heads * t; i += kThreads) {
    const int row = i / t;
    md[row * kTokensPerPage + i - row * t] = ms[row * kTokensPerPage + i - row * t];
  }
}

}  // namespace

int kv_cache_fork(const KvForkArgs& a) {
  QS_REQUIRE(a.layers >= 1 && a.layers <= 65535 && a.batch >= 0 && a.num_pairs >= 0 && a.max_blocks >= 1 && a.num_kv_heads >= 1,
             "kv_cache_fork: layers=%d (1 .. 65535) batch=%d num_pairs=%d max_blocks=%d kv_heads=%d", a.layers, a.batch, a.num_pairs, a.max_blocks,
             a.num_kv_heads);
  QS_REQUIRE(a.num_pairs <= 0x3fffffff, "kv_cache_fork: num_pairs=%d too large", a.num_pairs);
  QS_REQUIRE(a.tokens_per_block == kTokensPerPage, "kv_cache_fork: tokens_per_block=%d, only 64 is supported", a.tokens_per_block);
  const int bits = a.int4_kv ? 4 : 8;
  QS_REQUIRE(a.size_per_token == a.num_kv_heads * 128 * bits / 8, "kv_cache_fork: size_per_token=%d does not match %d kv heads x %d bits",
             a.size_per_token, a.num_kv_heads, bits);
  if (a.batch == 0 || a.num_pairs == 0) return QS_OK;
  QS_REQUIRE(a.kv_pointers && a.parents && a.children && a.lens, "kv_cache_fork: null pointer");
  const int code_bytes = kTokensPerPage * a.size_per_token;
  return launch(a.int4_kv ? kv_fork_kernel<4> : kv_fork_kernel<8>, dim3(static_cast<unsigned>(a.num_pairs) * 2u, static_cast<unsigned>(a.layers)),
                dim3(kThreads), 0, 0, a.stream, "kv_cache_fork", a.kv_pointers, a.parents, a.children, a.lens, a.batch, a.max_blocks, a.num_kv_heads,
                code_bytes);
}

}  // namespace qs
