"""Pure-Python restatement of qs_inflight_schedule_pool_cache (include/qserve_b200.h, DESIGN.md 3.12 "Prefix cache"): the pool schedule of
tests/kv_pool_oracle.py with automatic prefix caching.  It keeps the cache's state as the kernel does: per page its ref, state (FREE, PRIVATE,
REGISTERED), epoch and key, the LRU list of the evictable pages (lru[0] is the head, evicted first), the index of registered keys, and per row
reg (its first reg[b] pages are registered and form a key chain) and the stop flag (`halted`).

The key of page j of a row is (parent, parent epoch, history[64 j .. 64 j + 64)), the parent being the row's page j - 1 (with its epoch at the
time) or -1 with epoch 0.  A page's epoch increases when it is registered and when it is evicted.  Rules of one schedule(chunk_budget) call:
  0. Register, over every row that holds pages in row order: cached = done (PREFILL) or seq_len - 1 (DECODE); pages j = reg .. cached // 64 - 1
     in order, unless stopped: a key already in the index stops the row (a duplicate); otherwise the page is registered (epoch + 1, into the
     index) and reg = j + 1.
  1. Retire as KvPoolOracle; a released row (retired or preempted) puts its private pages onto the free stack in page order, then from its
     last registered page to its first decrements ref, and a page at ref 0 joins the LRU tail.  reg = stop = 0.
  2. Admit as KvPoolOracle.
  3. Decode growth as KvPoolOracle, but a page comes from the free stack, else from the evicted LRU head (out of the index, epoch + 1); only
     when neither exists is the youngest page holder preempted, repeatedly until a page can be taken or the requester was the victim.
  4. Starts, strictly first-come-first-served: m = the longest registered chain matching history[0 .. 64 m) with m <= (target - 1) // 64, e =
     how many of its pages are evictable; the row starts when top + evictable - e >= ceil(target / 64) - m, taking the m pages (out of the
     LRU, ref + 1) and the rest as in 3; done = 64 m, reg = m.
  5. and 6. as KvPoolOracle.
The hashes (token_hash, key_hash) are the kernel's, so that a test can probe the device index; the oracle's index is a dict.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

from tests.inflight_oracle import PREFILL
from tests.kv_pool_oracle import PAGE, KvPoolOracle

PAGE_FREE, PAGE_PRIVATE, PAGE_REGISTERED = 0, 1, 2
M32 = 0xFFFFFFFF


def fmix32(x: int) -> int:
    x &= M32
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & M32
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & M32
    x ^= x >> 16
    return x


def token_hash(tokens) -> int:
    return sum(fmix32((int(t) & M32) + i * 0x9E3779B9) for i, t in enumerate(tokens)) & M32


def key_hash(tokens, parent: int, parent_epoch: int) -> int:
    """The index hash of a key (unsigned 32 bits; the device stores it as int32)."""
    return fmix32(token_hash(tokens) ^ fmix32((parent & M32) * 0x27D4EB2F + (parent_epoch & M32)))


Key = Tuple[int, int, Tuple[int, ...]]


class PrefixCacheOracle(KvPoolOracle):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        P, B = self.pages, self.batch
        self.ref, self.state, self.epoch = [0] * P, [PAGE_FREE] * P, [0] * P
        self.key: List[Key] = [None] * P
        self.index: Dict[Key, int] = {}
        self.lru: List[int] = []
        self.reg, self.halted = [0] * B, [0] * B  # halted: the stop flag of the header (self.stop holds the stop ids)
        self.hit_pages = self.registrations = self.evictions = self.duplicates = 0
        self.events.update(multi_victim=0, hit_start=0)

    # ---- what the cache changes in KvPoolOracle's page steps ----
    def _key(self, b: int, j: int) -> Key:
        parent = self.row_pages[b][j - 1] if j else -1
        return (parent, self.epoch[parent] if j else 0, tuple(self.history[b][PAGE * j:PAGE * (j + 1)]))

    def _take(self) -> int:
        if self.free:
            q = self.free.pop()
        else:
            q = self.lru.pop(0)
            del self.index[self.key[q]]
            self.epoch[q] += 1
            self.evictions += 1
        self.ref[q], self.state[q] = 1, PAGE_PRIVATE
        return q

    def _takeable(self, match=()) -> int:
        return len(self.free) + len(self.lru) - sum(self.ref[q] == 0 for q in match)

    def _release(self, b: int) -> None:
        pages, R = self.row_pages[b], self.reg[b]
        for q in pages[R:]:
            self.ref[q], self.state[q] = 0, PAGE_FREE
        for q in reversed(pages[:R]):
            self.ref[q] -= 1
            if self.ref[q] == 0:
                self.lru.append(q)
        self.reg[b] = self.halted[b] = 0
        self.row_pages[b] = pages[R:]  # the private pages go onto the free stack
        super()._release(b)

    def match(self, b: int) -> List[int]:
        """The longest chain of registered pages matching row b's history, at most (target - 1) // 64 pages."""
        out, parent, pe = [], -1, 0
        for j in range((self.target[b] - 1) // PAGE):
            q = self.index.get((parent, pe, tuple(self.history[b][PAGE * j:PAGE * (j + 1)])))
            if q is None:
                break
            out.append(q)
            parent, pe = q, self.epoch[q]
        return out

    def _share(self, b: int, match: List[int]) -> None:
        for q in match:
            if self.ref[q] == 0:
                self.lru.remove(q)
            self.ref[q] += 1
        self.reg[b] = len(match)
        self.hit_pages += len(match)
        self.events["hit_start"] += bool(match)

    def _evictable(self) -> List[int]:
        return self.lru

    def _shared(self, q: int) -> bool:
        return self.state[q] == PAGE_REGISTERED

    def _register(self) -> None:
        for b in range(self.batch):
            if not self.row_pages[b] or self.halted[b]:
                continue
            cached = self.done[b] if self.phase[b] == PREFILL else self.seq_lens[b] - 1
            for j in range(self.reg[b], cached // PAGE):
                k = self._key(b, j)
                if k in self.index:
                    self.halted[b] = 1
                    self.duplicates += 1
                    break
                q = self.row_pages[b][j]
                self.state[q] = PAGE_REGISTERED
                self.epoch[q] += 1
                self.key[q] = k
                self.index[k] = q
                self.reg[b] = j + 1
                self.registrations += 1

    def cache_counters(self) -> List[int]:
        """The device's counters: LRU head, LRU tail, evictable, registered, hit pages, registrations, evictions, duplicates."""
        return [self.lru[0] if self.lru else -1, self.lru[-1] if self.lru else -1, len(self.lru), len(self.index), self.hit_pages,
                self.registrations, self.evictions, self.duplicates]

    def check_cache(self) -> None:
        """Every page is in exactly one of FREE, HELD and EVICTABLE; ref counts page-list occurrences and a private page has ref 1; the index
        holds exactly the registered pages, each key once; every row's first reg pages form its key chain."""
        occ = [0] * self.pages
        for b in range(self.batch):
            for q in self.row_pages[b]:
                occ[q] += 1
        free, lru = set(self.free), set(self.lru)
        assert len(free) == len(self.free) and len(lru) == len(self.lru) and not free & lru
        for q in range(self.pages):
            assert self.ref[q] == occ[q], q
            if q in free:
                assert self.state[q] == PAGE_FREE and occ[q] == 0, q
            elif q in lru:
                assert self.state[q] == PAGE_REGISTERED and occ[q] == 0, q
            else:
                assert occ[q] >= 1 and self.state[q] in (PAGE_PRIVATE, PAGE_REGISTERED), q
                assert self.state[q] == PAGE_REGISTERED or occ[q] == 1, q
        registered = {q for q in range(self.pages) if self.state[q] == PAGE_REGISTERED}
        assert set(self.index.values()) == registered and len(self.index) == len(registered)
        for k, q in self.index.items():
            assert self.key[q] == k
            # the LRU queues a chain's tail before its head, and a held page's parent is held: a parent is never evicted before its children
            assert k[0] < 0 or (self.state[k[0]] == PAGE_REGISTERED and self.epoch[k[0]] == k[1]), q
        for b in range(self.batch):
            pages = self.row_pages[b]
            assert self.reg[b] <= len(pages)
            for j in range(self.reg[b]):
                q = pages[j]
                assert self.state[q] == PAGE_REGISTERED and self.key[q] == self._key(b, j), (b, j)
            for q in pages[self.reg[b]:]:
                assert self.state[q] == PAGE_PRIVATE, (b, q)
