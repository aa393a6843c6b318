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

from tests.inflight_oracle import BUDGET, DECODE, EOS, FREE, MAX_STOPS, PREFILL, STOP, Plan
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

    # ---- page helpers ----
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

    def _pop(self, b: int) -> None:
        self.row_pages[b].append(self._take())
        self.peak = max(self.peak, self.held_pages())

    def _release(self, b: int) -> None:
        pages, R = self.row_pages[b], self.reg[b]
        for q in pages[R:]:
            self.free.append(q)
            self.ref[q], self.state[q] = 0, PAGE_FREE
        for q in reversed(pages[:R]):
            self.ref[q] -= 1
            if self.ref[q] == 0:
                self.lru.append(q)
        self.row_pages[b] = []
        self.reg[b] = self.halted[b] = 0

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

    def held_pages(self) -> int:
        return self.pages - len(self.free) - len(self.lru)

    # ---- rules 1, 2, 5 and 6 of KvPoolOracle.schedule, unchanged ----
    def _retire(self, b: int) -> None:
        r, p, L = self.row_req[b], self.prompt_lens[b], self.seq_lens[b]
        last = self.history[b][L - 1] if L > 0 else -1
        reason = BUDGET
        if last >= 0 and last == self.eos[b]:
            reason = EOS
        elif last >= 0 and last in self.stop[b]:
            reason = STOP
        assert r not in self.outputs, f"request {r} retired twice"
        self.outputs[r] = (list(self.history[b][p:L]), reason)
        self.ring.append(r)
        self.retired += 1
        self.phase[b], self.row_req[b] = FREE, -1

    def _admit(self, chunk_budget: int) -> None:
        if chunk_budget <= 0:
            return
        for b in range(self.batch):
            if self.phase[b] == FREE and self.head < self.tail:
                r = self.head
                self.head += 1
                q = self.requests[r]
                n = len(q.prompt)
                self.history[b] = list(q.prompt)
                self.prompt_lens[b] = self.seq_lens[b] = self.target[b] = n
                self.eos[b] = q.eos
                self.stop[b] = tuple(q.stop) + (-1,) * (MAX_STOPS - len(q.stop))
                self.budget[b] = q.max_tokens
                self.done[b] = 0
                self.adm[b] = self.admitted
                self.admitted += 1
                self.row_req[b] = r
                self.phase[b] = PREFILL

    def _plan(self, chunk_budget: int, order: List[int], keep: List[int]) -> Plan:
        B, C = self.batch, self.chunk
        take, used = [0] * B, 0
        for b in order:
            if self.phase[b] == PREFILL and self.row_pages[b]:
                take[b] = min(self.target[b] - self.done[b], chunk_budget - used)
                used += take[b]
        cu = [0]
        for b in range(B):
            cu.append(cu[-1] + take[b])
        tokens = [self.tokens_in[b] if self.phase[b] == DECODE else 0 for b in range(B)] + [0] * C
        pad = [C - 1 - t for t in range(C)]
        for b in range(B):
            for j in range(take[b]):
                tokens[B + cu[b] + j] = self.history[b][self.done[b] + j]
                pad[cu[b] + j] = b * C - cu[b]
        plan = Plan(cu, take, [self.done[b] if self.phase[b] == PREFILL else 0 for b in range(B)],
                    [self.seq_lens[b] if self.phase[b] == DECODE else 0 for b in range(B)], tokens, pad, list(range(B)), used)
        for b in range(B):
            if self.phase[b] == PREFILL:
                self.done[b] += take[b]
                if self.done[b] == self.target[b]:
                    self.phase[b] = DECODE
                    self.start_pos[b] = self.target[b]
                    plan.logit_rows[b] = B + cu[b + 1] - 1
                    self.finished[b] = 0
                else:
                    self.finished[b] = 1
            elif self.phase[b] == DECODE:
                self.finished[b] = 0
            else:
                self.finished[b] = 1
        for b in range(B):
            for j in range(keep[b], len(self.row_pages[b])):
                for li in range(self.layers):
                    for kv in range(2):
                        self.tables[(li, b, kv, j)] = self.row_pages[b][j]
        return plan

    # ---- one schedule call ----
    def schedule(self, chunk_budget: int) -> Plan:
        B = self.batch
        keep = [len(p) for p in self.row_pages]
        # 0. register
        for b in range(B):
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
        # 1. retire
        for b in range(B):
            if self.phase[b] == DECODE and self.finished[b]:
                self._retire(b)
                self._release(b)
                keep[b] = 0
        # 2. admit
        self._admit(chunk_budget)
        order = sorted((b for b in range(B) if self.phase[b] != FREE), key=lambda b: self.adm[b])
        # 3. decode growth
        for i, b in enumerate(order):
            if self.phase[b] != DECODE or len(self.row_pages[b]) > (self.seq_lens[b] - 1) // PAGE:
                continue
            victims = 0
            while not self.free and not self.lru:
                v = next((o for o in reversed(order[i + 1:]) if self.row_pages[o]), b)
                self.events["self_preemption" if v == b else "decode_victim" if self.phase[v] == DECODE else "prefill_victim"] += 1
                self._release(v)
                keep[v] = 0
                self.phase[v], self.done[v], self.target[v] = PREFILL, 0, self.seq_lens[v]
                self.preemptions += 1
                victims += 1
                if v == b:
                    break
            self.events["multi_victim"] += victims > 1
            if self.phase[b] == DECODE:
                self._pop(b)
        # 4. starts
        for b in order:
            if self.phase[b] != PREFILL or self.row_pages[b]:
                continue
            m = self.match(b)
            need = -(-self.target[b] // PAGE)
            e = sum(self.ref[q] == 0 for q in m)
            if len(self.free) + len(self.lru) - e < need - len(m):
                self.events["blocked_start"] += 1
                break
            for q in m:
                if self.ref[q] == 0:
                    self.lru.remove(q)
                self.ref[q] += 1
            self.row_pages[b] = list(m)
            while len(self.row_pages[b]) < need:
                self._pop(b)
            self.done[b] = PAGE * len(m)
            self.reg[b] = len(m)
            self.hit_pages += len(m)
            self.events["hit_start"] += bool(m)
            self.starts += 1
        # 5. plan, 6. table writes
        return self._plan(chunk_budget, order, keep)

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

    def check_conservation(self) -> None:
        """Every page is free, evictable or held; a DECODE row holds at least the pages of its cached tokens; a started PREFILL row holds its
        target's pages."""
        held = {q for b in range(self.batch) for q in self.row_pages[b]}
        assert sorted(list(held) + self.free + self.lru) == list(range(self.pages)), "a page is lost or in two places"
        for b in range(self.batch):
            n = len(self.row_pages[b])
            if self.phase[b] == FREE:
                assert n == 0, b
            elif self.phase[b] == PREFILL:
                assert n in (0, -(-self.target[b] // PAGE)), b
                assert n or self.done[b] == 0, b
            else:
                assert n >= -(-(self.seq_lens[b] - 1) // PAGE) and n <= self.blocks, b
