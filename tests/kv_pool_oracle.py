"""Pure-Python restatement of qs_inflight_schedule_pool (include/qserve_b200.h, DESIGN.md 3.12): the in-flight schedule of
tests/inflight_oracle.py over a shared KV page pool.  It steps on the kernel's inputs and keeps the pool's state as the kernel does: the free
stack (free[-1] is popped first), every row's page list and prefill target, the counters and the page tables of every layer, K and V (as
(layer, kv, page) triples instead of addresses).

Rules of one schedule(chunk_budget) call, in this order:
  1. Retire as InflightOracle; a retired row's pages go back onto the free stack, in row order and then page order.
  2. Admit as InflightOracle, without a page check: target = the prompt length.
  3. Decode growth, over the DECODE rows in admission order: a row of context seq_len that does not own page ceil(seq_len / 64) - 1 pops one.
     If the stack is empty it first preempts the page-holding row with the highest admission number (itself included): the victim's pages go
     back onto the stack in page order, and it becomes PREFILL with done = 0 and target = seq_len, idle in this step.  A requester that
     preempted itself pops nothing.
  4. Starts, over the PREFILL rows that hold no pages, in admission order: a row starts when the free pages cover ceil(target / 64) and takes
     them all at once; the first row that cannot start blocks every later one.
  5. Plan and tail masks as InflightOracle over the started PREFILL rows, with target in place of the prompt length.
  6. Table writes: entries [keep, count) of every row, where keep is the count before the call, or 0 if the row lost its pages in the call.
It also counts events: decode victims, prefill victims, self-preemptions and calls whose starts were blocked.
Rules 1, 2 and 5 are InflightOracle.schedule's; this class adds the page steps through its hooks, and PrefixCacheOracle changes how a page
is taken and released and what a start reuses.
"""
from __future__ import annotations

from collections import Counter
from typing import Dict, List, Tuple

from tests.inflight_oracle import DECODE, FREE, PREFILL, InflightOracle

PAGE = 64


def min_pages(prompt_cols: int, max_tokens: int) -> int:
    """The smallest pool the schedule accepts: one request of prompt_cols prompt and max_tokens generated tokens, and its root."""
    return -(-(prompt_cols + max_tokens + 1) // PAGE)


class KvPoolOracle(InflightOracle):
    def __init__(self, batch: int, queue: int, chunk: int, max_tokens: int, prompt_cols: int, pages: int, blocks: int, layers: int = 1):
        super().__init__(batch, queue, chunk, max_tokens)
        need = min_pages(prompt_cols, max_tokens)
        if pages < need or blocks < need:
            raise ValueError(f"pages={pages} and blocks={blocks} must each be at least {need}")
        self.pages, self.blocks, self.layers = pages, blocks, layers
        self.free: List[int] = list(range(pages - 1, -1, -1))
        self.row_pages: List[List[int]] = [[] for _ in range(batch)]
        self.keep = [0] * batch  # leading page-list entries whose table entries are written
        self.peak = self.preemptions = self.starts = 0
        self.tables: Dict[Tuple[int, int, int, int], int] = {}  # (layer, row, kv, block) -> page
        self.events = {"decode_victim": 0, "prefill_victim": 0, "self_preemption": 0, "blocked_start": 0}

    # ---- the pages a row can take ----
    def _take(self) -> int:
        return self.free.pop()

    def _takeable(self, match=()) -> int:
        """How many pages a take can reach, besides the pages of a start's match: the free stack."""
        return len(self.free)

    def _pop(self, b: int) -> None:
        self.row_pages[b].append(self._take())
        self.peak = max(self.peak, self.pages - self._takeable())

    def _release(self, b: int) -> None:
        self.free.extend(self.row_pages[b])
        self.row_pages[b] = []
        self.keep[b] = 0

    def match(self, b: int) -> List[int]:
        """The cached pages a start of row b reuses: none without the prefix cache."""
        return []

    def _share(self, b: int, match: List[int]) -> None:
        """A start takes the pages of its match (the prefix cache's refs and LRU)."""

    # ---- the page steps of InflightOracle.schedule ----
    def _started(self, b: int) -> bool:
        return bool(self.row_pages[b])

    def _grow(self, order: List[int]) -> None:
        for i, b in enumerate(order):
            if self.phase[b] != DECODE or len(self.row_pages[b]) > (self.seq_lens[b] - 1) // PAGE:
                continue
            victims = 0
            while not self._takeable():
                v = next((o for o in reversed(order[i + 1:]) if self.row_pages[o]), b)
                self.events["self_preemption" if v == b else "decode_victim" if self.phase[v] == DECODE else "prefill_victim"] += 1
                self._release(v)
                self.phase[v], self.done[v], self.target[v] = PREFILL, 0, self.seq_lens[v]
                self.preemptions += 1
                victims += 1
                if v == b:
                    break
            if victims > 1:  # only the prefix cache's victim can free no page: all of its pages may be shared
                self.events["multi_victim"] += 1
            if self.phase[b] == DECODE:
                self._pop(b)

    def _start(self, order: List[int]) -> None:
        for b in order:
            if self.phase[b] != PREFILL or self.row_pages[b]:
                continue
            m = self.match(b)
            need = -(-self.target[b] // PAGE)
            if self._takeable(m) < need - len(m):
                self.events["blocked_start"] += 1
                break
            self._share(b, m)
            self.row_pages[b] = list(m)
            while len(self.row_pages[b]) < need:
                self._pop(b)
            self.done[b] = PAGE * len(m)
            self.starts += 1

    def _write_tables(self) -> None:
        for b in range(self.batch):
            for j in range(self.keep[b], len(self.row_pages[b])):
                for li in range(self.layers):
                    for kv in range(2):
                        self.tables[(li, b, kv, j)] = self.row_pages[b][j]
            self.keep[b] = len(self.row_pages[b])

    @property
    def top(self) -> int:
        return len(self.free)

    def counters(self) -> List[int]:
        return [self.top, self.peak, self.preemptions, self.starts]

    def _evictable(self) -> List[int]:
        """The pages no row holds that are not free: the prefix cache's LRU list."""
        return []

    def _shared(self, q: int) -> bool:
        """Whether page q may be held by several rows: only a registered page of the prefix cache."""
        return False

    def check_conservation(self) -> None:
        """Every page is free, held or (with the prefix cache) evictable, in one place; only a shared page is held more than once; FREE rows
        hold none; a PREFILL row holds none (waiting) or the ceil(target / 64) pages of its start; a DECODE row holds at least the pages of
        the tokens it has cached."""
        held = Counter(q for b in range(self.batch) for q in self.row_pages[b])
        assert sorted(list(held) + self.free + self._evictable()) == list(range(self.pages)), "a page is lost or in two places"
        assert all(n == 1 or self._shared(q) for q, n in held.items()), "a private page is held twice"
        for b in range(self.batch):
            n = len(self.row_pages[b])
            if self.phase[b] == FREE:
                assert n == 0, b
            elif self.phase[b] == PREFILL:
                assert n in (0, -(-self.target[b] // PAGE)), b
                assert n or self.done[b] == 0, b
            else:
                assert n >= -(-(self.seq_lens[b] - 1) // PAGE) and n <= self.blocks, b
