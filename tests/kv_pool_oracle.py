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
"""
from __future__ import annotations

from typing import Dict, List, Tuple

from tests.inflight_oracle import BUDGET, DECODE, EOS, FREE, MAX_STOPS, PREFILL, STOP, InflightOracle, Plan

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
        self.target = [0] * batch
        self.peak = self.preemptions = self.starts = 0
        self.tables: Dict[Tuple[int, int, int, int], int] = {}  # (layer, row, kv, block) -> page
        self.events = {"decode_victim": 0, "prefill_victim": 0, "self_preemption": 0, "blocked_start": 0}

    def _pop(self, b: int) -> None:
        self.row_pages[b].append(self.free.pop())
        self.peak = max(self.peak, self.pages - len(self.free))

    def _release(self, b: int) -> None:
        self.free.extend(self.row_pages[b])
        self.row_pages[b] = []

    def schedule(self, chunk_budget: int) -> Plan:
        B, C = self.batch, self.chunk
        keep = [len(p) for p in self.row_pages]
        # 1. retire
        for b in range(B):
            if self.phase[b] == DECODE and self.finished[b]:
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
                self._release(b)
                keep[b] = 0
        # 2. admit
        if chunk_budget > 0:
            for b in range(B):
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
        order = sorted((b for b in range(B) if self.phase[b] != FREE), key=lambda b: self.adm[b])
        # 3. decode growth
        for i, b in enumerate(order):
            if self.phase[b] != DECODE or len(self.row_pages[b]) > (self.seq_lens[b] - 1) // PAGE:
                continue
            if not self.free:
                v = next((o for o in reversed(order[i + 1:]) if self.row_pages[o]), b)
                self.events["self_preemption" if v == b else "decode_victim" if self.phase[v] == DECODE else "prefill_victim"] += 1
                self._release(v)
                keep[v] = 0
                self.phase[v], self.done[v], self.target[v] = PREFILL, 0, self.seq_lens[v]
                self.preemptions += 1
                if v == b:
                    continue
            self._pop(b)
        # 4. starts
        for b in order:
            if self.phase[b] != PREFILL or self.row_pages[b]:
                continue
            need = -(-self.target[b] // PAGE)
            if need > len(self.free):
                self.events["blocked_start"] += 1
                break
            for _ in range(need):
                self._pop(b)
            self.starts += 1
        # 5. plan
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
        # 6. table writes
        for b in range(B):
            for j in range(keep[b], len(self.row_pages[b])):
                for li in range(self.layers):
                    for kv in range(2):
                        self.tables[(li, b, kv, j)] = self.row_pages[b][j]
        return plan

    @property
    def top(self) -> int:
        return len(self.free)

    def counters(self) -> List[int]:
        return [self.top, self.peak, self.preemptions, self.starts]

    def check_conservation(self) -> None:
        """Every page is free or held by exactly one row, exactly once; FREE rows hold none; a PREFILL row holds none (waiting) or the
        ceil(target / 64) pages of its start; a DECODE row holds at least the pages of the tokens it has cached."""
        held = [p for b in range(self.batch) for p in self.row_pages[b]]
        assert sorted(held + self.free) == list(range(self.pages)), "a page is lost or held twice"
        for b in range(self.batch):
            n = len(self.row_pages[b])
            if self.phase[b] == FREE:
                assert n == 0, b
            elif self.phase[b] == PREFILL:
                assert n in (0, -(-self.target[b] // PAGE)), b
                assert n or self.done[b] == 0, b
            else:
                assert n >= -(-(self.seq_lens[b] - 1) // PAGE) and n <= self.blocks, b

    def pending_prompt_tokens(self) -> int:
        queued = sum(len(self.requests[r].prompt) for r in range(self.head, self.tail))
        return queued + sum(self.target[b] - self.done[b] for b in range(self.batch) if self.phase[b] == PREFILL)
