"""Pure-Python restatement of qs_inflight_schedule (include/qserve_b200.h, DESIGN.md 3.12): the schedule at the start of every in-flight step of
DecodeRunner(inflight=Q).  It steps on the same inputs as the kernel: the request queue (head, tail), the row state (phase, request, prompt
tokens cached, admission number) and the per-row vectors the step's commit leaves behind (history, lengths, finished).  `commit` restates the
plain step's spec_commit_stops (one token per unfinished row) so that scripts can be driven without a model.

Rules of one schedule(chunk_budget) call, in this order:
  1. Retire: every DECODE row with finished = 1, in row order, hands its generated tokens history[prompt_len : seq_len] and a reason (EOS when
     the last token is the row's eos, STOP when it is one of its stop ids, BUDGET otherwise) to its request's outputs, appends the request to
     the retired ring, and becomes FREE.
  2. Admit (chunk_budget > 0 only): while requests are queued, the lowest-index FREE row takes the oldest one: history = the prompt,
     prompt_len = seq_len = len, the request's eos / stop ids / max_tokens as the row's, done = 0, the next admission number, PREFILL.
  3. Plan: PREFILL rows in admission order take c_b = min(len - done, chunk_budget - used) prompt tokens; the chunk segment of C slots is laid
     out in row order (cu_seqlens over rows, prefix_lens = done, the tokens history[done : done + c_b], padding_offset = b C - cu_b); slots
     t >= used are padding (token 0, padding_offset = C - 1 - t: position C - 1 of row 0, which takes fewer than C tokens whenever padding
     exists, so the append skips it).  Decode segment: context_lens = seq_len and token = tokens_in for DECODE rows, 0 and token 0 otherwise.
  4. Tail masks: a row whose prompt completes becomes DECODE with logit row B + cu_seqlens[b + 1] - 1 and start_pos = len; DECODE rows use
     logit row b; every other row gets logit row b and finished = 1 (the commit skips it); completing and decoding rows get finished = 0.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

FREE, PREFILL, DECODE = 0, 1, 2
EOS, STOP, BUDGET = 1, 2, 3
REASONS = {EOS: "eos", STOP: "stop", BUDGET: "budget"}
MAX_STOPS = 8


@dataclass
class Request:
    prompt: List[int]
    max_tokens: int
    eos: int = -1
    stop: tuple = ()


@dataclass
class Plan:
    cu_seqlens: List[int]
    chunk_lens: List[int]
    prefix_lens: List[int]
    context_lens: List[int]
    tokens: List[int]          # B decode tokens, then the C chunk-segment slots
    padding_offset: List[int]  # [C]
    logit_rows: List[int]
    used: int


@dataclass
class InflightOracle:
    batch: int
    queue: int
    chunk: int
    max_tokens: int
    requests: List[Request] = field(default_factory=list)  # by request id
    head: int = 0
    retired: int = 0
    admitted: int = 0

    def __post_init__(self):
        B = self.batch
        self.phase = [FREE] * B
        self.row_req = [-1] * B
        self.done = [0] * B
        self.adm = [0] * B
        self.history: List[List[int]] = [[] for _ in range(B)]
        self.prompt_lens = [0] * B
        self.seq_lens = [0] * B
        self.finished = [0] * B
        self.eos = [-1] * B
        self.stop = [(-1,) * MAX_STOPS for _ in range(B)]
        self.budget = [self.max_tokens] * B
        self.start_pos = [0] * B
        self.tokens_in = [0] * B
        self.ring: List[int] = []  # retired request ids, in retire order
        self.outputs: dict = {}    # request id -> (tokens, reason)

    @property
    def tail(self) -> int:
        return len(self.requests)

    def submit(self, req: Request) -> int:
        self.requests.append(req)
        return len(self.requests) - 1

    def schedule(self, chunk_budget: int) -> Plan:
        B, C = self.batch, self.chunk
        # 1. retire
        for b in range(B):
            if self.phase[b] == DECODE and self.finished[b]:
                r, p, L = self.row_req[b], self.prompt_lens[b], self.seq_lens[b]
                toks = self.history[b][p:L]
                last = self.history[b][L - 1] if L > 0 else -1
                reason = BUDGET
                if last >= 0 and last == self.eos[b]:
                    reason = EOS
                elif last >= 0 and last in self.stop[b]:
                    reason = STOP
                assert r not in self.outputs, f"request {r} retired twice"
                self.outputs[r] = (list(toks), reason)
                self.ring.append(r)
                self.retired += 1
                self.phase[b], self.row_req[b] = FREE, -1
        # 2. admit
        if chunk_budget > 0:
            for b in range(B):
                if self.phase[b] == FREE and self.head < self.tail:
                    r = self.head
                    self.head += 1
                    q = self.requests[r]
                    n = len(q.prompt)
                    self.history[b] = list(q.prompt)
                    self.prompt_lens[b] = self.seq_lens[b] = n
                    self.eos[b] = q.eos
                    self.stop[b] = tuple(q.stop) + (-1,) * (MAX_STOPS - len(q.stop))
                    self.budget[b] = q.max_tokens
                    self.done[b] = 0
                    self.adm[b] = self.admitted
                    self.admitted += 1
                    self.row_req[b] = r
                    self.phase[b] = PREFILL
        # 3. plan
        order = sorted((b for b in range(B) if self.phase[b] == PREFILL), key=lambda b: self.adm[b])
        take, used = [0] * B, 0
        for b in order:
            take[b] = min(self.prompt_lens[b] - self.done[b], chunk_budget - used)
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
        # 4. tail masks
        for b in range(B):
            if self.phase[b] == PREFILL:
                self.done[b] += take[b]
                if self.done[b] == self.prompt_lens[b]:
                    self.phase[b] = DECODE
                    self.start_pos[b] = self.prompt_lens[b]
                    plan.logit_rows[b] = B + cu[b + 1] - 1
                    self.finished[b] = 0
                else:
                    self.finished[b] = 1
            elif self.phase[b] == DECODE:
                self.finished[b] = 0
            else:
                self.finished[b] = 1
        return plan

    def commit(self, tokens) -> None:
        """spec_commit_stops of a plain step (one token per row): every unfinished row appends its token, and finishes on eos, a stop id or
        its budget; start_pos / context length / tokens_in follow the new length."""
        for b in range(self.batch):
            if self.finished[b]:
                continue
            t = int(tokens[b])
            L, p = self.seq_lens[b], self.prompt_lens[b]
            if self.budget[b] - (L - p) <= 0:
                continue
            self.history[b] = self.history[b][:L] + [t]
            self.seq_lens[b] = L + 1
            self.start_pos[b] = L
            self.tokens_in[b] = t
            stop = (self.eos[b] >= 0 and t == self.eos[b]) or t in [s for s in self.stop[b] if s >= 0]
            if stop or L + 1 - p >= self.budget[b]:
                self.finished[b] = 1

    def pending_prompt_tokens(self) -> int:
        """Prompt tokens still to prefill: the queued requests' and the prefilling rows' remaining ones."""
        queued = sum(len(self.requests[r].prompt) for r in range(self.head, self.tail))
        return queued + sum(self.prompt_lens[b] - self.done[b] for b in range(self.batch) if self.phase[b] == PREFILL)


def appended_positions(plan: Plan, row_req: List[int], batch: int, chunk: int) -> list:
    """The (request, position) pairs the chunk segment appends, by the append kernel's own rule: slot t maps through padding_offset to
    (row, cpos) = divmod(t + padding_offset[t], C) and is appended iff cpos < chunk_lens[row], at prefix_lens[row] + cpos."""
    out = []
    for t in range(chunk):
        b, cpos = divmod(t + plan.padding_offset[t], chunk)
        assert 0 <= b < batch
        if cpos < plan.chunk_lens[b]:
            out.append((row_req[b], plan.prefix_lens[b] + cpos, plan.tokens[batch + t]))
    return out
