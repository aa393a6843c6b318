"""CPU tests of the in-flight schedule's contract (tests/inflight_oracle.py, which qs_inflight_schedule follows bit for bit on the GPU): under
seeded random scripts of arrivals, prompt lengths 1 .. ctx, budgets, stop rules and chunk budgets C from 1 to more than B * ctx, every step
keeps the chunk segment within C, admits first-come-first-served, never gives a row two requests, appends every prompt token exactly once and
in order (by the append kernel's own padding-offset rule), and every submitted request retires exactly once; a budget-0 call admits nothing."""
import random

import pytest

from tests.inflight_oracle import DECODE, FREE, PREFILL, InflightOracle, Request, appended_positions


def _run_script(seed: int, B: int, Q: int, C: int, ctx: int, T: int, n_req: int, vocab: int = 50):
    rng = random.Random(seed)
    o = InflightOracle(B, Q, C, T)
    arrivals = sorted(rng.randrange(0, 3 * n_req) for _ in range(n_req)) if rng.random() < 0.7 else [0] * n_req
    appended: dict = {}
    polled = 0
    step = 0
    prev_adm_req = -1
    while len(o.outputs) < n_req:
        assert step < 100000, "script does not terminate"
        # submissions of this step, within the queue: request r may reuse slot r % Q once request r - Q has retired
        while o.tail < n_req and arrivals[o.tail] <= step and (o.tail - Q < 0 or (o.tail - Q) in o.outputs):
            n = rng.randint(1, ctx)
            stop = tuple(rng.sample(range(vocab), rng.randint(0, 3)))
            o.submit(Request([rng.randrange(vocab) for _ in range(n)], rng.randint(1, T), rng.choice([-1, rng.randrange(vocab)]), stop))
        budget = 0 if rng.random() < 0.1 else C
        head0, phase0, req0 = o.head, list(o.phase), list(o.row_req)
        plan = o.schedule(budget)
        if budget == 0:
            assert o.head == head0, "a budget-0 call admitted a request"
        # first-come-first-served: admitted in id order, into the lowest free rows
        new = [b for b in range(B) if o.row_req[b] >= 0 and o.row_req[b] != req0[b]]
        assert sorted(o.row_req[b] for b in new) == list(range(head0, o.head))
        assert [o.row_req[b] for b in sorted(new)] == list(range(head0, o.head))
        if new:
            assert min(o.row_req[b] for b in new) > prev_adm_req
            prev_adm_req = max(o.row_req[b] for b in new)
        live = [o.row_req[b] for b in range(B) if o.row_req[b] >= 0]
        assert len(live) == len(set(live)), "a request in two rows"
        assert all((o.row_req[b] >= 0) == (o.phase[b] != FREE) for b in range(B))
        # the chunk segment: within C, row order, earlier admissions served first
        assert plan.used == plan.cu_seqlens[B] == sum(plan.chunk_lens) <= budget
        served = sorted((o.adm[b], plan.chunk_lens[b], o.prompt_lens[b] - plan.prefix_lens[b]) for b in range(B)
                        if o.row_req[b] >= 0 and (o.phase[b] == PREFILL or plan.chunk_lens[b]))
        short = False
        for _, c, rem in served:
            assert not (short and c), "a later admission took prompt tokens before an earlier one was served"
            short = short or c < rem
        for b in range(B):
            if plan.chunk_lens[b]:
                assert plan.cu_seqlens[b + 1] - plan.cu_seqlens[b] == plan.chunk_lens[b]
        for r, pos, tok in appended_positions(plan, o.row_req, B, C):
            got = appended.setdefault(r, [])
            assert pos == len(got), f"request {r}: position {pos} appended after {len(got)} tokens"
            assert tok == o.requests[r].prompt[pos]
            got.append(tok)
        for b in range(B):
            assert plan.context_lens[b] == (o.seq_lens[b] if phase0[b] == DECODE and o.phase[b] == DECODE and o.row_req[b] == req0[b]
                                            and plan.logit_rows[b] == b else 0)
        # the commit: one token per unfinished row
        o.commit([rng.randrange(vocab) for _ in range(B)])
        polled = len(o.ring)
        step += 1
    assert polled == n_req
    assert sorted(o.ring) == list(range(n_req)), "every request retires exactly once"
    for r, q in enumerate(o.requests):
        assert appended[r] == q.prompt, f"request {r}: prompt not appended exactly once in order"
        toks, reason = o.outputs[r]
        assert 1 <= len(toks) <= q.max_tokens
        if len(toks) < q.max_tokens:
            assert toks[-1] == q.eos or toks[-1] in q.stop
    assert o.pending_prompt_tokens() == 0
    return step


@pytest.mark.parametrize("seed", range(12))
def test_random_scripts(seed):
    rng = random.Random(1000 + seed)
    B, ctx = rng.choice([1, 2, 3, 5, 8]), rng.choice([1, 4, 17, 64])
    C = rng.choice([1, 2, 7, ctx, B * ctx, B * ctx + 5])
    Q = rng.choice([1, B, 2 * B + 1])
    _run_script(seed, B, Q, C, ctx, rng.choice([1, 3, 9]), rng.randint(1, 30))


def test_budget_zero_admits_nothing_and_retires():
    o = InflightOracle(2, 4, 8, 4)
    o.submit(Request([1, 2, 3], 1))
    plan = o.schedule(0)
    assert o.head == 0 and o.phase == [FREE, FREE] and plan.used == 0 and plan.cu_seqlens == [0, 0, 0]
    assert o.finished == [1, 1]
    o.schedule(8)
    assert o.phase == [DECODE, FREE] and o.row_req == [0, -1]
    o.commit([5, 0])
    assert o.finished[0] == 1  # budget 1
    o.schedule(0)
    assert o.outputs[0] == ([5], 3) and o.phase == [FREE, FREE]


def test_padding_slots_map_past_row_zero():
    """Padding slots map through padding_offset to position C - 1 of row 0, which never takes C tokens when padding exists."""
    o = InflightOracle(3, 3, 10, 2)
    for n in (2, 3):
        o.submit(Request(list(range(n)), 2))
    plan = o.schedule(10)
    assert plan.used == 5 and plan.cu_seqlens == [0, 2, 5, 5]
    for t in range(5, 10):
        b, cpos = divmod(t + plan.padding_offset[t], 10)
        assert (b, cpos) == (0, 9) and cpos >= plan.chunk_lens[0]
    assert plan.logit_rows == [3 + 1, 3 + 4, 2]
    assert plan.tokens[3:8] == [0, 1, 0, 1, 2]
