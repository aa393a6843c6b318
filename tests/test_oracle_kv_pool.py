"""CPU tests of the shared KV page pool's schedule contract (tests/kv_pool_oracle.py, which qs_inflight_schedule_pool follows bit for bit on
the GPU): with a pool that never runs dry it plans exactly as the own-pages schedule; at the smallest pool every seeded random script
finishes; after every call each page is free or held by exactly one row; a preemption takes the youngest page holder and starts are strictly
first-come-first-served; invalid pools raise."""
import random

import pytest

from tests.inflight_oracle import DECODE, FREE, PREFILL, InflightOracle, Request
from tests.kv_pool_oracle import KvPoolOracle, min_pages


def _request(rng, ctx, T, vocab):
    n = rng.randint(1, ctx)
    return Request([rng.randrange(vocab) for _ in range(n)], rng.randint(1, T), rng.choice([-1, rng.randrange(vocab)]),
                   tuple(rng.sample(range(vocab), rng.randint(0, 3))))


def _drive(oracles, seed, B, Q, C, ctx, T, n_req, vocab=50, check=None, max_steps=100000):
    """One seeded script of arrivals, chunk budgets and commits, applied to every oracle in `oracles` alike; check(step, plans) runs after
    every schedule call.  Returns the number of steps."""
    rng = random.Random(seed)
    reqs = [_request(rng, ctx, T, vocab) for _ in range(n_req)]
    lead = oracles[0]
    nxt = step = 0
    while len(lead.outputs) < n_req:
        assert step < max_steps, "script does not terminate"
        while nxt < n_req and rng.random() < 0.6 and (nxt - Q < 0 or (nxt - Q) in lead.outputs):
            for o in oracles:
                o.submit(reqs[nxt])
            nxt += 1
        budget = 0 if rng.random() < 0.1 else C
        plans = [o.schedule(budget) for o in oracles]
        if check:
            check(step, plans)
        toks = [rng.randrange(vocab) for _ in range(B)]
        for o in oracles:
            o.commit(toks)
        step += 1
    for r, q in enumerate(reqs):
        toks, _ = lead.outputs[r]
        assert 1 <= len(toks) <= q.max_tokens
        if len(toks) < q.max_tokens:
            assert toks[-1] == q.eos or toks[-1] in q.stop
    return step


def _config(seed):
    rng = random.Random(2000 + seed)
    B, ctx = rng.choice([1, 2, 3, 5, 8]), rng.choice([1, 17, 64, 100, 200])
    T = rng.choice([1, 9, 70])
    return B, rng.choice([1, B, 2 * B + 1]), rng.choice([1, 7, 40, ctx, B * ctx + 5]), ctx, T, rng.randint(1, 30)


@pytest.mark.parametrize("seed", range(10))
def test_ample_pool_plans_as_own_pages(seed):
    """P >= B x blocks: no start waits and nothing is preempted, so every plan and row state equals InflightOracle's."""
    B, Q, C, ctx, T, n = _config(seed)
    blocks = min_pages(ctx, T)
    own, pool = InflightOracle(B, Q, C, T), KvPoolOracle(B, Q, C, T, ctx, B * blocks, blocks)

    def check(step, plans):
        assert plans[0] == plans[1], step
        assert own.phase == pool.phase and own.done == pool.done and own.finished == pool.finished, step
        pool.check_conservation()

    _drive([own, pool], seed, B, Q, C, ctx, T, n, check=check)
    assert own.outputs == pool.outputs and pool.preemptions == 0 and pool.starts == n


@pytest.mark.parametrize("seed", range(16))
def test_smallest_pool_finishes_and_conserves_pages(seed):
    """P = ceil((ctx + T + 1) / 64): every script finishes, pages are conserved after every call, victims are the youngest page holders and
    starts are strictly first-come-first-served."""
    B, Q, C, ctx, T, n = _config(seed)
    P = min_pages(ctx, T)
    o = KvPoolOracle(B, Q, C, T, ctx, P, P, layers=2)
    before = {}

    def snapshot():
        before.update(pages=[list(p) for p in o.row_pages], phase=list(o.phase), req=list(o.row_req), pre=o.preemptions, events=dict(o.events))

    def check(step, plans):
        o.check_conservation()
        assert o.counters()[0] == len(o.free) and o.peak <= P
        # victims: held pages before, still hold the same request, lost the pages without retiring
        victims = [b for b in range(B) if before["pages"][b] and o.row_req[b] == before["req"][b] and o.phase[b] == PREFILL
                   and not o.row_pages[b] and before["phase"][b] != FREE]
        assert len(victims) == o.preemptions - before["pre"]
        kept = [b for b in range(B) if before["pages"][b] and o.row_pages[b] and o.row_req[b] == before["req"][b]]
        for v in victims:
            assert plans[0].context_lens[v] == 0 and plans[0].chunk_lens[v] == 0 and o.finished[v] == 1 and o.done[v] == 0
            assert all(o.adm[k] < o.adm[v] for k in kept), (step, v)
        # FCFS: every row started in this call is older than every row still waiting for pages
        started = [b for b in range(B) if o.row_pages[b] and not (before["pages"][b] and o.row_req[b] == before["req"][b])]
        waiting = [b for b in range(B) if o.phase[b] == PREFILL and not o.row_pages[b]]
        for s in started:
            assert all(o.adm[s] < o.adm[w] for w in waiting), (step, s)
        # page tables: every held page's entries in every layer, K and V
        for b in range(B):
            for j, page in enumerate(o.row_pages[b]):
                assert all(o.tables[(li, b, kv, j)] == page for li in range(2) for kv in range(2))
        snapshot()

    snapshot()
    _drive([o], seed, B, Q, C, ctx, T, n, check=check)
    assert o.top == P and all(not p for p in o.row_pages)


def test_every_event_kind_occurs():
    """The script of tests/test_gpu_kv_pool.py's kernel test preempts decode and prefill rows, preempts a requester itself and blocks starts."""
    B, Q, C, ctx, T = 6, 7, 40, 150, 60
    o = KvPoolOracle(B, Q, C, T, ctx, 7, min_pages(ctx, T))
    _drive([o], 31, B, Q, C, ctx, T, 40, vocab=400, check=lambda s, p: o.check_conservation())
    assert all(v > 0 for v in o.events.values()), o.events


def test_preempted_row_recomputes_its_history():
    """Two rows over the smallest pool: the younger one needs a page when none is free and preempts itself (it is the youngest page holder),
    waits while the older one holds the pages, then starts again with target = its seq_len, carries history[0 : target) through the chunk
    segment in one piece and decodes on from start_pos = target; its outputs are history[prompt_len : seq_len)."""
    P = min_pages(100, 40)
    o = KvPoolOracle(2, 4, 200, 40, 100, P, P)
    o.submit(Request(list(range(100)), 40))     # request 0: 2 pages
    o.submit(Request(list(range(1, 64)), 40))   # request 1: 1 page, its third generated token needs a second
    o.schedule(200)
    assert o.phase == [DECODE, DECODE] and [len(p) for p in o.row_pages] == [2, 1] and o.top == P - 3 == 0
    k = 0
    while o.preemptions == 0:
        o.commit([1000 + k, 2000 + k])
        k += 1
        plan = o.schedule(200)
    L1 = o.seq_lens[1]
    assert L1 == 65 and o.events["self_preemption"] == 1 and o.phase[1] == PREFILL and o.target[1] == L1 and o.done[1] == 0
    assert plan.context_lens == [o.seq_lens[0], 0] and o.finished == [0, 1] and o.events["blocked_start"] == 1
    history = list(o.history[1][:L1])
    while o.phase[1] == PREFILL:  # row 0 decodes to its budget and retires; then row 1 takes the three pages
        o.commit([3000 + k, 4000 + k])
        k += 1
        plan = o.schedule(200)
    assert 0 in o.outputs and o.starts == 3 and o.preemptions == 1 and len(o.row_pages[1]) == 2
    assert plan.chunk_lens[1] == L1 and plan.prefix_lens[1] == 0 and plan.tokens[2:2 + L1] == history
    assert plan.logit_rows[1] == 2 + L1 - 1 and o.start_pos[1] == L1
    while 1 not in o.outputs:
        o.commit([0, 5000 + k])
        k += 1
        o.schedule(200)
    toks, _ = o.outputs[1]
    assert toks[:L1 - 63] == history[63:] and len(toks) == 40


def test_invalid_pools_raise():
    with pytest.raises(ValueError):
        KvPoolOracle(2, 2, 8, 64, 100, min_pages(100, 64) - 1, 8)
    with pytest.raises(ValueError):
        KvPoolOracle(2, 2, 8, 64, 100, 8, min_pages(100, 64) - 1)
    assert min_pages(100, 64) == 3 and min_pages(126, 1) == 2 and min_pages(127, 1) == 3


BAD_RUNNERS = [
    dict(kv_pool_pages=8, generate=True, max_new_tokens=8, prompt_tokens=64),                          # no inflight
    dict(kv_pool_pages=8),                                                                               # no inflight
    dict(kv_pool_pages=1, inflight=4, generate=True, max_new_tokens=64, prompt_tokens=64),             # below ceil((100 + 64 + 1) / 64)
    dict(kv_pool_pages=-2, inflight=4, generate=True, max_new_tokens=8, prompt_tokens=64),
    dict(kv_pool_pages=8, inflight=4, generate=True, max_new_tokens=8, prompt_tokens=64, tp_size=2),
]


@pytest.mark.parametrize("kw", BAD_RUNNERS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) for kw in BAD_RUNNERS])
def test_invalid_runner_pool_raises(kw):
    """DecodeRunner refuses a pool without in-flight batching, below the smallest size, or on more than one GPU, before it allocates anything."""
    from qserve_b200.decode import DecodeRunner

    with pytest.raises(RuntimeError):
        DecodeRunner("tiny", "w4a8kv4", batch=4, ctx=100, **kw)
