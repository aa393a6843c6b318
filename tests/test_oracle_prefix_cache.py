"""CPU tests of the prefix cache's schedule contract (tests/prefix_cache_oracle.py, which qs_inflight_schedule_pool_cache follows bit for bit
on the GPU): without shared full pages it plans exactly as the pool schedule; on scripts with shared system prompts, repeated prompts and
multi-turn continuations every page is in one state, refs count page-list occurrences, the index holds exactly the registered pages, rows
hold key chains, no plan writes into a registered page and every script finishes; matches, the epoch rule, single-victim preemption and the LRU
order at hand-built edges; invalid runners raise."""
import random
from collections import deque

import pytest

from tests.inflight_oracle import PREFILL, Request
from tests.kv_pool_oracle import PAGE, KvPoolOracle, min_pages
from tests.prefix_cache_oracle import PrefixCacheOracle
from tests.test_oracle_kv_pool import _config, _drive


@pytest.mark.parametrize("seed", range(10))
def test_no_sharing_plans_as_pool(seed):
    """Prompts that share no full page, a pool that never preempts: plans, row states, starts and outputs equal KvPoolOracle's (page ids may
    differ: released pages are cached and evicted instead of freed)."""
    B, Q, C, ctx, T, n = _config(seed)
    blocks = min_pages(ctx, T)
    pool, cache = KvPoolOracle(B, Q, C, T, ctx, B * blocks, blocks), PrefixCacheOracle(B, Q, C, T, ctx, B * blocks, blocks)

    def check(step, plans):
        assert plans[0] == plans[1], step
        assert pool.phase == cache.phase and pool.done == cache.done and pool.finished == cache.finished, step
        assert [len(p) for p in pool.row_pages] == [len(p) for p in cache.row_pages], step
        cache.check_cache()
        cache.check_conservation()

    _drive([pool, cache], seed, B, Q, C, ctx, T, n, check=check)
    assert pool.outputs == cache.outputs and pool.starts == cache.starts and pool.preemptions == cache.preemptions == 0
    assert cache.hit_pages == 0


def _shared_requests(rng, ctx, T, vocab, n):
    """Requests over one system prompt (unique tails), exact repeats of earlier prompts and unique prompts."""
    system = [rng.randrange(vocab) for _ in range(min(ctx - 1, rng.choice([64, 100, 128, 192])))]
    reqs = []
    for _ in range(n):
        u = rng.random()
        if u < 0.5:
            tail = [rng.randrange(vocab) for _ in range(rng.randint(1, max(1, ctx - len(system))))]
            prompt = (system + tail)[:ctx]
        elif u < 0.7 and reqs:
            prompt = list(rng.choice(reqs).prompt)
        else:
            prompt = [rng.randrange(vocab) for _ in range(rng.randint(1, ctx))]
        reqs.append(Request(prompt, rng.randint(1, T), rng.choice([-1, rng.randrange(vocab)]), tuple(rng.sample(range(vocab), rng.randint(0, 2)))))
    return reqs


def drive_shared(oracles, seed, B, Q, C, ctx, T, n_req, vocab=50, check=None, turns=3, max_steps=100000):
    """A seeded script of _shared_requests in which some requests are conversations: when turn k retires, turn k + 1 (its prompt, its answer
    and 1 .. 64 new tokens, if that fits in ctx) joins the queue.  check(step, plans) runs after every schedule call.  Returns the requests
    in submission order."""
    rng = random.Random(seed)
    lead = oracles[0]
    pending = deque(_shared_requests(rng, ctx, T, vocab, n_req))
    talk = {}            # submitted request id -> turns left
    seen, step = 0, 0
    while pending or len(lead.outputs) < lead.tail:
        assert step < max_steps, "script does not terminate"
        while pending and rng.random() < 0.6 and (lead.tail - Q < 0 or (lead.tail - Q) in lead.outputs):
            req = pending.popleft()
            r = [o.submit(req) for o in oracles][0]
            talk.setdefault(r, turns - 1 if rng.random() < 0.4 else 0)
        budget = 0 if rng.random() < 0.1 else C
        plans = [o.schedule(budget) for o in oracles]
        if check:
            check(step, plans)
        for r in lead.ring[seen:]:
            prompt = lead.requests[r].prompt + lead.outputs[r][0] + [rng.randrange(vocab) for _ in range(rng.randint(1, 64))]
            if talk.get(r, 0) and len(prompt) <= ctx:
                pending.appendleft(Request(prompt, rng.randint(1, T)))
                talk[lead.tail + len(pending) - 1] = talk[r] - 1  # the id it will get if nothing is submitted before it
        seen = len(lead.ring)
        toks = [rng.randrange(vocab) for _ in range(B)]
        for o in oracles:
            o.commit(toks)
        step += 1
    return lead.requests


def _shared_config(seed):
    rng = random.Random(3000 + seed)
    B, ctx, T = rng.choice([1, 2, 3, 5, 8]), rng.choice([130, 200, 300]), rng.choice([9, 70])
    return B, rng.choice([B, 2 * B + 1]), rng.choice([7, 40, 64, ctx, B * ctx + 5]), ctx, T, rng.randint(8, 30), rng.choice([1, 1, 2, 3])


def _check_writes(o, plan):
    """No plan position lies in a registered page: the chunk positions [done, done + c) and the decode position seq_len - 1."""
    for b in range(o.batch):
        if plan.chunk_lens[b]:
            assert plan.prefix_lens[b] // PAGE >= o.reg[b], b
        if plan.context_lens[b]:
            assert (plan.context_lens[b] - 1) // PAGE >= o.reg[b], b


@pytest.mark.parametrize("seed", range(16))
def test_shared_scripts_keep_the_invariants(seed):
    B, Q, C, ctx, T, n, scale = _shared_config(seed)
    P = min_pages(ctx, T) * scale
    o = PrefixCacheOracle(B, Q, C, T, ctx, P, min_pages(ctx, T) + 1, layers=2)

    def check(step, plans):
        o.check_cache()
        o.check_conservation()
        _check_writes(o, plans[0])
        assert o.peak <= P

    drive_shared([o], seed, B, Q, C, ctx, T, n, check=check)
    assert o.top + len(o.lru) == P and all(not p for p in o.row_pages)


def test_shared_scripts_hit_evict_and_preempt():
    """Across the seeded scripts every event occurs: hits, evictions, duplicates, preemptions and blocked starts."""
    total = dict(hit=0, evictions=0, duplicates=0, preemptions=0, blocked=0)
    for seed in range(16):
        B, Q, C, ctx, T, n, scale = _shared_config(seed)
        o = PrefixCacheOracle(B, Q, C, T, ctx, min_pages(ctx, T) * scale, min_pages(ctx, T) + 1)
        drive_shared([o], seed, B, Q, C, ctx, T, n)
        total["hit"] += o.hit_pages
        total["evictions"] += o.evictions
        total["duplicates"] += o.duplicates
        total["preemptions"] += o.preemptions
        total["blocked"] += o.events["blocked_start"]
    assert all(v > 0 for v in total.values()), total


# ---------------------------------------------------------------------------------------------------------------------------------------------
def _run_until(o, cond, tok=7, budget=None, limit=1000):
    for _ in range(limit):
        if cond():
            return
        o.commit([tok] * o.batch)
        o.schedule(o.chunk if budget is None else budget)
    raise AssertionError("condition not reached")


def _prompt(n, seed):
    rng = random.Random(seed)
    return [rng.randrange(1000) for _ in range(n)]


def test_matches_recompute_the_rest():
    """A 192-token prompt, once cached, gives the same prompt 2 pages (one token must be computed: 64 are) and a 150-token prefix of it 2
    pages (22 computed)."""
    o = PrefixCacheOracle(2, 4, 256, 8, 256, 20, 6)
    A = _prompt(192, 1)
    o.submit(Request(A, 1))
    o.schedule(256)
    o.commit([5, 5])
    o.schedule(256)  # registers A's three full pages and retires it
    assert o.registrations == 3 and 0 in o.outputs and len(o.lru) == 3
    o.submit(Request(A, 1))
    o.submit(Request(A[:150], 1))
    plan = o.schedule(256)
    assert plan.prefix_lens[:2] == [128, 128] and plan.chunk_lens[:2] == [64, 22]
    assert o.row_pages[0][:2] == o.row_pages[1][:2] and o.reg[:2] == [2, 2] and o.hit_pages == 4
    assert all(o.ref[q] == 2 for q in o.row_pages[0][:2]) and len(o.lru) == 1
    o.check_cache()


def test_epoch_rule_rejects_a_stale_child():
    """A chain's child keeps its parent's epoch: when the parent is evicted and re-registered with other content, a prompt that starts with
    the new content and continues with the child's tokens does not match the child.  (The LRU evicts children before parents, so the
    schedule never leaves such a child behind; the order is forced here.)"""
    o = PrefixCacheOracle(1, 4, 256, 4, 256, 6, 6)
    a0, a1, x = _prompt(64, 2), _prompt(64, 3), _prompt(64, 4)
    o.submit(Request(a0 + a1 + [1], 1))
    o.schedule(256)
    o.commit([5])
    o.schedule(256)  # pages p0 (a0) and p1 (a1, child of p0) registered, then released
    p1, p0 = o.lru
    assert o.key[p1][0] == p0
    o.lru = [p0, p1]
    saved, o.free = o.free, []  # the next page must come from the LRU head
    o.submit(Request(x, 1))
    o.schedule(256)
    assert o.row_pages[0] == [p0] and o.evictions == 1
    o.commit([5])
    o.free = saved
    o.submit(Request(x + a1 + [9], 1))
    plan = o.schedule(256)  # registers p0 with content x and retires it, then starts the new prompt
    assert o.key[p0] == (-1, 0, tuple(x)) and o.epoch[p0] == 3 and o.key[p1] == (p0, 1, tuple(a1)) and p1 in o.index.values()
    assert o.row_pages[0][0] == p0 and p1 not in o.row_pages[0] and plan.prefix_lens[0] == 64 and o.hit_pages == 1


def test_one_victim_always_frees_a_page():
    """Under first-come-first-served starts and youngest-first preemption a victim's pages are never all shared (a row that shares the pages
    it took itself is younger and holds pages, so it would have been the victim), so across the seeded scripts the preemption loop of rule 3
    never needs a second victim."""
    for seed in range(16):
        B, Q, C, ctx, T, n, scale = _shared_config(seed)
        o = PrefixCacheOracle(B, Q, C, T, ctx, min_pages(ctx, T) * scale, min_pages(ctx, T) + 1)
        drive_shared([o], seed, B, Q, C, ctx, T, n)
        assert o.events["multi_victim"] == 0, seed


def test_lru_order_tails_first_oldest_release_first():
    """A retired row's registered pages join the LRU from its last to its first; two retirements queue in retire order; evictions take the
    head."""
    o = PrefixCacheOracle(2, 4, 512, 4, 256, 12, 6)
    o.submit(Request(_prompt(192, 6) + [1], 1))
    o.submit(Request(_prompt(128, 7) + [1], 2))
    o.schedule(512)
    a, b = list(o.row_pages[0][:3]), list(o.row_pages[1][:2])
    o.commit([5, 5])
    o.schedule(512)  # row 0 retires (budget 1)
    assert o.lru == a[::-1]
    o.commit([5, 5])
    o.schedule(512)  # row 1 retires
    assert o.lru == a[::-1] + b[::-1]
    o.free = []
    o.submit(Request(_prompt(64, 8), 1))
    o.schedule(512)
    assert o.row_pages[0] == [a[2]] and o.lru == a[1::-1] + b[::-1] and o.evictions == 1


def test_preempted_row_rematches_its_own_pages():
    """A row that registered a page and then preempted itself (the youngest holder) restarts, once the older row retires, on that page: it
    recomputes only the rest of its history."""
    P = min_pages(200, 60)
    o = PrefixCacheOracle(2, 4, 400, 60, 200, P, P)
    o.submit(Request(_prompt(190, 9), 60))  # 3 pages, a fourth at seq_len 193
    o.submit(Request(_prompt(60, 10), 60))  # 1 page, a second at seq_len 65: none is left
    o.schedule(400)
    _run_until(o, lambda: o.preemptions > 0)
    assert o.events["self_preemption"] == 1 and o.phase[1] == PREFILL and o.target[1] == 65 and len(o.lru) == 1
    own = o.lru[0]
    _run_until(o, lambda: o.row_pages[1])
    assert 0 in o.outputs and o.row_pages[1][0] == own and o.done[1] == 65 and o.hit_pages == 1
    o.check_cache()
    o.check_conservation()


BAD_RUNNERS = [
    dict(prefix_cache=True, inflight=4, generate=True, max_new_tokens=8, prompt_tokens=64),                     # no pool
    dict(prefix_cache=True, kv_pool_pages=8, generate=True, max_new_tokens=8, prompt_tokens=64),                # no inflight
    dict(prefix_cache=True, kv_pool_pages=8, inflight=4, generate=True, max_new_tokens=8, prompt_tokens=64, tp_size=2),
]


@pytest.mark.parametrize("kw", BAD_RUNNERS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) for kw in BAD_RUNNERS])
def test_invalid_runner_cache_raises(kw):
    """DecodeRunner refuses prefix_cache without the pool, without in-flight batching or on more than one GPU, before it allocates."""
    from qserve_b200.decode import DecodeRunner

    with pytest.raises(RuntimeError):
        DecodeRunner("tiny", "w4a8kv4", batch=4, ctx=100, **kw)
