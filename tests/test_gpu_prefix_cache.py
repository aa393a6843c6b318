"""GPU: automatic prefix caching over the shared KV page pool (DecodeRunner(inflight=Q, kv_pool_pages=P, prefix_cache=True),
qs_inflight_schedule_pool_cache, DESIGN.md 3.12 "Prefix cache").

* The schedule kernel equals tests/prefix_cache_oracle.py after every call of a shared-prefix script with hits, revivals of evictable pages,
  evictions, duplicates and preemptions: row state, plan, free stack, page lists, tables, refs, states, epochs, LRU order, counters, and every
  registered key resolves through the device index to its page.
* Without shared full pages every request's tokens, reasons and log-probabilities equal the prefix_cache=False pool runner's bit for bit.
* An exact hit: B = A's 128-token prompt + 100 tokens computes 100 tokens and equals, bit for bit, the cache-off run that carries it as
  [0, 128) and [128, 228); so do B's first two pages in every layer.
* Under pressure every request finishes, registered pages keep their bytes until evicted, first-token logits agree with the cache-off run to
  a cosine of 0.99; captured steps equal eager ones with no host synchronisation; Llama-3-8B with a shared system prompt hits."""
import random

import pytest
import torch

from tests.kv_pool_oracle import min_pages
from tests.prefix_cache_oracle import PAGE_REGISTERED, PrefixCacheOracle
from tests.test_gpu_inflight import _Device, _reason, _runner, _submit
from tests.test_gpu_kv_pool import _fill_random, _reqs, _serve_watch
from tests.test_oracle_prefix_cache import drive_shared

pytestmark = pytest.mark.gpu


def test_schedule_matches_oracle(dev):
    Bn, Q, Cn, ctx, Tn, L = 5, 7, 64, 200, 40, 2
    P = min_pages(ctx, Tn) * 2
    o = PrefixCacheOracle(Bn, Q, Cn, Tn, ctx, P, min_pages(ctx, Tn) + 1, layers=L)
    d = _Device(dev, Bn, Q, Cn, ctx, Tn, P, L, cache=True)
    drive_shared([o, d], 11, Bn, Q, Cn, ctx, Tn, 30, vocab=50, check=lambda step, plans: d.check(o, plans[0], step))
    assert o.hit_pages > 0 and o.evictions > 0 and o.duplicates > 0 and o.preemptions > 0, o.cache_counters()
    assert any(o.ref[q] == 0 for q in o.lru)


# ---------------------------------------------------------------------------------------------------------------------------------------------
B, CTX, T = 4, 100, 100
C = B * (CTX + T)
BLOCKS = (max(CTX + T + 1, CTX + T - 1 + C) + 63) // 64


def test_no_sharing_matches_the_pool(dev):
    """Prompts share no full page, the pools start with random bytes: the cache runner equals the pool runner bit for bit."""
    reqs = _reqs(14, 41)
    step = lambda r: r.inflight_forward(True, logprobs=1)
    res, stats = [], []
    for cache in (False, True):
        run = _runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=6, kv_pool_pages=B * BLOCKS, prefix_cache=cache)
        _fill_random(run, 5)
        res.append(_serve_watch(run, reqs, dev, step))
        stats.append(run.pool_stats())
    for i in range(len(reqs)):
        assert res[1][i][1:] == res[0][i][1:], i
    assert stats[1].preemptions == stats[0].preemptions and stats[1].starts == stats[0].starts == len(reqs)
    assert run.prefix_cache_stats().hit_pages == 0 and run.prefix_cache_stats().registrations > 0


def _page_bytes(run, pages):
    return torch.stack([torch.stack([run.kpools[li][pages], run.vpools[li][pages]]) for li in range(run.L)])


def test_exact_hit_matches_chunked_prefill(dev):
    """A's prompt is 128 tokens (two pages, one 128-row query block) and C = 128; B = A + 100 tokens arrives after A's prompt is cached.
    With the cache B computes 100 tokens over A's pages; without it B is carried as [0, 128) and [128, 228).  Tokens, reasons,
    log-probabilities and B's first two pages in every layer are equal bit for bit."""
    rng = random.Random(5)
    A = [rng.randrange(1024) for _ in range(128)]
    reqs = [dict(prompt=A, max_tokens=30, eos=-1, stop=[]), dict(prompt=A + [rng.randrange(1024) for _ in range(100)], max_tokens=30, eos=-1, stop=[])]
    res, first_pages = [], []
    for cache in (False, True):
        run = _runner(dev, ctx=256, max_new_tokens=40, prompt_tokens=128, inflight=4, kv_pool_pages=64, prefix_cache=cache)
        _fill_random(run, 7)
        done, pages = {}, []
        _submit(run, [reqs[0]], dev)
        run.inflight_forward(True, logprobs=1)  # A's whole prompt
        _submit(run, [reqs[1]], dev)
        for _ in range(200):
            run.inflight_forward(True, logprobs=1)
            req, phase = run.i_rows.request.tolist(), run.i_rows.phase.tolist()
            if not pages and 1 in req and phase[req.index(1)] == 2:
                b = req.index(1)
                pages = run.i_pool.pages[b, :2].tolist()
                first_pages.append(_page_bytes(run, pages).clone())
            for e in run.poll(logprobs=True).finished:
                done[e[0]] = e
            if len(done) == 2:
                break
        res.append(done)
        if cache:
            st = run.prefix_cache_stats()
            assert st.hit_pages == 2 and st.hit_tokens == 128
    assert res[0] == res[1]
    assert torch.equal(first_pages[0], first_pages[1])


def _shared_reqs(n, seed, system_len=150, ctx=CTX + 100):
    rng = random.Random(seed)
    system = [rng.randrange(1024) for _ in range(system_len)]
    out = []
    for i in range(n):
        tail = [rng.randrange(1024) for _ in range(rng.randint(1, ctx - system_len))]
        prompt = system + tail if i % 4 != 3 else [rng.randrange(1024) for _ in range(rng.randint(1, ctx))]
        out.append(dict(prompt=prompt, max_tokens=rng.randint(1, T), eos=rng.choice([-1, rng.randrange(1024)]), stop=rng.sample(range(1024), 2)))
    return out


def test_pressure_keeps_registered_pages_and_finishes(dev):
    ctx = CTX + 100
    reqs = _shared_reqs(16, 3, ctx=ctx)
    first = []
    for cache in (False, True):
        run = _runner(dev, ctx=ctx, max_new_tokens=T, prompt_tokens=256, inflight=8, kv_pool_pages=min_pages(ctx, T) + 3, prefix_cache=cache)
        logits, snap = {}, {}

        def watch(r):
            req, rows = r.i_rows.request.tolist(), r.i_plan.logit_rows.tolist()
            for b in range(B):
                if rows[b] >= B and req[b] >= 0 and req[b] not in logits:
                    logits[req[b]] = r.last_logits[b].float().clone()
            free, held = int(r.i_pool.counters[0]), r.i_pool.count.tolist()
            if r.i_cache is None:
                return
            state, epoch = r.i_cache.state.tolist(), r.i_cache.epoch.tolist()
            ev = int(r.i_cache.counters[2])
            held_pages = {q for b, n in enumerate(held) for q in r.i_pool.pages[b, :n].tolist()}
            assert free + ev + len(held_pages) == r.kv_pool_pages
            for q in range(r.kv_pool_pages):
                if state[q] != PAGE_REGISTERED:
                    snap.pop(q, None)
                    continue
                now = _page_bytes(r, [q])
                if q in snap and snap[q][0] == epoch[q]:
                    assert torch.equal(snap[q][1], now), q
                else:
                    snap[q] = (epoch[q], now.clone())

        got = _serve_watch(run, reqs, dev, lambda r: r.inflight_forward(True), watch=watch)
        for i, r in enumerate(reqs):
            toks, reason = got[i][1], got[i][2]
            assert 1 <= len(toks) <= r["max_tokens"] and reason == _reason(toks, r), i
        first.append(logits)
        if cache:
            st, ps = run.prefix_cache_stats(), run.pool_stats()
            assert st.hit_pages > 0 and st.evictions > 0 and ps.preemptions > 0, (st, ps)
            assert ps.free_pages + st.evictable_pages == run.kv_pool_pages
    for i in range(len(reqs)):
        cos = torch.nn.functional.cosine_similarity(first[0][i], first[1][i], dim=0).item()
        assert cos >= 0.99, (i, cos)


def test_captured_equals_eager_with_hits(dev):
    from tests.test_gpu_inflight import _serve

    ctx = CTX + 100
    reqs = _shared_reqs(12, 9, ctx=ctx)
    res, stats = [], []
    for captured in (False, True):
        run = _runner(dev, ctx=ctx, max_new_tokens=T, prompt_tokens=256, inflight=6, kv_pool_pages=min_pages(ctx, T) + 3, prefix_cache=True)
        if captured:
            run.capture_inflight(True)
            run.capture_inflight(False)
        k = [0]

        def step(r):
            mixed = k[0] % 3 != 2
            k[0] += 1
            (r.inflight_step if captured else r.inflight_forward)(mixed)

        res.append(_serve(run, reqs, dev, step, nosync=True))
        stats.append((run.pool_stats(), run.prefix_cache_stats()))
    assert res[0] == res[1] and stats[0] == stats[1]
    assert stats[0][1].hit_pages > 0 and stats[0][1].evictions > 0


def test_llama3_8b_shared_system_prompt_under_pressure(dev):
    with torch.no_grad():
        ctx, Tn = 192, 32
        run = _runner(dev, model="llama-3-8b", batch=4, ctx=ctx, max_new_tokens=Tn, prompt_tokens=256, inflight=5,
                      kv_pool_pages=min_pages(ctx, Tn) + 2, prefix_cache=True)
        rng = random.Random(17)
        system = [rng.randrange(128256) for _ in range(128)]
        reqs = [dict(prompt=system + [rng.randrange(128256) for _ in range(rng.randint(1, 64))], max_tokens=rng.randint(1, Tn), eos=-1, stop=[])
                for _ in range(10)]

        def conserved(r):
            held = {q for b, n in enumerate(r.i_pool.count.tolist()) for q in r.i_pool.pages[b, :n].tolist()}
            assert int(r.i_pool.counters[0]) + int(r.i_cache.counters[2]) + len(held) == r.kv_pool_pages

        got = _serve_watch(run, reqs, dev, lambda r: r.inflight_forward(True), watch=conserved)
        for i, r in enumerate(reqs):
            toks, reason = got[i][1], got[i][2]
            assert 1 <= len(toks) <= r["max_tokens"] and reason == _reason(toks, r), i
        assert run.prefix_cache_stats().hit_pages > 0
