"""GPU: in-flight batching over a shared KV page pool (DecodeRunner(inflight=Q, kv_pool_pages=P), qs_inflight_schedule_pool, DESIGN.md 3.12).

* The schedule kernel equals tests/kv_pool_oracle.py after every call of a scripted run that preempts decode and prefill rows, preempts a
  requester itself and blocks starts: row state, plan, free stack, page lists, counters and every layer's table entries.
* Without pressure (P = B x blocks, the pool first filled with random bytes) every request gets the own-pages runner's tokens, reasons and
  log-probabilities bit for bit, with pages recycled across requests.
* Under pressure every request finishes; requests never preempted keep those tokens bit for bit, preempted ones up to the preemption; a
  recomputed row's layer-0 pages equal a whole-prompt prefill of its history and its completing logits agree to a cosine of 0.99.
* Captured steps equal eager ones with preemptions, with no host synchronisation between submit and poll; Llama-3-8B under pressure."""
import pytest
import torch

from tests.kv_pool_oracle import KvPoolOracle, min_pages
from tests.test_gpu_inflight import _Device, _reason, _runner, _script, _submit
from tests.test_oracle_kv_pool import _drive

pytestmark = pytest.mark.gpu

B, CTX, T = 4, 100, 100
C = B * (CTX + T)  # every prefill, recomputations included, is carried in one piece, so a row's bits do not depend on the schedule
BLOCKS = (max(CTX + T + 1, CTX + T - 1 + C) + 63) // 64


def test_schedule_matches_oracle(dev):
    """The kernel against the oracle after every call, with random commits in between, at a pool small enough for every event kind."""
    Bn, Q, Cn, ctx, Tn, P, L = 6, 7, 40, 150, 60, 7, 3
    o = KvPoolOracle(Bn, Q, Cn, Tn, ctx, P, min_pages(ctx, Tn) + 1, layers=L)
    d = _Device(dev, Bn, Q, Cn, ctx, Tn, P, L)
    _drive([o, d], 31, Bn, Q, Cn, ctx, Tn, 40, vocab=400, check=lambda step, plans: d.check(o, plans[0], step))
    assert all(v > 0 for v in o.events.values()), o.events
    for r, (toks, reason) in o.outputs.items():
        s = r % Q
        if r >= len(o.requests) - Q:  # slots not reused since
            assert d.out.tokens[s, : len(toks)].tolist() == toks and int(d.out.length[s]) == len(toks) and int(d.out.reason[s]) == reason


# ---------------------------------------------------------------------------------------------------------------------------------------------
def _pool_state(run):
    """(free pages, {row: page list}) read back from the device."""
    p = run.i_pool
    top = int(p.counters[0])
    return p.free[:top].tolist(), {b: p.pages[b, :n].tolist() for b, n in enumerate(p.count.tolist())}


def _conserved(run):
    free, held = _pool_state(run)
    pages = free + [x for v in held.values() for x in v]
    assert sorted(pages) == list(range(run.kv_pool_pages)), "a page is lost or held twice"


def _serve_watch(run, reqs, dev, step, watch=None, max_steps=3000):
    """Submit reqs as queue room allows and step until every request is polled; watch(run) runs after every step.  Returns {id: entry}."""
    done, nxt = {}, 0
    for _ in range(max_steps):
        while nxt < len(reqs) and (nxt - run.inflight < 0 or (nxt - run.inflight) in done):
            _submit(run, [reqs[nxt]], dev)
            nxt += 1
        step(run)
        if watch:
            watch(run)
        for e in run.poll(logprobs=True).finished:
            done[e[0]] = e
        if len(done) == len(reqs):
            return done
    raise AssertionError("script did not finish")


def _fill_random(run, seed):
    """Random page bytes with finite fp16 scales and zeros, so that a read of a page no request wrote would show."""
    g = torch.Generator(device=run.dev).manual_seed(seed)
    cb = 64 * run.size_per_token
    for pool in run.kpools + run.vpools:
        pool.copy_(torch.randint(0, 256, pool.shape, dtype=torch.uint8, device=run.dev, generator=g))
        meta = pool[:, cb:].view(torch.float16)
        meta.copy_((torch.rand(meta.shape, device=run.dev, generator=g) * 4).half())


def _reqs(n, seed):
    return _script(n, CTX, T, 1024, seed=seed)


def _no_pressure(dev, reqs):
    """The own-pages in-flight runner and a pool of B x blocks pages, greedy with log-probabilities, on the same script."""
    step = lambda r: r.inflight_forward(True, logprobs=1)
    own = _serve_watch(_runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=6), reqs, dev, step)
    run = _runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=6, kv_pool_pages=B * BLOCKS)
    _fill_random(run, 5)
    pooled = _serve_watch(run, reqs, dev, step, watch=_conserved)
    return own, pooled, run


def test_no_pressure_matches_own_pages(dev):
    reqs = _reqs(14, 41)
    own, pooled, run = _no_pressure(dev, reqs)
    for i in range(len(reqs)):
        assert pooled[i][1:] == own[i][1:], i
    stats = run.pool_stats()
    assert stats.preemptions == 0 and stats.starts == len(reqs) and stats.free_pages == B * BLOCKS
    assert stats.peak_pages < B * BLOCKS  # the pool holds tokens, not worst cases


def test_pressure_finishes_and_recomputes(dev):
    """P = ceil((ctx + T + 1) / 64) for 4 rows: preemptions happen, every request ends by its stop rules; never-preempted requests keep
    the no-pressure tokens bit for bit, preempted ones up to their preemption; each recomputed row's completing step leaves layer-0 pages equal
    to a whole-prompt prefill of history[:target] and logits within cosine 0.99 of that prefill's."""
    from tests.test_gpu_prefill_runner import _slots

    reqs = _reqs(14, 41)
    want, _, _ = _no_pressure(dev, reqs)
    P = min_pages(CTX, T)
    run = _runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=6, kv_pool_pages=P)
    preempted: dict = {}   # request -> tokens generated before its first preemption
    recomputed = []        # (history[:target], layer-0 slot bytes, completing logits)
    prev = {}

    def watch(r):
        _conserved(r)
        phase, req, seq, plen = (t.tolist() for t in (r.i_rows.phase, r.i_rows.request, r.s_seq_lens, r.s_prompt_lens))
        target, rows = r.i_pool.target.tolist(), r.i_plan.logit_rows.tolist()
        for b in range(B):
            if req[b] >= 0 and prev.get(b) == (req[b], 2) and phase[b] == 1:
                preempted.setdefault(req[b], seq[b] - plen[b])
            if rows[b] >= B and target[b] > plen[b]:  # a recomputed row completed in this step
                n = target[b]
                pages = r.i_pool.pages[b, : (n + 63) // 64].tolist()
                recomputed.append((r.s_history[b, :n].clone(), _pool_slots(r, pages, n), r.last_logits[b].float().clone()))
            prev[b] = (req[b], phase[b])

    got = _serve_watch(run, reqs, dev, lambda r: r.inflight_forward(True, logprobs=1), watch=watch)
    stats = run.pool_stats()
    assert stats.preemptions > 0 and preempted and recomputed and stats.free_pages == P and stats.peak_pages <= P
    for i, r in enumerate(reqs):
        toks, reason = got[i][1], got[i][2]
        assert 1 <= len(toks) <= r["max_tokens"] and reason == _reason(toks, r), i
        assert reason != "budget" or len(toks) == r["max_tokens"], i
        if i in preempted:
            g = preempted[i]
            assert toks[:g] == want[i][1][:g], i
        else:
            assert got[i][1:] == want[i][1:], i
    ref = _runner(dev, ctx=CTX + T, max_new_tokens=T, prompt_tokens=B * (CTX + T))
    for hist, slots, logits in recomputed:
        n = hist.numel()
        p = torch.zeros((B, n), dtype=torch.int64, device=dev)
        p[0] = hist
        ref.prefill(p, torch.tensor([n] + [1] * (B - 1), dtype=torch.int32, device=dev))
        assert torch.equal(slots, _slots(ref, 0, n, layers=[0])), n
        cos = torch.nn.functional.cosine_similarity(logits, ref.last_logits[0].float(), dim=0).item()
        assert cos >= 0.99, (n, cos)


def _pool_slots(run, pages, n):
    """The bytes of slots 0 .. n - 1 of layer 0 through a pool page list, in the order of test_gpu_prefill_runner._slots."""
    kRow, cb = 128 * run.kv_bits // 8, 64 * run.size_per_token
    out = []
    for pool in (run.kpools[0], run.vpools[0]):
        for j, pg in enumerate(pages):
            s = min(64, n - 64 * j)
            page = pool[pg]
            out += [page[:cb].view(run.Hkv, 64, kRow)[:, :s].flatten(), page[cb:].view(2, run.Hkv, 128)[:, :, : 2 * s].flatten()]
    return torch.cat(out)


def test_captured_equals_eager_with_preemptions(dev):
    """Captured mixed and decode-only steps, interleaved, equal the eager sequence under pressure; no host synchronisation between submit and
    poll."""
    from tests.test_gpu_inflight import _serve

    reqs = _reqs(10, 43)
    res, pre = [], []
    for captured in (False, True):
        run = _runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=5, kv_pool_pages=min_pages(CTX, T))
        if captured:
            run.capture_inflight(True)
            run.capture_inflight(False)
        k = [0]

        def step(r):
            mixed = k[0] % 3 != 2
            k[0] += 1
            (r.inflight_step if captured else r.inflight_forward)(mixed)

        res.append(_serve(run, reqs, dev, step, nosync=True))
        pre.append(run.pool_stats())
        _conserved(run)
    assert res[0] == res[1] and pre[0] == pre[1] and pre[0].preemptions > 0


def test_pool_refuses_own_page_steps(dev):
    run = _runner(dev, ctx=CTX, max_new_tokens=T, prompt_tokens=C, inflight=4, kv_pool_pages=min_pages(CTX, T))
    p = torch.zeros((B, 8), dtype=torch.int64, device=dev)
    lens = torch.full((B,), 8, dtype=torch.int32, device=dev)
    for call in (lambda: run.prefill(p, lens), lambda: run.fork(0, 1), lambda: run.reset_generation(torch.zeros((B, CTX + 1), dtype=torch.int64, device=dev))):
        with pytest.raises(RuntimeError):
            call()


def test_llama3_8b_full_model_under_pressure(dev):
    """All 32 layers of Llama-3-8B W4A8KV4, 4 rows over a pool of ceil((ctx + T + 1) / 64) pages: every request finishes by its stop rules
    and the pages are conserved after every step."""
    with torch.no_grad():
        ctx, Tn = 64, 64
        run = _runner(dev, model="llama-3-8b", batch=4, ctx=ctx, max_new_tokens=Tn, prompt_tokens=4 * (ctx + Tn), inflight=5,
                      kv_pool_pages=min_pages(ctx, Tn))
        reqs = _script(8, ctx, Tn, 128256, seed=17)
        got = _serve_watch(run, reqs, dev, lambda r: r.inflight_forward(True), watch=_conserved)
        for i, r in enumerate(reqs):
            toks, reason = got[i][1], got[i][2]
            assert 1 <= len(toks) <= r["max_tokens"] and reason == _reason(toks, r), i
        stats = run.pool_stats()
        assert stats.free_pages == run.kv_pool_pages and stats.preemptions > 0
