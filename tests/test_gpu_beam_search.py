"""GPU: beam search -- backend.beam_select against tests/beam_oracle.py, backend.beam_reorder against a torch gather-and-copy, and
DecodeRunner(beam_width=W) end to end (oracle in the loop, a torch-reordered twin with bitwise equal logits, W = 1 against greedy
generation, captured against eager, unchanged draws, and the shared-prefix route)."""
import numpy as np
import pytest
import torch

from tests import beam_oracle as bo

pytestmark = pytest.mark.gpu
F32 = np.float32


def _candidates(rng, B, W, vocab, nan_p=0.1, short_p=0.2):
    C = 2 * W
    ids = np.full((B, C), -1, np.int64)
    lps = np.full((B, C), np.nan, F32)
    for b in range(B):
        if rng.random() < nan_p:
            continue
        i = rng.choice(vocab, size=C, replace=False).astype(np.int64)
        lp = -(rng.integers(0, 12, C) * F32(0.25) + F32(0.03125) * rng.integers(0, 2, C)).astype(F32)
        o = np.lexsort((i, -lp))
        ids[b], lps[b] = i[o], lp[o]
        if rng.random() < short_p:
            k = int(rng.integers(1, C))
            ids[b, k:], lps[b, k:] = -1, -np.inf
    return ids, lps


def _to_dev(st, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in st.items()}


def _gpu_select(st, prm, ids, lps, dev):
    from qserve_b200 import backend

    d = _to_dev(st, dev)
    pool = backend.BeamPool(d["pool_tokens"], d["pool_len"], d["pool_cum"], d["pool_score"], d["pool_count"])
    p = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in prm.items() if k != "max_model_len"}
    backend.beam_select(torch.from_numpy(ids).to(dev), torch.from_numpy(lps).to(dev), d["live"], d["cum"], d["seq_lens"], d["context_lens"],
                        d["tokens"], d["parents"], d["prompt_lens"], d["history"], p["length_penalty"], p["early_stopping"], p["eos"], p["stop_ids"],
                        p["budget"], d["done"], pool, prm["max_model_len"])
    return {k: v.cpu().numpy() for k, v in d.items()}


def _same_beams(a, b, check_cum=True):
    """Equal beam state: done, live, parents, the live slots' tokens and cum bits, lengths."""
    live = a["live"].astype(bool)
    ok = all(np.array_equal(a[k], b[k]) for k in ("done", "live", "parents", "seq_lens", "context_lens"))
    ok = ok and np.array_equal(a["tokens"][live], b["tokens"][live])
    return ok and (not check_cum or np.array_equal(a["cum"][live].view(np.uint32), b["cum"][live].view(np.uint32)))


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("lp", [1.0, 0.0, 0.5, 2.0, -1.0])
@pytest.mark.parametrize("es", [0, 1, 2])
def test_beam_select_matches_oracle(dev, W, lp, es):
    """Every step starts the kernel and the oracle from the same (oracle) state.  At length_penalty 0 and 1 every request matches bitwise; at
    other penalties a request may differ only where the oracle's deciding comparison was a near tie (beam_oracle.NEAR_TIE)."""
    exact, excused = lp in (0.0, 1.0), 0
    for seed in range(3):
        rng = np.random.default_rng(100 * W + 10 * seed + es)
        R, T, vocab = 3, int(rng.integers(3, 10)), 2 * W + 4
        P0 = [int(x) for x in rng.integers(1, 80, R)]
        stops = np.full((R, 8), -1, np.int64)
        stops[:, 0] = rng.integers(0, vocab, R)
        prm = bo.params(R, T, 70, lp, es, eos=int(rng.integers(0, vocab)), stop_ids=stops)
        prm["budget"] = rng.integers(1, T + 1, R).astype(np.int32)
        st = bo.init_state(P0, W, T, max(P0) + T + 2)
        for _ in range(12):
            ids, lps = _candidates(rng, R * W, W, vocab)
            margins = []
            want = bo.select(st, prm, ids, lps, margins)
            got = _gpu_select(st, prm, ids, lps, dev)
            bad = bo.mismatched(got, want, exact)
            assert not bad if exact else all(margins[r] <= bo.NEAR_TIE for r in bad), (seed, W, lp, es, bad, [margins[r] for r in bad])
            excused += len(bad)
            st = bo.reorder_history(want)
            if st["done"].all():
                break
    assert excused <= 2, f"{excused} requests decided differently at near ties"


def test_early_stopping_never_at_negative_length_penalty(dev):
    """early_stopping 2 with length_penalty <= 0 bounds the best running child at its current length, not at the maximum length: the case
    of test_oracle_beam.guard_case decides differently under the two rules, far from any near tie."""
    from tests.test_oracle_beam import guard_case

    st, prm, ids, lps = guard_case()
    want = bo.select(st, prm, ids, lps)
    got = _gpu_select(st, prm, ids, lps, dev)
    assert bo.mismatched(got, want, exact=False) == [] and got["done"][0] == 0


def _page_pools(L, B, blocks, Hkv, bits, dev, gen):
    """One pool per (layer, K / V) with B * blocks pages of random bytes, and each row's own table."""
    spt = Hkv * 128 * bits // 8
    page_bytes = 64 * spt + Hkv * 64 * 4
    pools = [[torch.randint(0, 256, (B * blocks, page_bytes), dtype=torch.uint8, device=dev, generator=gen) for _ in range(2)] for _ in range(L)]
    blk = torch.arange(B * blocks, device=dev, dtype=torch.int64).view(B, blocks)
    tables = torch.stack([torch.stack([p[0].data_ptr() + blk * page_bytes, p[1].data_ptr() + blk * page_bytes], dim=1) for p in pools]).contiguous()
    return pools, tables, spt, page_bytes


def _torch_reorder(tables, parents, ctx_lens, prompt_lens, tokens, history, W):
    """The table and history part of the reorder by torch gathers, on clones."""
    B = tables.shape[1]
    old_t, tables, old_h, history = tables.clone(), tables.clone(), history.clone(), history.clone()
    par, P_all, P0_all = parents.tolist(), (ctx_lens - 1).tolist(), prompt_lens.tolist()
    for s in range(B):
        p, P, P0 = par[s], P_all[s - s % W], P0_all[s]  # one P per request: its first slot's
        if not s - s % W <= p < s - s % W + W:
            continue
        if p != s:
            tables[:, s, :, : P // 64] = old_t[:, p, :, : P // 64]
            history[s, P0:P] = old_h[p, P0:P]
        history[s, P] = tokens[s]
    return tables, history


@pytest.mark.parametrize("bits", [4, 8])
def test_beam_reorder_matches_torch(dev, bits):
    from qserve_b200 import backend

    gen = torch.Generator(device=dev).manual_seed(5)
    L, W, R, blocks, Hkv = 3, 4, 3, 4, 2
    B = R * W
    pools, tables, spt, page_bytes = _page_pools(L, B, blocks, Hkv, bits, dev, gen)
    # swap + self, a 3-cycle + dead, repeats of one parent
    parents = torch.tensor([1, 0, 2, 3, 5, 6, 4, -1, 9, 9, 9, 8], dtype=torch.int32, device=dev)
    P = [64 * 2 + 1] * 4 + [64 * 1 + 63] * 4 + [64 * 3] * 4  # P % 64 in {1, 63, 0}
    ctx = torch.tensor([x + 1 for x in P], dtype=torch.int32, device=dev)
    P0 = torch.tensor([70] * 4 + [5] * 4 + [100] * 4, dtype=torch.int32, device=dev)
    tokens = torch.randint(0, 1000, (B,), dtype=torch.int64, device=dev, generator=gen)
    history = torch.randint(0, 1000, (B, 260), dtype=torch.int64, device=dev, generator=gen)
    before = [[p.clone() for p in lp] for lp in pools]
    want_t, want_h = _torch_reorder(tables, parents, ctx, P0, tokens, history, W)
    old_t = tables.clone()
    backend.beam_reorder(tables, parents, ctx, P0, tokens, history, W, Hkv, 64, spt, bits == 4)
    torch.cuda.synchronize()
    assert torch.equal(tables, want_t), "block tables differ"
    assert torch.equal(history, want_h), "history differs"
    # pages: the child's own tail page gets the parent's slots 0 .. t - 1 (codes, scale, zero of every head); every other byte is unchanged
    kRow = 128 * bits // 8
    code = 64 * spt
    want = [[p.clone() for p in lp] for lp in before]
    for s in range(B):
        p, Ps = int(parents[s]), P[s]
        n, t = Ps // 64, Ps % 64
        if p < 0 or p == s or t == 0:
            continue
        for li in range(L):
            for kv in range(2):
                pidx = (int(old_t[li, p, kv, n]) - pools[li][kv].data_ptr()) // page_bytes
                cidx = (int(old_t[li, s, kv, n]) - pools[li][kv].data_ptr()) // page_bytes
                src, dst = before[li][kv][pidx], want[li][kv][cidx]
                for h in range(Hkv):
                    o = h * 64 * kRow
                    dst[o: o + t * kRow] = src[o: o + t * kRow]
                    for row in range(2):
                        m = code + (row * Hkv + h) * 128
                        dst[m: m + 2 * t] = src[m: m + 2 * t]
    for li in range(L):
        for kv in range(2):
            assert torch.equal(pools[li][kv], want[li][kv]), f"layer {li} kv {kv}: page bytes differ"


# ---------------------------------------------------------------------------------------------------------------------------------------------
# the runner
# ---------------------------------------------------------------------------------------------------------------------------------------------
CTX, T = 200, 96


def _runner(dev, W, R, **kw):
    from qserve_b200.decode import DecodeRunner

    return DecodeRunner("tiny", "w4a8kv4", batch=R * W, ctx=CTX, device=dev, seed=3, prompt_tokens=R * CTX, max_new_tokens=T, beam_width=W, **kw)


def _prompts(dev, R, seed=13):
    g = torch.Generator(device=dev).manual_seed(seed)
    lens = torch.randint(60, 131, (R,), device=dev, generator=g).int()
    return torch.randint(0, 1024, (R, CTX), device=dev, generator=g), lens


def _set_params(run, lp=1.0, es=0, eos=-1, budget=80):
    run.b_length_penalty.fill_(lp)
    run.b_early_stopping.fill_(es)
    run.b_eos.fill_(eos)
    run.b_budget.fill_(budget)
    run.s_repetition.fill_(1.2)
    run.s_presence.fill_(0.3)
    run.s_frequency.fill_(0.1)


def _runner_state(run):
    st = {"live": run.b_live, "cum": run.b_cum, "seq_lens": run.s_seq_lens, "context_lens": run.context_lens, "tokens": run.tokens_in,
          "parents": run.b_parent, "prompt_lens": run.s_prompt_lens, "history": run.s_history, "done": run.b_done, "pool_tokens": run.b_pool.tokens,
          "pool_len": run.b_pool.length, "pool_cum": run.b_pool.cum, "pool_score": run.b_pool.score, "pool_count": run.b_pool.count}
    return {k: v.cpu().numpy() for k, v in st.items()}


def _oracle_params(run):
    R = run.batch // run.beam_width
    prm = bo.params(R, T, run.max_model_len, run.b_length_penalty.cpu().numpy(), run.b_early_stopping.cpu().numpy(), run.b_eos.cpu().numpy(),
                    run.b_stop.cpu().numpy())
    prm["budget"] = run.b_budget.cpu().numpy()
    return prm


def _check_oracle_step(run, st, prm):
    cand = run.b_top_ids.cpu().numpy(), run.b_top_logprobs.cpu().numpy()
    want = bo.step(st, prm, *cand)
    got = _runner_state(run)
    assert _same_beams(got, want) and bo.same_pool(got, want)
    assert np.array_equal(got["history"], want["history"])
    return want


def _finish_children(runs, src):
    """Set every request's stop ids (and eos) in all runners to the tokens of its first W + 1 children under the candidates src holds before
    its selection, so at least W + 1 of the 2 W children finish and at most W - 1 run on: slots die."""
    W = src.beam_width
    ids, lps = src.b_top_ids.cpu().numpy(), src.b_top_logprobs.cpu().numpy()
    live, cum = src.b_live.cpu().numpy(), src.b_cum.cpu().numpy()
    stop = np.full((src.batch // W, _MAX_STOPS + 1), -1, np.int64)
    for r in range(src.batch // W):
        cands = sorted((F32(cum[b] + lps[b, k]), b, k) for b in range(r * W, r * W + W) if live[b] for k in range(2 * W) if ids[b, k] >= 0)
        cands.sort(key=lambda c: (-float(c[0]), c[1], c[2]))
        toks = []
        for _, b, k in cands[: W + 1]:
            if int(ids[b, k]) not in toks:
                toks.append(int(ids[b, k]))
        stop[r, : len(toks)] = toks
    for run in runs:
        run.b_stop.copy_(torch.from_numpy(stop[:, :_MAX_STOPS]))
        run.b_eos.copy_(torch.from_numpy(stop[:, _MAX_STOPS]))


_MAX_STOPS = 8


@pytest.mark.parametrize("W, stops", [(1, False), (4, False), (8, False), (4, True), (8, True)])
@pytest.mark.parametrize("penalties", [False, True])
def test_runner_follows_the_oracle_and_a_torch_reordered_twin(dev, W, stops, penalties):
    """(a) each step the oracle consumes the runner's own candidates and must reach the runner's state; (b) a twin that re-parents with torch
    ops gives bitwise equal logits on every step, so the pages realise every beam's lineage.  Without stop ids every request keeps W running
    beams up to the budget and crosses page boundaries.  With stops, every sixth step's stop ids and eos are the tokens of each request's first
    W + 1 children (early_stopping "never"): at least W + 1 children finish, slots die mid-search, keep being computed while dead, and are
    revived on the next step by taking another beam's tables, tail pages and history."""
    R = 16 // W if W > 1 else 4
    with torch.no_grad():
        prompts, lens = _prompts(dev, R)
        run, twin = _runner(dev, W, R), _runner(dev, W, R)
        for r in (run, twin):
            _set_params(r, lp=1.0, es=2 if stops else 0, budget=80)
        # the twin: same prefill, select by the kernel, reorder by torch; it steps first, so with stops its tail sets every sixth step's stop
        # ids in both runners from that step's candidates before either selects
        twin._beam_tail = lambda logits, t=twin: _twin_tail(t, logits)
        twin.beam_start(prompts, lens, penalties=penalties)
        run.beam_start(prompts, lens, penalties=penalties)
        st = bo.init_state(lens.tolist(), W, T, run.s_history.size(1), prompts.cpu().numpy())
        st = _check_oracle_step(run, st, _oracle_params(run))
        assert torch.equal(run.last_logits, twin.last_logits)
        steps, died, revived = 0, 0, 0
        while steps < 85 and not bool(run.b_done.all()):
            before = st["live"].copy()
            if stops:
                twin._test_hook = (lambda t=twin: _finish_children((run, twin), t)) if steps % 6 == 2 else None
                if steps % 6 == 3:
                    for r in (run, twin):
                        r.b_stop.fill_(-1)
                        r.b_eos.fill_(-1)
            twin.beam_forward(penalties)
            run.beam_forward(penalties)
            assert torch.equal(run.last_logits, twin.last_logits), f"step {steps}: logits differ from the torch-reordered twin"
            st = _check_oracle_step(run, st, _oracle_params(run))
            active = np.repeat(st["done"] == 0, W)
            died += int(((before == 1) & (st["live"] == 0) & active).sum())
            revived += int(((before == 0) & (st["live"] == 1)).sum())
            steps += 1
        if not stops:
            assert bool(run.b_done.all()) and steps == 79
            res = run.beam_results()
            assert all(len(x) == W and all(len(h[0]) == 80 for h in x) for x in res)
        else:
            assert died >= 2 and revived >= 2, (died, revived)


def _twin_tail(run, logits):
    """beam_tail with the reorder done by torch ops: tables gathered, tail pages cloned, history copied."""
    from qserve_b200 import backend as _ext

    W = run.beam_width
    _ext.logprobs_rows(logits, run.tokens_in, 2 * W, run.b_logprob, run.b_top_ids, run.b_top_logprobs)
    if getattr(run, "_test_hook", None) is not None:
        run._test_hook()
    _ext.beam_select(run.b_top_ids, run.b_top_logprobs, run.b_live, run.b_cum, run.s_seq_lens, run.context_lens, run.tokens_in, run.b_parent,
                     run.s_prompt_lens, run.s_history, run.b_length_penalty, run.b_early_stopping, run.b_eos, run.b_stop, run.b_budget, run.b_done,
                     run.b_pool, run.max_model_len)
    par, P_all, P0_all = run.b_parent.tolist(), (run.context_lens - 1).tolist(), run.s_prompt_lens.tolist()
    old_t, old_h = run.block_tables.clone(), run.s_history.clone()
    pools = [run.kpools + run.kpools_gen, run.vpools + run.vpools_gen]
    bases = [[(p.data_ptr(), p) for p in ps] for ps in pools]

    def page(kv, addr):
        for b, p in bases[kv]:
            if b <= addr < b + p.numel():
                return p[(addr - b) // run.page_bytes]
        raise AssertionError("page address outside the pools")

    copies = []
    for s in range(run.batch):
        p, P, P0 = par[s], P_all[s], P0_all[s]
        if p < 0 or p == s:
            continue
        n = P // 64
        run.block_tables[:, s, :, :n] = old_t[:, p, :, :n]
        if P % 64:
            for li in range(run.L):
                for kv in range(2):
                    copies.append((page(kv, int(old_t[li, s, kv, n])), page(kv, int(old_t[li, p, kv, n])).clone()))
        run.s_history[s, P0:P] = old_h[p, P0:P]
    for dst, src in copies:
        dst.copy_(src)
    live = torch.tensor([x >= 0 for x in par], device=run.dev)
    cols = (run.context_lens - 1).long().unsqueeze(1)
    run.s_history.scatter_(1, cols, torch.where(live, run.tokens_in, run.s_history.gather(1, cols).squeeze(1)).unsqueeze(1))


def test_width_one_is_greedy(dev):
    """(c) W = 1, early_stopping 1: the best hypothesis is generate_forward's greedy output with the same eos, or of max_tokens tokens
    without one.  With vLLM's rules an eos among a step's two candidates (even second) ends a W = 1 search, so each request's eos is a token
    of its own greedy output that is not among the two candidates of any earlier step (found by a first greedy run with logprobs = 2)."""
    from qserve_b200.decode import DecodeRunner

    R, budget = 4, 40
    with torch.no_grad():
        greedy = DecodeRunner("tiny", "w4a8kv4", batch=R, ctx=CTX, device=dev, seed=3, prompt_tokens=R * CTX, max_new_tokens=T, generate=True)
        greedy.g_budget.fill_(budget)
        prompts, lens = _prompts(dev, R)
        greedy.prefill(prompts, lens, logprobs=2)
        for _ in range(budget - 1):
            greedy.generate_forward(1, logprobs=2)
        top2 = greedy.g_top_view(2)[0].cpu().numpy()
        eos = []
        for r in range(R):
            n = int(lens[r])
            toks, seen = greedy.s_history[r, n: n + budget].tolist(), set()
            pick = -1
            for i, t in enumerate(toks):
                if i >= 5 and t not in seen:
                    pick = t
                    break
                seen.update(int(x) for x in top2[r, n + i])
            eos.append(pick)
        assert sum(e >= 0 for e in eos) >= 2, eos
        run = _runner(dev, 1, R)
        _set_params(run, es=1, budget=budget)
        run.b_eos.copy_(torch.tensor(eos, dtype=torch.int64, device=dev))
        run.beam_start(prompts, lens)
        for _ in range(budget - 1):
            if bool(run.b_done.all()):
                break
            run.beam_forward()
        assert bool(run.b_done.all())
        greedy.g_eos.copy_(run.b_eos)
        greedy.prefill(prompts, lens)
        for _ in range(budget - 1):
            greedy.generate_forward(1)
        res = run.beam_results(1)
        for r in range(R):
            n, m = int(lens[r]), int(greedy.s_seq_lens[r])
            want = greedy.s_history[r, n: m].tolist()
            assert res[r][0][0] == want, f"request {r}"
            assert (want[-1] == eos[r]) == (eos[r] >= 0), f"request {r}: the greedy output does not end at its eos"


def test_captured_equals_eager(dev):
    """(d) the captured beam_step equals eager beam_forward."""
    W, R = 4, 4
    with torch.no_grad():
        eager, graph = _runner(dev, W, R), _runner(dev, W, R)
        for r in (eager, graph):
            _set_params(r, lp=0.5, es=2, eos=11, budget=60)
        graph.capture_beam(penalties=True)
        prompts, lens = _prompts(dev, R, seed=17)
        for r in (eager, graph):
            r.beam_start(prompts, lens, penalties=True)
        for _ in range(50):
            eager.beam_forward(True)
            graph.beam_step(True)
        a, b = _runner_state(eager), _runner_state(graph)
        for k in a:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
        # tables hold absolute page addresses: compare each runner's against its own pages
        assert torch.equal(eager.block_tables - eager.own_tables, graph.block_tables - graph.own_tables)


def test_beam_width_zero_draws_the_same(dev):
    """(e) weights and pages of a beam runner are those of beam_width = 0."""
    from qserve_b200.decode import DecodeRunner

    with torch.no_grad():
        a = _runner(dev, 4, 2)
        b = DecodeRunner("tiny", "w4a8kv4", batch=8, ctx=CTX, device=dev, seed=3, prompt_tokens=2 * CTX, max_new_tokens=T)
        assert all(torch.equal(x, y) for x, y in zip(a.kpools + a.vpools, b.kpools + b.vpools))
        assert torch.equal(a.embed, b.embed) and torch.equal(a.lm_head, b.lm_head)
        assert all(torch.equal(x["qkv"].qweight, y["qkv"].qweight) for x, y in zip(a.layers, b.layers))


def test_shared_prefix_route(dev, monkeypatch):
    """4. shared_prefix=True with the route forced: entries below S stay equal across each group after every step, and the oracle holds."""
    from qserve_b200 import decode

    monkeypatch.setattr(decode, "SHARED_PREFIX_MIN_PAGES", 1)
    W, R = 4, 4
    with torch.no_grad():
        run = _runner(dev, W, R, shared_prefix=True)
        _set_params(run, es=0, eos=3, budget=70)
        prompts, lens = _prompts(dev, R, seed=23)
        lens = lens.clamp(min=64)
        run.beam_start(prompts, lens)
        assert run._sp_layout is not None, "the shared route was not taken"
        S = [int(x) // 64 for x in lens.tolist()]
        st = bo.init_state(lens.tolist(), W, T, run.s_history.size(1), prompts.cpu().numpy())
        prm = _oracle_params(run)
        st = _check_oracle_step(run, st, prm)
        for _ in range(70):
            if bool(run.b_done.all()):
                break
            run.beam_forward()
            st = _check_oracle_step(run, st, prm)
            for r in range(R):
                t = run.block_tables[:, r * W: r * W + W, :, : S[r]]
                assert torch.equal(t, t[:, :1].expand_as(t)), f"request {r}: shared entries diverged"
