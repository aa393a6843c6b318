"""GPU: in-flight batching in the decode runner (DecodeRunner(inflight=Q), qs_inflight_schedule, DESIGN.md 3.12).

* The schedule kernel equals tests/inflight_oracle.py bit for bit after every call of a scripted run whose rows end by eos, stop id and budget.
* Idle rows (length 0) of single_query_attention[_quant] and the padding slots of the chunk segment write no page byte and give zero rows.
* Greedy in-flight runs give every request the tokens, reasons and log-probabilities of a separate runner that prefills the prompt with
  prefill(chunk=C) and runs generate_forward(1), including rows reused by later requests; split prompts leave whole-prompt layer-0 pages.
* Captured steps equal eager ones, and inflight=0 changes nothing."""
import random

import pytest
import torch

from tests.inflight_oracle import InflightOracle, Request

pytestmark = pytest.mark.gpu

B, CTX, T = 4, 40, 8


def _runner(dev, model="tiny", precision="w4a8kv4", **kw):
    from qserve_b200.decode import DecodeRunner

    kw.setdefault("batch", B)
    kw.setdefault("ctx", CTX)
    kw.setdefault("max_new_tokens", T)
    return DecodeRunner(model, precision, device=dev, seed=3, generate=True, **kw)


def _script(n, ctx, T, vocab, seed, stops=True):
    rng = random.Random(seed)
    reqs = []
    for _ in range(n):
        ln = rng.randint(1, ctx)
        reqs.append(dict(prompt=[rng.randrange(vocab) for _ in range(ln)], max_tokens=rng.randint(1, T),
                         eos=rng.choice([-1, rng.randrange(vocab)]), stop=rng.sample(range(vocab), rng.randint(0, 3)) if stops else []))
    return reqs


def _submit(run, reqs, dev, **kw):
    width = max(len(r["prompt"]) for r in reqs)
    p = torch.tensor([r["prompt"] + [0] * (width - len(r["prompt"])) for r in reqs], dtype=torch.int64)
    return run.submit(p, [len(r["prompt"]) for r in reqs], max_tokens=[r["max_tokens"] for r in reqs], eos=[r["eos"] for r in reqs],
                      stop=[list(r["stop"]) for r in reqs], **kw)


def _serve(run, reqs, dev, step, max_steps=2000, logprobs=False, nosync=False, **kw):
    """Submit reqs as queue room allows, step(run) until every request is polled; returns {id: entry}.  nosync=True: submit and the step run
    under torch's sync debug mode "error", so any host synchronisation between two polls raises."""
    done, nxt = {}, 0
    for _ in range(max_steps):
        if nosync:
            torch.cuda.set_sync_debug_mode("error")
        try:
            while nxt < len(reqs) and (nxt - run.inflight < 0 or (nxt - run.inflight) in done):
                _submit(run, [reqs[nxt]], dev, **kw)
                nxt += 1
            step(run)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        for e in run.poll(logprobs=logprobs).finished:
            done[e[0]] = e
        if len(done) == len(reqs):
            return done
    raise AssertionError("script did not finish")


def _reason(toks, r):
    if r["eos"] >= 0 and toks[-1] == r["eos"]:
        return "eos"
    return "stop" if toks[-1] in r["stop"] else "budget"


def _reference(dev, reqs, C, penalties=False, logprobs=0, model="tiny", layers=None, **kw):
    """Every request through a separate runner of the same seed: prefill(chunk=C) of B prompts at a time, then generate_forward(1) to the same
    stop rule.  Returns [(tokens, reason, log-probabilities)]."""
    run = _runner(dev, model=model, prompt_tokens=C, layers=layers, **kw)
    out = []
    Bn = run.batch
    for i in range(0, len(reqs), Bn):
        grp = reqs[i:i + Bn]
        grp = grp + [grp[-1]] * (Bn - len(grp))
        width = max(len(r["prompt"]) for r in grp)
        p = torch.tensor([r["prompt"] + [0] * (width - len(r["prompt"])) for r in grp], dtype=torch.int64, device=dev)
        lens = torch.tensor([len(r["prompt"]) for r in grp], dtype=torch.int32, device=dev)
        run.g_budget.copy_(torch.tensor([r["max_tokens"] for r in grp], dtype=torch.int32))
        run.g_eos.copy_(torch.tensor([r["eos"] for r in grp], dtype=torch.int64))
        run.g_stop.copy_(torch.tensor([list(r["stop"]) + [-1] * (8 - len(r["stop"])) for r in grp], dtype=torch.int64))
        if penalties:
            run.s_repetition.fill_(1.3); run.s_presence.fill_(0.5); run.s_frequency.fill_(0.25)
        run.prefill(p, lens, chunk=C, penalties=penalties, logprobs=logprobs)
        for _ in range(T):
            run.generate_forward(1, penalties=penalties, logprobs=logprobs)
        for b, r in enumerate(reqs[i:i + Bn]):
            n0, n1 = int(lens[b]), int(run.s_seq_lens[b])
            toks = run.s_history[b, n0:n1].tolist()
            lp = run.g_logprob[b, n0:n1].tolist() if logprobs else None
            out.append((toks, _reason(toks, r), lp))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------------
def test_schedule_matches_oracle(dev):
    """The kernel against the oracle after every call: row state, plan, per-row vectors and outputs, with a plain commit of random tokens
    (spec_commit_stops) in between; requests end by eos, stop ids and budget; queue slots are reused."""
    from qserve_b200 import backend as ext

    Bn, Q, C, ctx, Tn, vocab = 6, 5, 20, 16, 6, 12
    H = ctx + 1 + Tn
    queue, rows, plan, out = ext.inflight_buffers(Bn, Q, C, ctx, Tn, dev)
    full = lambda shape, v, dt: torch.full(shape, v, dtype=dt, device=dev)
    history, plen, slen = full((Bn, H), -1, torch.int64), full((Bn,), 0, torch.int32), full((Bn,), 0, torch.int32)
    temp, topk, topp = full((Bn,), 1.0, torch.float32), full((Bn,), 1, torch.int32), full((Bn,), 1.0, torch.float32)
    rep, pres, freq = full((Bn,), 1.0, torch.float32), full((Bn,), 0.0, torch.float32), full((Bn,), 0.0, torch.float32)
    eos, stop, budget = full((Bn,), -1, torch.int64), full((Bn, 8), -1, torch.int64), full((Bn,), Tn, torch.int32)
    offs, fin, start, tin = full((Bn,), 7, torch.int64), full((Bn,), 0, torch.int32), full((Bn,), 0, torch.int32), full((Bn,), 0, torch.int64)
    logprob, ctxl = full((Bn, H), float("nan"), torch.float32), full((Bn,), 0, torch.int32)
    path, acc = full((Bn, 1), 0, torch.int32), full((Bn,), 1, torch.int32)
    o = InflightOracle(Bn, Q, C, Tn)
    rng = random.Random(7)
    reqs = _script(40, ctx, Tn, vocab, seed=11)
    nxt, reasons, prev = 0, set(), 0
    for step in range(400):
        while nxt < len(reqs) and rng.random() < 0.5 and (nxt - Q < 0 or (nxt - Q) in o.outputs):
            r = reqs[nxt]
            s = nxt % Q
            queue.prompts[s].fill_(-1)
            queue.prompts[s, : len(r["prompt"])] = torch.tensor(r["prompt"])
            queue.lens[s], queue.max_tokens[s], queue.eos[s] = len(r["prompt"]), r["max_tokens"], r["eos"]
            queue.stop[s] = torch.tensor(list(r["stop"]) + [-1] * (8 - len(r["stop"])))
            o.submit(Request(r["prompt"], r["max_tokens"], r["eos"], tuple(r["stop"])))
            nxt += 1
            queue.counters[1] = nxt
        cb = 0 if rng.random() < 0.15 else C
        ext.inflight_schedule(queue, rows, history, plen, slen, temp, topk, topp, rep, pres, freq, eos, stop, budget, offs, fin, start, tin,
                              logprob, plan, out, cb)
        want = o.schedule(cb)
        got = lambda t: t.tolist()
        assert got(rows.phase) == o.phase and got(rows.request) == o.row_req, step
        assert [d for d, ph in zip(got(rows.done), o.phase) if ph] == [d for d, ph in zip(o.done, o.phase) if ph]
        assert got(plan.cu_seqlens) == want.cu_seqlens and got(plan.chunk_lens) == want.chunk_lens, step
        assert got(plan.prefix_lens) == want.prefix_lens and got(plan.context_lens) == want.context_lens, step
        assert got(plan.tokens) == want.tokens and got(plan.padding_offset) == want.padding_offset, step
        assert got(plan.logit_rows) == want.logit_rows and got(fin) == o.finished, step
        assert got(queue.counters)[:3] == [o.head, o.tail, o.retired]
        for b in range(Bn):
            if o.row_req[b] >= 0:
                assert int(plen[b]) == o.prompt_lens[b] and int(slen[b]) == o.seq_lens[b] and int(budget[b]) == o.budget[b]
                assert int(eos[b]) == o.eos[b] and tuple(stop[b].tolist()) == o.stop[b]
                assert history[b, : o.seq_lens[b]].tolist() == o.history[b][: o.seq_lens[b]]
                if o.phase[b] == 2:
                    assert int(start[b]) == o.start_pos[b]
        ring = got(out.ids)
        for i in range(prev, len(o.ring)):
            r = o.ring[i]
            assert ring[i % Q] == r
            toks, reason = o.outputs[r]
            assert out.tokens[r % Q, : len(toks)].tolist() == toks and int(out.length[r % Q]) == len(toks) and int(out.reason[r % Q]) == reason
            reasons.add(reason)
        prev = len(o.ring)
        tok = torch.tensor([rng.randrange(vocab) for _ in range(Bn)], dtype=torch.int64, device=dev)
        ext.spec_commit(tok.view(Bn, 1), path, acc, tok, history, slen, plen, budget, eos, fin, start, ctxl, tin, stop_ids=stop)
        o.commit(tok.tolist())
        if len(o.outputs) == len(reqs):
            break
    assert len(o.outputs) == len(reqs) and reasons == {1, 2, 3}


@pytest.mark.parametrize("int4", [True, False])
def test_idle_rows_in_decode_attention(dev, int4):
    """Rows of length 0: pages untouched, zero outputs (zero int8 row, scale, sum); the other rows bit-identical to the same call with those
    rows active; a following all-active call is unaffected (the split and per-token counters are intact)."""
    from qserve_b200 import backend as ext

    run = _runner(dev, precision="w4a8kv4" if int4 else "w8a8kv8", batch=6, ctx=1100, max_new_tokens=8)
    g = torch.Generator(device=dev).manual_seed(2)
    Hq, Hkv, D = run.Hq, run.Hkv, 128
    qkv = torch.randn((6, (Hq + 2 * Hkv) * D), device=dev, generator=g).half()
    q, k, v = run._heads(qkv)
    table, pools = run.block_tables[0], [run.kpools[0], run.vpools[0]]
    saved = [p.clone() for p in pools]
    active = torch.tensor([900, 1000, 77, 513, 1, 640], dtype=torch.int32, device=dev)
    idle = active.clone()
    idle[[1, 4]] = 0

    def call(lens, quant):
        for p, s in zip(pools, saved):
            p.copy_(s)
        if quant:
            oq = torch.full((6, Hq * D), 5, dtype=torch.int8, device=dev)
            sc, sm = torch.full((6,), 3.0, dtype=torch.half, device=dev), torch.full((6,), 3.0, dtype=torch.half, device=dev)
            ext.single_query_attention_quant(q, k, v, table, lens, 8192, 64, run.size_per_token, 1109, D, 10000.0, int4, True, oq, sc, sm)
            res = (oq, sc, sm)
        else:
            res = (ext.single_query_attention(q, k, v, table, lens, None, 8192, 64, run.size_per_token, 1109, D, 10000.0, True, int4, True),)
        torch.cuda.synchronize()
        return res, [p.clone() for p in pools]

    for quant in (False, True):
        ref, ref_pages = call(active, quant)
        got, got_pages = call(idle, quant)
        keep = torch.tensor([0, 2, 3, 5], device=dev)
        for a, b in zip(ref, got):
            assert torch.equal(a[keep], b[keep])
            assert (b[torch.tensor([1, 4], device=dev)] == 0).all()
        for p, s, r in zip(got_pages, saved, ref_pages):
            for row, n in ((1, None), (4, None), (0, 900), (2, 77), (3, 513), (5, 640)):
                pages = slice(row * run.blocks_per_seq, (row + 1) * run.blocks_per_seq)
                assert torch.equal(p[pages], (s if n is None else r)[pages]), (row, quant)
        again, _ = call(active, quant)
        for a, b in zip(ref, again):
            assert torch.equal(a, b)


def test_padding_slots_write_nothing_and_attend_to_nothing(dev):
    """A chunk segment of C = 40 slots with 12 used: the append writes the bytes of the unpadded call and nothing else, and the prompt
    attention gives the unpadded rows and zero padding rows."""
    from qserve_b200 import backend as ext

    run = _runner(dev, ctx=100, max_new_tokens=8)
    Bn, C = run.batch, 40
    g = torch.Generator(device=dev).manual_seed(4)
    clens = torch.tensor([5, 0, 7, 0], dtype=torch.int32, device=dev)
    cu = torch.tensor([0, 5, 5, 12, 12], dtype=torch.int32, device=dev)
    prefix = torch.tensor([30, 0, 64, 0], dtype=torch.int32, device=dev)
    pad = torch.tensor([0] * 5 + [2 * C - 5] * 7 + [C - 1 - t for t in range(12, C)], dtype=torch.int32, device=dev)
    base = torch.randn((C, (run.Hq + 2 * run.Hkv) * 128), device=dev, generator=g).half()
    table, pools = run.block_tables[0], [run.kpools[0], run.vpools[0]]
    saved = [p.clone() for p in pools]
    res = []
    for T_, pd in ((12, ext.compute_padding_offsets(cu, C, 12)), (C, pad)):
        for p, s in zip(pools, saved):
            p.copy_(s)
        qkv = base[:T_].clone()
        ext.apply_bias_rope_update_kv_cache_at(qkv, clens, pd, prefix, table, run.Hq, run.Hkv, C, 64, run.size_per_token, 128, 10000.0, 8192, True, True,
                                               True)
        attn = ext.prefix_prefill_attention(*run._heads(qkv), cu, C, prefix, 80, table, 64, run.size_per_token, True)
        torch.cuda.synchronize()
        res.append((attn, [p.clone() for p in pools]))
    (a12, p12), (a40, p40) = res
    assert torch.equal(a12, a40[:12]) and (a40[12:] == 0).all()
    assert all(torch.equal(x, y) for x, y in zip(p12, p40))


@pytest.mark.parametrize("penalties,logprobs", [(False, 0), (True, 2)])
def test_greedy_matches_separate_runner(dev, penalties, logprobs):
    """Prompts that fit one piece (C = B ctx): every request's tokens, reasons and chosen-token log-probabilities equal a separate runner's
    prefill(chunk=C) + generate_forward(1); Q > B, so rows are reused by later requests."""
    C = B * CTX
    reqs = _script(14, CTX, T, 1024, seed=5, stops=False)
    for r in reqs:
        r["eos"], r["max_tokens"] = -1, T
    # end requests by eos, by a stop id and by their budget: the ids come from each prompt's greedy continuation
    for i, (toks, _, _) in enumerate(_reference(dev, reqs, C, penalties=penalties)):
        if i % 3 == 0:
            reqs[i]["eos"] = toks[2]
        elif i % 3 == 1:
            reqs[i]["stop"] = [toks[1], 7]
        else:
            reqs[i]["max_tokens"] = 1 + i % T
    run = _runner(dev, prompt_tokens=C, inflight=6)
    kw = dict(repetition=1.3, presence=0.5, frequency=0.25) if penalties else {}
    got = _serve(run, reqs, dev, lambda r: r.inflight_forward(True, penalties=penalties, logprobs=logprobs), logprobs=bool(logprobs), **kw)
    want = _reference(dev, reqs, C, penalties=penalties, logprobs=logprobs)
    reasons = set()
    for i, (toks, reason, lp) in enumerate(want):
        e = got[i]
        assert e[1] == toks and e[2] == reason, (i, e[:3], toks, reason)
        reasons.add(reason)
        if logprobs:
            assert e[3] == lp, i
    assert reasons == {"eos", "stop", "budget"}


def test_split_prompts_keep_layer0_pages(dev):
    """A chunk budget that splits prompts: layer-0 page bytes of every request equal its whole-prompt prefill's, and the first token's logits
    agree to a cosine of 0.99."""
    from tests.test_gpu_prefill_runner import _slots

    C = 16
    run = _runner(dev, prompt_tokens=C, inflight=B)
    reqs = _script(B, CTX, T, 1024, seed=9, stops=False)
    for r, n in zip(reqs, (40, 17, 33, 5)):
        r["prompt"] = (r["prompt"] * 40)[:n]
    _submit(run, reqs, dev)
    first = {}
    for _ in range(20):
        run.inflight_forward(True)
        rows = run.i_plan.logit_rows.tolist()
        for b in range(B):
            if rows[b] >= B:
                first[b] = run.last_logits[b].float().clone()
        if len(first) == B:
            break
    assert len(first) == B
    ref = _runner(dev, prompt_tokens=B * CTX)
    width = CTX
    p = torch.tensor([r["prompt"] + [0] * (width - len(r["prompt"])) for r in reqs], dtype=torch.int64, device=dev)
    lens = torch.tensor([len(r["prompt"]) for r in reqs], dtype=torch.int32, device=dev)
    ref.prefill(p, lens)
    for b in range(B):  # all submitted at once into an empty runner: request b in row b
        r = b
        n = len(reqs[r]["prompt"])
        assert torch.equal(_slots(run, b, n, layers=[0]), _slots(ref, r, n, layers=[0])), b
        cos = torch.nn.functional.cosine_similarity(first[b], ref.last_logits[r].float(), dim=0).item()
        assert cos >= 0.99, (b, cos)


def test_captured_equals_eager(dev):
    """Captured mixed and decode-only steps, interleaved, equal the eager sequence; no host synchronisation between submit and poll."""
    C = 24
    reqs = _script(9, CTX, T, 1024, seed=13)
    res = []
    for captured in (False, True):
        run = _runner(dev, prompt_tokens=C, inflight=5)
        if captured:
            run.capture_inflight(True)
            run.capture_inflight(False)
        k = [0]

        def step(r):
            mixed = k[0] % 3 != 2
            k[0] += 1
            (r.inflight_step if captured else r.inflight_forward)(mixed)

        res.append(_serve(run, reqs, dev, step, nosync=True))
    assert res[0] == res[1]


@pytest.mark.parametrize("C", [24, B * CTX])
def test_runner_steps_follow_the_oracle(dev, C):
    """Through the runner's captured steps (mixed and decode-only interleaved): after every replay the device row state and plan equal the
    oracle's, the oracle's commit of the tokens the step chose gives the device's lengths, histories and finished flags, and every poll
    returns the oracle's retired outputs.  C = 24 splits prompts; with C = B ctx every prompt is carried whole, so the eos / stop ids taken
    from the separate runner's greedy continuations are reached and requests end by eos, stop id and budget."""
    from tests.inflight_oracle import REASONS

    Q = 5
    reqs = _script(11, CTX, T, 1024, seed=19, stops=False)
    for r in reqs:
        r["eos"], r["max_tokens"] = -1, T
    for i, (toks, _, _) in enumerate(_reference(dev, reqs, B * CTX)):  # eos / stop ids from each prompt's greedy continuation
        if i % 3 == 0:
            reqs[i]["eos"] = toks[2]
        elif i % 3 == 1:
            reqs[i]["stop"] = [toks[1], 7]
        else:
            reqs[i]["max_tokens"] = 1 + i % T
    run = _runner(dev, prompt_tokens=C, inflight=Q)
    run.capture_inflight(True)
    run.capture_inflight(False)
    o = InflightOracle(B, Q, C, T)
    done, nxt, reasons = {}, 0, set()
    for step in range(400):
        while nxt < len(reqs) and (nxt - Q < 0 or (nxt - Q) in done):
            r = reqs[nxt]
            _submit(run, [r], dev)
            o.submit(Request(r["prompt"], r["max_tokens"], r["eos"], tuple(r["stop"])))
            nxt += 1
        mixed = step % 4 != 3
        run.inflight_step(mixed)
        want = o.schedule(C if mixed else 0)
        plan, rows = run.i_plan, run.i_rows
        assert rows.phase.tolist() == o.phase and rows.request.tolist() == o.row_req, step
        assert plan.cu_seqlens.tolist() == want.cu_seqlens and plan.chunk_lens.tolist() == want.chunk_lens, step
        assert plan.prefix_lens.tolist() == want.prefix_lens and plan.context_lens.tolist() == want.context_lens, step
        assert plan.logit_rows.tolist() == want.logit_rows and plan.padding_offset.tolist() == want.padding_offset, step
        assert plan.tokens.tolist()[:B + (C if mixed else 0)] == want.tokens[:B + (C if mixed else 0)], step
        o.commit(run.tokens_out.tolist())
        assert run.g_finished.tolist() == o.finished and run.tokens_in.tolist() == o.tokens_in, step
        for b in range(B):
            if o.row_req[b] >= 0:
                L = o.seq_lens[b]
                assert int(run.s_seq_lens[b]) == L and run.s_history[b, :L].tolist() == o.history[b][:L], (step, b)
        for e in run.poll().finished:
            toks, reason = o.outputs[e[0]]
            assert e[1] == toks and e[2] == REASONS[reason], (step, e)
            done[e[0]] = e
            reasons.add(e[2])
        if len(done) == len(reqs):
            break
    assert sorted(done) == list(range(len(reqs))) and sorted(o.ring) == list(range(len(reqs)))
    if C == B * CTX:
        assert reasons == {"eos", "stop", "budget"}


def test_inflight_zero_changes_nothing(dev):
    """inflight > 0 draws the same weights and pages, and the prompt and generation steps give the same results."""
    C = 48
    runs = [_runner(dev, prompt_tokens=C, inflight=q) for q in (0, 4)]
    assert all(torch.equal(a, b) for a, b in zip(runs[0].kpools + runs[0].vpools, runs[1].kpools + runs[1].vpools))
    assert torch.equal(runs[0].embed, runs[1].embed) and torch.equal(runs[0].lm_head, runs[1].lm_head)
    assert all(torch.equal(a["qkv"].qweight, b["qkv"].qweight) for a, b in zip(runs[0].layers, runs[1].layers))
    g = torch.Generator(device=dev).manual_seed(21)
    p = torch.randint(0, 1024, (B, CTX), device=dev, generator=g)
    lens = torch.tensor([40, 3, 17, 29], dtype=torch.int32, device=dev)
    out = []
    for run in runs:
        t0 = run.prefill(p, lens, chunk=8)
        run.capture_generate(1)
        for _ in range(4):
            run.generate_step(1)
        out.append((t0, run.s_history.clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_llama3_8b_full_model_short_script(dev):
    """All 32 layers of Llama-3-8B W4A8KV4: a short greedy script equals the separate runner."""
    with torch.no_grad():
        kw = dict(batch=4, ctx=96, max_new_tokens=6)
        C = 4 * 96
        run = _runner(dev, model="llama-3-8b", prompt_tokens=C, inflight=5, **kw)
        reqs = _script(6, 96, 6, 128256, seed=17)
        got = _serve(run, reqs, dev, lambda r: r.inflight_forward(True))
        del run
        torch.cuda.empty_cache()
        want = _reference(dev, reqs, C, model="llama-3-8b", **kw)
        for i, (toks, reason, _) in enumerate(want):
            assert got[i][1] == toks and got[i][2] == reason, i
