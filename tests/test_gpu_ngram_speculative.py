"""GPU: prompt-lookup drafting (qs_ngram_propose) and the commit (qs_spec_commit) bitwise against the oracle (tests/ngram_oracle.py), and the
decode runner's generation loop: speculative steps emit the tokens of plain decoding.

Where the speculative loop and the plain loop differ, the cause must be the fp32 summation order in which multi-token and decode attention
differ (DESIGN.md section 3.6): at the first differing position of a row, the plain step's two largest logits must lie within
1e-2 * max |logit| of each other, and the row is not compared past it.
"""
import numpy as np
import pytest
import torch

from tests import ngram_oracle as ng

pytestmark = pytest.mark.gpu


def _backend():
    from qserve_b200 import backend
    return backend


def _history(rng, B, H, alphabet=40):
    """Random ids from a small alphabet with the row's last tokens planted at a few earlier places (long matches), some -1, ragged L."""
    h = rng.integers(0, alphabet, (B, H)).astype(np.int64)
    L = rng.integers(0, H + 1, B).astype(np.int32)
    L[: min(B, 4)] = [0, 1, 2, H][: min(B, 4)]
    for b in range(B):
        if L[b] > 20:
            key = h[b, L[b] - 8: L[b]].copy()
            for _ in range(3):
                g = int(rng.integers(1, 9))
                at = int(rng.integers(g, L[b] - 8))
                h[b, at - g: at] = key[8 - g:]
        h[b, rng.random(H) < 0.01] = -1
    return h, L


@pytest.mark.parametrize("B,H", [(1, 4096), (7, 32768), (64, 1024)])
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_ngram_propose_matches_oracle(dev, B, H, n):
    be = _backend()
    rng = np.random.default_rng(B * 1000 + H + n)
    h, L = _history(rng, B, H)
    ht, Lt = torch.from_numpy(h).to(dev), torch.from_numpy(L).to(dev)
    for n_min, n_max, branches in ((1, 4, 1), (2, 8, 4), (1, 1, 8), (3, 5, 2)):
        tok, mask = be.ngram_propose(ht, Lt, n, n_min, n_max, branches)
        want_t, want_m = ng.ngram_propose(h, L, n, n_min, n_max, branches)
        assert np.array_equal(tok.cpu().numpy(), want_t), (n_min, n_max, branches)
        assert np.array_equal(mask.cpu().numpy(), want_m), (n_min, n_max, branches)


def _commit_case(rng, B, n, H):
    draft = rng.integers(0, 50, (B, n)).astype(np.int64)
    acc = rng.integers(1, n + 1, B).astype(np.int32)
    path = np.full((B, n), -1, np.int32)
    for b in range(B):
        path[b, 0] = 0
        path[b, 1: acc[b]] = np.sort(rng.choice(np.arange(1, n), acc[b] - 1, replace=False)) if acc[b] > 1 else []
    bonus = rng.integers(0, 50, B).astype(np.int64)
    prompt = rng.integers(1, H // 2, B).astype(np.int32)
    L = (prompt + rng.integers(0, H // 2, B)).astype(np.int32)
    L[: min(B, 2)] = H - 1  # appends past the last column
    budget = rng.integers(0, 40, B).astype(np.int32)
    eos = np.where(rng.random(B) < 0.5, rng.integers(0, 50, B), -1).astype(np.int64)
    fin = (rng.random(B) < 0.2).astype(np.int32)
    hist = rng.integers(0, 50, (B, H)).astype(np.int64)
    return draft, path, acc, bonus, hist, L, prompt, budget, eos, fin


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_spec_commit_matches_oracle(dev, B, n):
    be = _backend()
    rng = np.random.default_rng(B * 17 + n)
    H = 300
    draft, path, acc, bonus, hist, L, prompt, budget, eos, fin = _commit_case(rng, B, n, H)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    g_hist, g_L, g_fin = t(hist), t(L), t(fin)
    sp = torch.full((B,), -7, dtype=torch.int32, device=dev)
    cl = torch.full((B,), -7, dtype=torch.int32, device=dev)
    roots = torch.full((B,), -7, dtype=torch.int64, device=dev)
    be.spec_commit(t(draft), t(path), t(acc), t(bonus), g_hist, g_L, t(prompt), t(budget), t(eos), g_fin, sp, cl, roots)
    w_hist, w_L, w_fin, w_sp, w_cl, w_root = ng.spec_commit(draft, path, acc, bonus, hist, L, prompt, budget, eos, fin)
    assert np.array_equal(g_hist.cpu().numpy(), w_hist) and np.array_equal(g_L.cpu().numpy(), w_L) and np.array_equal(g_fin.cpu().numpy(), w_fin)
    for b in range(B):
        want = (-7, -7, -7) if w_sp[b] is None else (w_sp[b], w_cl[b], w_root[b])
        assert (int(sp[b]), int(cl[b]), int(roots[b])) == want, b
    # optional outputs left out
    g2 = t(hist)
    be.spec_commit(t(draft), t(path), t(acc), t(bonus), g2, t(L), t(prompt), t(budget), t(eos), t(fin), sp.clone())
    assert np.array_equal(g2.cpu().numpy(), w_hist)


def test_ops_deterministic_and_graph_replay(dev):
    be = _backend()
    rng = np.random.default_rng(5)
    B, H, n = 64, 8192, 8
    h, L = _history(rng, B, H)
    ht, Lt = torch.from_numpy(h).to(dev), torch.from_numpy(L).to(dev)
    tok = torch.empty((B, n), dtype=torch.int64, device=dev)
    mask = torch.empty((B, n), dtype=torch.int32, device=dev)
    a = [x.clone() for x in be.ngram_propose(ht, Lt, n, 1, 4, 4)]
    b = [x.clone() for x in be.ngram_propose(ht, Lt, n, 1, 4, 4)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.ngram_propose(ht, Lt, n, 1, 4, 4, tokens=tok, tree_mask=mask)
    for _ in range(3):
        tok.fill_(0); mask.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(tok, a[0]) and torch.equal(mask, a[1])
    # the commit inside a graph: each replay appends again
    draft, path, acc, bonus, hist, Lc, prompt, budget, eos, fin = _commit_case(rng, B, n, 300)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    args = [t(draft), t(path), t(acc), t(bonus), t(hist), t(Lc), t(prompt), t(budget), t(eos), t(fin), t(Lc - 1)]
    snap = [x.clone() for x in args]
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        be.spec_commit(*args)
    g2.replay()
    eager = [x.clone() for x in snap]
    be.spec_commit(*eager)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(args, eager))


def test_argument_errors(dev):
    be = _backend()
    h = torch.zeros((2, 16), dtype=torch.int64, device=dev)
    L = torch.zeros(2, dtype=torch.int32, device=dev)
    for bad in (dict(num_nodes=0), dict(num_nodes=17), dict(num_nodes=4, n_min=0), dict(num_nodes=4, n_min=3, n_max=2),
                dict(num_nodes=4, n_max=9), dict(num_nodes=4, branches=0), dict(num_nodes=4, branches=9)):
        with pytest.raises(RuntimeError):
            be.ngram_propose(h, L, **bad)
    for hh, LL in ((h.int(), L), (h, L.long()), (h, L[:1]), (h.cpu(), L.cpu()), (torch.zeros((2, 32769), dtype=torch.int64, device=dev), L)):
        with pytest.raises(RuntimeError):
            be.ngram_propose(hh, LL, 4)
    with pytest.raises(RuntimeError):
        be.ngram_propose(h, L, 4, tokens=torch.empty((2, 3), dtype=torch.int64, device=dev))
    d = torch.zeros((2, 4), dtype=torch.int64, device=dev)
    p = torch.zeros((2, 4), dtype=torch.int32, device=dev)
    i32 = lambda: torch.zeros(2, dtype=torch.int32, device=dev)
    i64 = lambda: torch.zeros(2, dtype=torch.int64, device=dev)
    ok = [d, p, i32(), i64(), h, i32(), i32(), i32(), i64(), i32(), i32()]
    be.spec_commit(*ok)
    for k, bad in ((0, d.int()), (1, p[:, :3].contiguous()), (2, i64()), (3, i32()), (4, h[:1]), (8, i32()), (10, i64())):
        args = list(ok)
        args[k] = bad
        with pytest.raises(RuntimeError):
            be.spec_commit(*args)
    with pytest.raises(RuntimeError):
        be.spec_commit(torch.zeros((2, 17), dtype=torch.int64, device=dev), torch.zeros((2, 17), dtype=torch.int32, device=dev), *ok[2:])


# ---------------------------------------------------------------------------------------------------------------------------------
# the decode runner's generation loop
# ---------------------------------------------------------------------------------------------------------------------------------
T = 32
CTX = 100
BATCH = 6


def _runner(dev, precision, **kw):
    from qserve_b200.decode import DecodeRunner

    return DecodeRunner("tiny", precision, batch=BATCH, ctx=CTX, device=dev, seed=11, verify_len=8, max_new_tokens=T, generate=True, **kw)


def _plain(run, prompt):
    """The plain loop: T decode steps.  Returns (tokens [B, T], top-2 gap [B, T], max |logit| [B, T])."""
    run.reset_generation(prompt)
    gaps, scale = [], []
    with torch.no_grad():
        for _ in range(T):
            run.generate_forward(1)
            lg = run.last_logits.float()
            top = lg.topk(2, dim=-1).values
            gaps.append(top[:, 0] - top[:, 1])
            scale.append(lg.abs().amax(dim=-1))
    torch.cuda.synchronize()
    out = run.s_history[:, CTX + 1:].clone()
    assert torch.equal(run.s_seq_lens, torch.full((BATCH,), CTX + 1 + T, dtype=torch.int32, device=run.dev))
    assert bool(run.g_finished.all())
    return out, torch.stack(gaps, 1), torch.stack(scale, 1)


def _speculative(run, prompt, n, branches, ngram=(1, 4), sampled=False):
    run.reset_generation(prompt)
    steps = 0
    with torch.no_grad():
        while not bool(run.g_finished.all()):
            run.generate_forward(n, branches, ngram, sampled)
            steps += 1
            assert steps <= T
    torch.cuda.synchronize()
    return run.s_history[:, CTX + 1:].clone(), steps


def _same_or_near_tie(got, plain, gaps, scale):
    """Row by row: equal, or the first difference is at a near-tie of the plain step.  Returns the rows that are equal."""
    equal = []
    for b in range(got.size(0)):
        diff = (got[b] != plain[b]).nonzero()
        if diff.numel() == 0:
            equal.append(b)
            continue
        k = int(diff[0])
        assert float(gaps[b, k]) < 1e-2 * float(scale[b, k]), f"row {b} differs at {k}: gap {float(gaps[b, k])}, max |logit| {float(scale[b, k])}"
    return equal


def _oracle_steps(prompt_row, plain_row, n, branches, ngram):
    """Steps of the oracle speculative loop whose target is the plain output."""
    full = list(prompt_row) + list(plain_row)
    # past the budget the target is never used: the commit cuts those tokens
    steps = ng.speculative_generate(prompt_row, lambda seq: full[len(seq)] if len(seq) < len(full) else 0, T, n, branches, ngram[0], ngram[1])
    assert steps[0] == list(plain_row)
    return steps[1]


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
def test_generate_emits_the_plain_tokens(dev, precision):
    run = _runner(dev, precision)
    g = torch.Generator(device=dev).manual_seed(3)
    prompt = torch.randint(0, run.cfg.vocab, (BATCH, CTX + 1), device=dev, generator=g)
    plain, gaps, scale = _plain(run, prompt)
    # wrong planting: a random prompt; the drafts are mostly rejected and the tokens stay the same
    for n, branches in ((4, 1), (8, 2)):
        got, _ = _speculative(run, prompt, n, branches)
        _same_or_near_tie(got, plain, gaps, scale)
    # correct planting: the key (the last 4 ids) and the plain output earlier in the prompt.  The ids of the history do not enter the model
    # (the pages are synthetic), so the plain output is the same; every step should accept up to n - 1 drafts.
    planted = prompt.clone()
    planted[:, 10:14] = prompt[:, CTX - 3:CTX + 1]
    planted[:, 14:14 + T] = plain
    for n, branches in ((4, 1), (8, 2)):
        got, steps = _speculative(run, planted, n, branches)
        equal = _same_or_near_tie(got, plain, gaps, scale)
        if len(equal) == BATCH:
            pr, pl = planted.cpu().numpy(), plain.cpu().numpy()
            want = max(_oracle_steps(pr[b], pl[b], n, branches, (1, 4)) for b in range(BATCH))
            assert steps == want
            key_and_out = [list(pr[b, CTX - 3:]) + list(pl[b]) for b in range(BATCH)]
            repeats = any(len({tuple(s[i:i + 4]) for i in range(len(s) - 3)}) < len(s) - 3 for s in key_and_out)
            if not repeats:  # a repeated 4-gram in the output would be the more recent match; without one, every draft comes from the plant
                assert steps <= -(-T // (n - 1)) + 2


def _expected(plain, budget, eos):
    rows = []
    for b in range(plain.size(0)):
        r = plain[b, : int(budget[b])].tolist()
        if int(eos[b]) >= 0 and int(eos[b]) in r:
            r = r[: r.index(int(eos[b])) + 1]
        rows.append(r)
    return rows


def test_generate_eos_and_budgets_stop_rows(dev):
    run = _runner(dev, "w4a8kv4")
    g = torch.Generator(device=dev).manual_seed(4)
    prompt = torch.randint(0, run.cfg.vocab, (BATCH, CTX + 1), device=dev, generator=g)
    plain, gaps, scale = _plain(run, prompt)
    budget = torch.tensor([T, 5, 1, 0, T, 17], dtype=torch.int32, device=dev)
    eos = torch.tensor([-1, -1, -1, -1, int(plain[4, 6]), int(plain[5, 9])], dtype=torch.int64, device=dev)
    want = _expected(plain, budget, eos)
    for n, branches in ((1, 1), (4, 1), (8, 2)):
        run.g_budget.copy_(budget); run.g_eos.copy_(eos)
        got, _ = _speculative(run, prompt, n, branches)
        lens = (run.s_seq_lens - (CTX + 1)).tolist()
        for b in range(BATCH):
            row = got[b, : lens[b]].tolist()
            if row != want[b]:  # only at a near-tie of the plain loop
                k = next(i for i in range(min(len(row), len(want[b]))) if row[i] != want[b][i])
                assert float(gaps[b, k]) < 1e-2 * float(scale[b, k])
                continue
            assert bool((got[b, lens[b]:] == -1).all())
        # finished rows are left alone by later steps
        hist, lens_t, tok = run.s_history.clone(), run.s_seq_lens.clone(), run.tokens_in.clone()
        with torch.no_grad():
            run.generate_forward(n, branches)
        torch.cuda.synchronize()
        assert torch.equal(run.s_history, hist) and torch.equal(run.s_seq_lens, lens_t) and torch.equal(run.tokens_in, tok)
    run.g_budget.fill_(T); run.g_eos.fill_(-1)


def _pages(run):
    return [p.clone() for p in run.kpools + run.vpools + run.kpools_gen + run.vpools_gen]


@pytest.mark.parametrize("n,branches", [(1, 1), (4, 1), (8, 2)])
def test_generate_graph_replays_the_eager_step(dev, n, branches):
    run = _runner(dev, "w4a8kv8")
    g = torch.Generator(device=dev).manual_seed(5)
    prompt = torch.randint(0, 64, (BATCH, CTX + 1), device=dev, generator=g)  # a small alphabet: many drafts
    run.reset_generation(prompt)
    run.capture_generate(n, branches)
    K = 6
    run.reset_generation(prompt)
    with torch.no_grad():
        for _ in range(K):
            run.generate_forward(n, branches)
    torch.cuda.synchronize()
    eager = (run.s_history.clone(), run.s_seq_lens.clone(), run.tokens_in.clone(), run.context_lens.clone(), run.g_start.clone(), _pages(run))
    run.reset_generation(prompt)
    for _ in range(K):
        run.generate_step(n, branches)
    torch.cuda.synchronize()
    assert torch.equal(run.s_history, eager[0]) and torch.equal(run.s_seq_lens, eager[1]) and torch.equal(run.tokens_in, eager[2])
    assert torch.equal(run.context_lens, eager[3]) and torch.equal(run.g_start, eager[4])
    assert all(torch.equal(a, b) for a, b in zip(_pages(run), eager[5]))


def test_generate_sampled_at_zero_temperature_is_greedy(dev):
    run = _runner(dev, "w4a8kv4")
    g = torch.Generator(device=dev).manual_seed(6)
    prompt = torch.randint(0, 64, (BATCH, CTX + 1), device=dev, generator=g)
    for n, branches in ((1, 1), (4, 1), (8, 2)):
        greedy, _ = _speculative(run, prompt, n, branches)
        run.s_temperature.fill_(0.0); run.s_top_k.fill_(-1); run.s_top_p.fill_(1.0)
        sampled, _ = _speculative(run, prompt, n, branches, sampled=True)
        assert torch.equal(greedy, sampled)


def test_generate_runner_keeps_weights_and_pages(dev):
    from qserve_b200.decode import DecodeRunner

    plain = DecodeRunner("tiny", "w4a8kv4", batch=BATCH, ctx=CTX, device=dev, seed=11, verify_len=8, max_new_tokens=T)
    gen = _runner(dev, "w4a8kv4")
    assert torch.equal(plain.embed, gen.embed) and torch.equal(plain.lm_head, gen.lm_head)
    for a, b in zip(plain.layers, gen.layers):
        assert torch.equal(a["qkv"].qweight, b["qkv"].qweight) and torch.equal(a["down"].s1, b["down"].s1)
    assert gen.blocks_per_seq == plain.blocks_per_seq and gen.table_blocks * 64 >= CTX + T + 8
    assert all(torch.equal(x, y) for x, y in zip(plain.kpools + plain.vpools, gen.kpools + gen.vpools))
    # every row's first blocks_per_seq table entries point at that row's pages of the same pools
    for li in range(gen.L):
        for kv, pools in ((0, gen.kpools), (1, gen.vpools)):
            base = pools[li].data_ptr()
            pb = plain.kpools[li].data_ptr() if kv == 0 else plain.vpools[li].data_ptr()
            assert torch.equal(gen.block_tables[li, :, kv, : gen.blocks_per_seq] - base, plain.block_tables[li, :, kv] - pb)


def test_llama3_8b_generate_step_drafts_equal_the_oracle(dev):
    from qserve_b200.decode import DecodeRunner

    B, C = 64, 1024
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=C, device=dev, seed=0, verify_len=8, max_new_tokens=8, generate=True)
    g = torch.Generator(device=dev).manual_seed(7)
    prompt = torch.randint(0, 200, (B, C + 1), device=dev, generator=g)
    run.reset_generation(prompt)
    hist, lens = run.s_history.cpu().numpy(), run.s_seq_lens.cpu().numpy()
    with torch.no_grad():
        run.generate_forward(8, 2)
    torch.cuda.synchronize()
    want_t, want_m = ng.ngram_propose(hist, lens, 8, 1, 4, 2)
    assert np.array_equal(run.g_tokens[: B * 8].view(B, 8).cpu().numpy(), want_t)
    assert np.array_equal(run.g_mask[: B * 8].view(B, 8).cpu().numpy(), want_m)
    acc = run.v_accept_len.cpu().numpy()
    assert np.array_equal(run.s_seq_lens.cpu().numpy(), lens + acc)
    assert bool((run.s_history[:, C + 1:][torch.arange(8, device=dev)[None, :] < torch.from_numpy(acc).to(dev)[:, None]] >= 0).all())
