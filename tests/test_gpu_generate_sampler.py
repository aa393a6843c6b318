"""GPU: penalties, log-probabilities and stop tokens in the generation loop.

The ops are checked bitwise: apply_penalties_tree against apply_penalties over the expanded per-node histories (and the CPU oracle,
tests/generate_sampler_oracle.py), logprobs_accepted against logprobs_rows on the gathered node rows, the stop-set commit against the oracle.
The runner is checked as the sequential loop it must reproduce: each penalised plain step against the ops on that step's logits, and the
speculative loop under penalties against the plain loop, with the near-tie rule of test_gpu_ngram_speculative.py (the verify and decode
attention sum in different fp32 orders, DESIGN.md section 3.6).
"""
import numpy as np
import pytest
import torch

from tests import generate_sampler_oracle as gso
from tests import ngram_oracle as ng

pytestmark = pytest.mark.gpu

V = 4096


def _backend():
    from qserve_b200 import backend
    return backend


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _hand_tree(rng, B, n):
    """Random trees (parent of node i drawn below i), tokens from a small alphabet, some padding nodes (token -1, mask 1)."""
    tok = rng.integers(0, 40, (B, n)).astype(np.int64)
    mask = np.zeros((B, n), np.int32)
    for b in range(B):
        for i in range(1, n):
            if rng.random() < 0.15:
                tok[b, i], mask[b, i] = -1, 1
                continue
            p = int(rng.integers(0, i))
            mask[b, i] = mask[b, p] | (1 << p)
    return tok, mask


def _penalty_case(rng, B, n, H):
    h = rng.integers(0, 40, (B, H)).astype(np.int64)
    h[rng.random((B, H)) < 0.01] = -1
    L = rng.integers(1, H + 1, B).astype(np.int32)
    L[: min(B, 3)] = [H, H + 5, 1][: min(B, 3)]  # L + depth past H, L past H (clamped), a root-only history
    pl = (L * rng.random(B)).astype(np.int32)
    pl[-1] = L[-1]  # a prompt-only row
    rep = rng.choice([1.0, 0.8, 1.3], B).astype(np.float32)
    pres = rng.choice([0.0, 0.4, -0.7], B).astype(np.float32)
    freq = rng.choice([0.0, 0.25, -0.5], B).astype(np.float32)
    rep[0], pres[0], freq[0] = 1.0, 0.0, 0.0  # a neutral row
    x = rng.standard_normal((B, n, V)).astype(np.float16) * np.float16(4)
    x[rng.random((B, n, V)) < 0.002] = np.nan
    return h, L, pl, rep, pres, freq, x


def _composition(be, dev, x, tok, mask, h, L, pl, rep, pres, freq):
    """The torch composition the kernel replaces: expanded per-node histories, then apply_penalties over B n rows."""
    B, n = tok.shape
    eh, epl, esl = gso.expand_histories(tok, mask, h, pl, L)
    r = lambda a: _t(np.repeat(a, n), dev)
    out = _t(x, dev).view(B * n, V).clone()
    be.apply_penalties(out, _t(eh, dev), _t(epl, dev), _t(esl, dev), r(rep), r(pres), r(freq))
    return out.view(B, n, V)


@pytest.mark.parametrize("B,H", [(1, 4096), (7, 32752), (7, 32768), (64, 1024)])
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_apply_penalties_tree_matches_composition_and_oracle(dev, B, H, n):
    be = _backend()
    rng = np.random.default_rng(B * 100 + n + H)
    h, L, pl, rep, pres, freq, x = _penalty_case(rng, B, n, H)
    for kind in ("ngram", "hand"):
        if kind == "ngram":
            tok, mask = (a.cpu().numpy() for a in be.ngram_propose(_t(h, dev), _t(L, dev), n, 1, 4, 4))
        else:
            tok, mask = _hand_tree(rng, B, n)
        got = _t(x, dev)
        be.apply_penalties_tree(got, _t(tok, dev), _t(mask, dev), _t(h, dev), _t(pl, dev), _t(L, dev), _t(rep, dev), _t(pres, dev), _t(freq, dev))
        if H + 16 <= be.MAX_PENALTY_HISTORY:  # the composition's expanded rows must fit apply_penalties' history limit
            comp = _composition(be, dev, x, tok, mask, h, L, pl, rep, pres, freq)
            assert torch.equal(got.view(torch.int16), comp.view(torch.int16)), kind  # bitwise, NaN included
        want = gso.apply_penalties_tree(x, tok, mask, h, pl, L, rep, pres, freq)
        assert np.array_equal(got.cpu().numpy().view(np.int16), want.view(np.int16)), kind
        assert np.array_equal(got[0].cpu().numpy().view(np.int16), x[0].view(np.int16))  # the neutral row is untouched


def test_apply_penalties_tree_deterministic_and_graph_replay(dev):
    be = _backend()
    rng = np.random.default_rng(7)
    B, n, H = 64, 8, 8192
    h, L, pl, rep, pres, freq, x = _penalty_case(rng, B, n, H)
    tok, mask = _hand_tree(rng, B, n)
    args = [_t(a, dev) for a in (tok, mask, h, pl, L, rep, pres, freq)]
    a, b = _t(x, dev), _t(x, dev)
    be.apply_penalties_tree(a, *args)
    be.apply_penalties_tree(b, *args)
    out = _t(x, dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.apply_penalties_tree(out, *args)
    for _ in range(2):
        out.copy_(_t(x, dev))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(out.view(torch.int16), a.view(torch.int16))


def _accepted_case(rng, B, n, W):
    tok = rng.integers(0, V, (B, n)).astype(np.int64)
    acc = rng.integers(1, n + 1, B).astype(np.int32)
    path = np.full((B, n), -1, np.int32)
    for b in range(B):
        path[b, 0] = 0
        path[b, 1: acc[b]] = np.sort(rng.choice(np.arange(1, n), acc[b] - 1, replace=False)) if acc[b] > 1 else []
    bonus = rng.integers(0, V, B).astype(np.int64)
    L = rng.integers(0, W, B).astype(np.int32)
    L[: min(B, 2)] = [W - 1, W - 2][: min(B, 2)]  # tokens past the last column are dropped
    fin = (rng.random(B) < 0.2).astype(np.int32)
    x = (rng.standard_normal((B, n, V)) * 3).astype(np.float16)
    return tok, path, acc, bonus, L, fin, x


@pytest.mark.parametrize("B,n", [(1, 1), (7, 4), (64, 8), (5, 16)])
def test_logprobs_accepted_matches_logprobs_rows(dev, B, n):
    be = _backend()
    rng = np.random.default_rng(B * 31 + n)
    W, K = 40, 5
    tok, path, acc, bonus, L, fin, x = _accepted_case(rng, B, n, W)
    lp = torch.full((B, W), 123.0, dtype=torch.float32, device=dev)  # poisoned sentinels: whatever is not written keeps them
    ids = torch.full((B, W, K), 777, dtype=torch.int64, device=dev)
    tlp = torch.full((B, W, K), 123.0, dtype=torch.float32, device=dev)
    logits = _t(x, dev)
    be.logprobs_accepted(logits, _t(tok, dev), _t(path, dev), _t(acc, dev), _t(bonus, dev), _t(L, dev), _t(fin, dev), K, lp, ids, tlp)
    entries = gso.accepted_entries(tok, path, acc, bonus, L, fin, W)
    written = torch.zeros((B, W), dtype=torch.bool, device=dev)
    if entries:
        bb, col, node, t = (torch.tensor(v, device=dev) for v in zip(*entries))
        w_lp, w_ids, w_tlp = be.logprobs_rows(logits[bb, node].contiguous(), t, K)
        assert torch.equal(lp[bb, col], w_lp) and torch.equal(ids[bb, col], w_ids) and torch.equal(tlp[bb, col], w_tlp)
        written[bb, col] = True
    assert bool((lp[~written] == 123.0).all()) and bool((ids[~written] == 777).all()) and bool((tlp[~written] == 123.0).all())
    # n_top = 0 writes only the log-probabilities
    lp0 = torch.full((B, W), 123.0, dtype=torch.float32, device=dev)
    be.logprobs_accepted(logits, _t(tok, dev), _t(path, dev), _t(acc, dev), _t(bonus, dev), _t(L, dev), _t(fin, dev), 0, lp0)
    assert torch.equal(lp0, lp)


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("n", [1, 4, 16])
def test_spec_commit_stops_matches_oracle(dev, B, n):
    be = _backend()
    rng = np.random.default_rng(B * 13 + n)
    H = 300
    draft = rng.integers(0, 30, (B, n)).astype(np.int64)
    acc = rng.integers(1, n + 1, B).astype(np.int32)
    path = np.zeros((B, n), np.int32)
    for b in range(B):
        path[b, 1: acc[b]] = np.sort(rng.choice(np.arange(1, n), acc[b] - 1, replace=False)) if acc[b] > 1 else []
    bonus = rng.integers(0, 30, B).astype(np.int64)
    prompt = rng.integers(1, H // 2, B).astype(np.int32)
    L = (prompt + rng.integers(0, H // 2, B)).astype(np.int32)
    L[0] = H - 1
    budget = rng.integers(0, 40, B).astype(np.int32)
    eos = np.where(rng.random(B) < 0.3, rng.integers(0, 30, B), -1).astype(np.int64)
    fin = (rng.random(B) < 0.2).astype(np.int32)
    hist = rng.integers(0, 30, (B, H)).astype(np.int64)
    for S in (1, 3, 8):
        stops = np.where(rng.random((B, S)) < 0.6, rng.integers(0, 30, (B, S)), -1).astype(np.int64)
        g = [_t(a, dev) for a in (hist, L, fin)]
        sp, cl, roots = (torch.full((B,), -7, dtype=dt, device=dev) for dt in (torch.int32, torch.int32, torch.int64))
        be.spec_commit(_t(draft, dev), _t(path, dev), _t(acc, dev), _t(bonus, dev), g[0], g[1], _t(prompt, dev), _t(budget, dev), _t(eos, dev), g[2],
                       sp, cl, roots, stop_ids=_t(stops, dev))
        w = gso.spec_commit_stops(draft, path, acc, bonus, hist, L, prompt, budget, eos, stops, fin)
        assert np.array_equal(g[0].cpu().numpy(), w[0]) and np.array_equal(g[1].cpu().numpy(), w[1]) and np.array_equal(g[2].cpu().numpy(), w[2])
        for b in range(B):
            want = (-7, -7, -7) if w[3][b] is None else (w[3][b], w[4][b], w[5][b])
            assert (int(sp[b]), int(cl[b]), int(roots[b])) == want
    # stop ids all -1 (and an empty set) give exactly the existing call
    outs = []
    for stops in (None, np.full((B, 8), -1, np.int64), np.zeros((B, 0), np.int64)):
        g = [_t(a, dev) for a in (hist, L, fin)]
        sp, cl, roots = (torch.full((B,), -7, dtype=dt, device=dev) for dt in (torch.int32, torch.int32, torch.int64))
        be.spec_commit(_t(draft, dev), _t(path, dev), _t(acc, dev), _t(bonus, dev), g[0], g[1], _t(prompt, dev), _t(budget, dev), _t(eos, dev), g[2],
                       sp, cl, roots, stop_ids=None if stops is None else _t(stops, dev))
        outs.append(g + [sp, cl, roots])
    assert all(torch.equal(a, b) for o in outs[1:] for a, b in zip(outs[0], o))
    with pytest.raises(RuntimeError):
        be.spec_commit(_t(draft, dev), _t(path, dev), _t(acc, dev), _t(bonus, dev), _t(hist, dev), _t(L, dev), _t(prompt, dev), _t(budget, dev),
                       _t(eos, dev), _t(fin, dev), _t(L, dev), stop_ids=torch.zeros((B, 9), dtype=torch.int64, device=dev))


# ---------------------------------------------------------------------------------------------------------------------------------
# the decode runner's generation loop
# ---------------------------------------------------------------------------------------------------------------------------------
T, CTX, BATCH = 32, 100, 6
PEN = dict(rep=1.3, pres=0.4, freq=0.3)


def _runner(dev, precision="w4a8kv4", **kw):
    from qserve_b200.decode import DecodeRunner

    return DecodeRunner("tiny", precision, batch=BATCH, ctx=CTX, device=dev, seed=11, verify_len=8, max_new_tokens=T, generate=True, **kw)


def _set_penalties(run, rep=1.0, pres=0.0, freq=0.0):
    run.s_repetition.fill_(rep); run.s_presence.fill_(pres); run.s_frequency.fill_(freq)


def _state(run):
    return [run.s_history, run.s_seq_lens, run.tokens_in, run.context_lens, run.g_start, run.g_finished]


def test_plain_step_is_the_ops_on_its_logits(dev):
    be = _backend()
    run = _runner(dev)
    _set_penalties(run, **PEN)
    g = torch.Generator(device=dev).manual_seed(1)
    prompt = torch.randint(0, 48, (BATCH, CTX + 1), device=dev, generator=g)
    run.reset_generation(prompt)
    K = 5
    with torch.no_grad():
        for step in range(8):
            snap = [t.clone() for t in _state(run)]
            run.generate_forward(1)  # the same step without penalties: its logits are the unpenalised ones
            raw = run.last_logits.clone()
            for t, s in zip(_state(run), snap):
                t.copy_(s)
            run.generate_forward(1, penalties=True, logprobs=K)
            pen = run.last_logits  # penalised in place
            want = be.apply_penalties(raw.clone(), snap[0], run.s_prompt_lens, snap[1], run.s_repetition, run.s_presence, run.s_frequency)
            assert torch.equal(pen, want), step
            tok = be.argmax_rows(want)
            lp, ids, tlp = be.logprobs_rows(want, tok, K)
            col = snap[1].long()
            rows = torch.arange(BATCH, device=dev)
            assert torch.equal(run.s_history[rows, col], tok)
            top_ids, top_lp = run.g_top_view(K)
            assert torch.equal(run.g_logprob[rows, col], lp) and torch.equal(top_ids[rows, col], ids) and torch.equal(top_lp[rows, col], tlp)


def _plain(run, prompt, **kw):
    """T plain steps: (tokens [B, T], top-2 gap [B, T], max |logit| [B, T]) of the logits the step picked from."""
    run.reset_generation(prompt)
    gaps, scale = [], []
    with torch.no_grad():
        for _ in range(T):
            run.generate_forward(1, **kw)
            lg = run.last_logits.float()
            top = lg.topk(2, dim=-1).values
            gaps.append(top[:, 0] - top[:, 1])
            scale.append(lg.abs().amax(dim=-1))
    torch.cuda.synchronize()
    return run.s_history[:, CTX + 1:].clone(), torch.stack(gaps, 1), torch.stack(scale, 1)


def _speculative(run, prompt, n, branches, **kw):
    run.reset_generation(prompt)
    steps = 0
    with torch.no_grad():
        while not bool(run.g_finished.all()):
            run.generate_forward(n, branches, **kw)
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


def _check_logprobs(run, plain_lp, equal, scale):
    """On rows equal to the plain loop, g_logprob agrees with the plain loop's within 1e-2 max |logit|: the logits differ by the fp32
    summation order of the verify and decode attention, the same bound as the near-tie rule."""
    got = run.g_logprob[:, CTX + 1: CTX + 1 + T]
    for b in equal:
        assert bool(torch.isfinite(got[b]).all())
        assert float((got[b] - plain_lp[b]).abs().max()) <= 1e-2 * float(scale[b].max()), b


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
def test_speculative_equals_plain_under_penalties(dev, precision):
    run = _runner(dev, precision)
    g = torch.Generator(device=dev).manual_seed(3)
    # random small-alphabet prompts: many drafts, and the repetition penalty acts on the prompt's ids
    small = torch.randint(0, 64, (BATCH, CTX + 1), device=dev, generator=g)
    unpen, _, _ = _plain(run, small)
    _set_penalties(run, **PEN)
    plain, gaps, scale = _plain(run, small, penalties=True, logprobs=5)
    plain_lp = run.g_logprob[:, CTX + 1: CTX + 1 + T].clone()
    assert not torch.equal(plain, unpen), "the penalties must change the plain output"
    for n, branches in ((4, 1), (8, 2)):
        got, _ = _speculative(run, small, n, branches, penalties=True, logprobs=5)
        _check_logprobs(run, plain_lp, _same_or_near_tie(got, plain, gaps, scale), scale)
    # planted: presence / frequency only (the repetition penalty counts prompt ids, so planting the output would change it)
    _set_penalties(run, pres=0.6, freq=0.4)
    rnd = torch.randint(0, run.cfg.vocab, (BATCH, CTX + 1), device=dev, generator=g)
    unpen, _, _ = _plain(run, rnd)
    plain, gaps, scale = _plain(run, rnd, penalties=True, logprobs=5)
    plain_lp = run.g_logprob[:, CTX + 1: CTX + 1 + T].clone()
    assert not torch.equal(plain, unpen), "the penalties must change the plain output"
    planted = rnd.clone()
    planted[:, 10:14] = rnd[:, CTX - 3:CTX + 1]
    planted[:, 14:14 + T] = plain
    for n, branches in ((4, 1), (8, 2)):
        got, steps = _speculative(run, planted, n, branches, penalties=True, logprobs=5)
        equal = _same_or_near_tie(got, plain, gaps, scale)
        _check_logprobs(run, plain_lp, equal, scale)
        if len(equal) == BATCH:
            pr, pl = planted.cpu().numpy(), plain.cpu().numpy()
            full = [list(pr[b]) + list(pl[b]) for b in range(BATCH)]
            want = max(ng.speculative_generate(pr[b], lambda s, f=full[b]: f[len(s)] if len(s) < len(f) else 0, T, n, branches)[1]
                       for b in range(BATCH))
            assert steps == want


def test_sampled_at_zero_temperature_with_penalties_is_greedy(dev):
    run = _runner(dev)
    g = torch.Generator(device=dev).manual_seed(6)
    prompt = torch.randint(0, 64, (BATCH, CTX + 1), device=dev, generator=g)
    _set_penalties(run, **PEN)
    for n, branches in ((1, 1), (4, 1), (8, 2)):
        run.s_temperature.fill_(1.0); run.s_top_k.fill_(1)
        greedy, _ = _speculative(run, prompt, n, branches, penalties=True)
        run.s_temperature.fill_(0.0); run.s_top_k.fill_(-1); run.s_top_p.fill_(1.0)
        sampled, _ = _speculative(run, prompt, n, branches, sampled=True, penalties=True)
        assert torch.equal(greedy, sampled), n


def _snapshot(run, K):
    pages = [p.clone() for p in run.kpools + run.vpools + run.kpools_gen + run.vpools_gen]
    return [t.clone() for t in _state(run)] + [run.g_logprob.clone(), *[t.clone() for t in run.g_top_view(K)]] + pages


@pytest.mark.parametrize("n,branches", [(1, 1), (4, 1), (8, 2)])
def test_graph_replay_equals_eager_with_penalties_logprobs_and_stops(dev, n, branches):
    run = _runner(dev, "w4a8kv8")
    g = torch.Generator(device=dev).manual_seed(5)
    prompt = torch.randint(0, 64, (BATCH, CTX + 1), device=dev, generator=g)
    _set_penalties(run, **PEN)
    K, steps = 5, 6
    plain, _, _ = _plain(run, prompt, penalties=True)
    run.g_stop[:, 0] = plain[:, 4]  # rows stop at (or before) their fifth plain token
    run.g_stop[:3, 1] = plain[:3, 2]
    run.reset_generation(prompt)
    run.capture_generate(n, branches, penalties=True, logprobs=K)
    run.g_logprob.fill_(float("nan"))
    run.reset_generation(prompt)
    with torch.no_grad():
        for _ in range(steps):
            run.generate_forward(n, branches, penalties=True, logprobs=K)
    torch.cuda.synchronize()
    eager = _snapshot(run, K)
    assert bool(run.g_finished.any())
    run.g_logprob.fill_(float("nan"))
    run.reset_generation(prompt)
    for _ in range(steps):
        run.generate_step(n, branches, penalties=True, logprobs=K)
    torch.cuda.synchronize()
    for a, b in zip(_snapshot(run, K), eager):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)


def test_prefill_hand_off_with_logprobs_and_stops(dev):
    run = _runner(dev, prompt_tokens=BATCH * CTX)
    g = torch.Generator(device=dev).manual_seed(9)
    lens_h = [1, 40, 63, 64, 99, 100]
    prompts = torch.randint(0, 64, (BATCH, CTX), device=dev, generator=g)
    lens = torch.tensor(lens_h, dtype=torch.int32, device=dev)
    _set_penalties(run, **PEN)
    K = 5
    first = run.prefill(prompts, lens, penalties=True, logprobs=K)
    run.capture_generate(1, penalties=True, logprobs=K)
    run.capture_generate(4, 1, penalties=True, logprobs=K)
    run.g_logprob.fill_(float("nan"))
    run.prefill(prompts, lens, penalties=True, logprobs=K)
    rows = torch.arange(BATCH, device=dev)
    assert torch.equal(run.g_logprob[rows, lens.long()], run.s_logprob)
    for i in range(8):
        run.generate_step(1 if i % 2 == 0 else 4, 1, penalties=True, logprobs=K)
    torch.cuda.synchronize()
    lp = run.g_logprob.cpu()
    for b in range(BATCH):
        end = int(run.s_seq_lens[b])
        assert end > lens_h[b] + 8
        assert bool(torch.isfinite(lp[b, lens_h[b]:end]).all()) and bool(torch.isnan(lp[b, :lens_h[b]]).all()), b
    # a stop id as the first token finishes the row
    run.g_stop.fill_(-1)
    run.g_stop[2, 3] = first[2]
    run.g_stop[4, 0] = first[4]
    run.prefill(prompts, lens, penalties=True, logprobs=K)
    assert run.g_finished.tolist() == [0, 0, 1, 0, 1, 0]
