"""GPU: repetition / presence / frequency penalties (qs_apply_penalties) and top-n log-probabilities (qs_logprobs_rows) against the oracle
(tests/penalty_logprob_oracle.py), and the decode runner's penalised / logprob steps.

Penalties are bitwise: the kernel and the oracle make the same IEEE fp32 operations and one fp16 rounding; the whole logit tensor is
compared, so neutral rows and logits outside the history must be untouched.  top_ids are exact (the order is decided on the fp16 logits).
logprob / top_logprobs agree to within 1e-5 + 1e-6 |lp|: the kernel sums fp32 expf weights (a few ulp each) in 64-bit fixed point after
rounding each to 2^-41, so log S is off by ~1e-7 relative; the float64 oracle is exact.
"""
import numpy as np
import pytest
import torch

from tests import penalty_logprob_oracle as opl

pytestmark = pytest.mark.gpu


def _backend():
    from qserve_b200 import backend
    return backend


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _t(a, dev, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if dt is None else t.to(dt)


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. penalties
# ---------------------------------------------------------------------------------------------------------------------------------
def _penalty_case(rng, R, V, H, special=True):
    x = (rng.standard_normal((R, V)) * 3).astype(np.float16)
    h = rng.integers(0, V, (R, H))
    hot = rng.integers(0, V, 16)
    dup = rng.random((R, H)) < 0.6
    h[dup] = hot[rng.integers(0, 16, dup.sum())]  # heavy duplication
    h[rng.random((R, H)) < 0.05] = -1
    h[rng.random((R, H)) < 0.03] = V + rng.integers(0, 5)
    h[rng.random((R, H)) < 0.01] = -7
    seq = rng.integers(0, H + 1, R).astype(np.int32)
    prompt = np.minimum(rng.integers(0, H + 1, R), seq).astype(np.int32)
    kinds = [(0, 0), (H, H), (H, 0), (H // 2, H), (-3, H + 50)]  # empty, prompt only, output only, ..., out-of-range lengths (clamped)
    for r, (p, s) in zip(range(1, R, 3), kinds):
        prompt[r], seq[r] = p, s
    if special:  # +-0, +-inf, NaN at history positions
        for r in range(R):
            t = h[r, : max(seq[r], 1)][:8]
            t = t[(t >= 0) & (t < V)]
            x[r, t] = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 65504, -65504, 1e-7], np.float16)[: t.size]
    rep = rng.choice([0.01, 0.5, 1.0, 1.2, 2.0], R).astype(np.float32)
    pres = rng.choice([-2.0, -0.4, 0.0, 0.9, 2.0], R).astype(np.float32)
    freq = rng.choice([-2.0, -0.25, 0.0, 0.6, 2.0], R).astype(np.float32)
    rep[2::4], pres[2::4], freq[2::4] = 1.0, 0.0, 0.0  # neutral rows
    rep[0], pres[0], freq[0], prompt[0], seq[0] = 1.2, 0.5, 0.6, H // 2, H  # row 0 always changes
    return x, h, prompt, seq, rep, pres, freq


def _run_penalties(dev, x, h, prompt, seq, rep, pres, freq):
    be = _backend()
    xd = _t(x, dev)
    pars = [p if np.isscalar(p) else _t(p, dev) for p in (rep, pres, freq)]
    out = be.apply_penalties(xd, _t(h, dev), _t(prompt, dev), _t(seq, dev), *pars)
    assert out.data_ptr() == xd.data_ptr()
    torch.cuda.synchronize()
    return xd.cpu().numpy()


@pytest.mark.parametrize("V,rows,H", [(1024, 1, 300), (1024, 7, 1000), (32000, 64, 4096), (128256, 200, 512), (128256, 7, 8192), (152064, 64, 2048)])
def test_penalties_match_oracle(dev, V, rows, H):
    rng = np.random.default_rng(V + rows + H)
    case = _penalty_case(rng, rows, V, H)
    got = _run_penalties(dev, *case)
    want = opl.apply_penalties(*case)
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    neutral = (case[4] == 1) & (case[5] == 0) & (case[6] == 0)
    assert np.array_equal(got[neutral].view(np.uint16), case[0][neutral].view(np.uint16))
    assert not np.array_equal(got.view(np.uint16), case[0].view(np.uint16))


@pytest.mark.parametrize("rep,pres,freq", [(2.0, -2.0, 2.0), (1e-3, 2.0, -2.0), (1.0, 0.0, 0.0), (1.0, 0.5, 0.0), (0.7, 0.0, 0.0)])
def test_penalties_scalar_parameters(dev, rep, pres, freq):
    rng = np.random.default_rng(7)
    x, h, prompt, seq, *_ = _penalty_case(rng, 64, 32000, 1024)
    got = _run_penalties(dev, x, h, prompt, seq, rep, pres, freq)
    want = opl.apply_penalties(x, h, prompt, seq, rep, pres, freq)
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))


def test_penalties_at_the_history_cap(dev):
    be = _backend()
    rng = np.random.default_rng(11)
    H = be.MAX_PENALTY_HISTORY
    case = _penalty_case(rng, 7, 32000, H)
    case[3][:] = H
    case[3][0] = H - 1
    got = _run_penalties(dev, *case)
    assert np.array_equal(got.view(np.uint16), opl.apply_penalties(*case).view(np.uint16))
    x = torch.zeros((1, 64), dtype=torch.half, device=dev)
    one = torch.ones(1, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x, torch.zeros((1, H + 1), dtype=torch.int64, device=dev), one, one, 1.1, 0.0, 0.0)


def test_penalties_are_deterministic_and_capturable(dev):
    be = _backend()
    rng = np.random.default_rng(3)
    x, h, prompt, seq, rep, pres, freq = _penalty_case(rng, 64, 128256, 2048)
    args = [_t(a, dev) for a in (h, prompt, seq, rep, pres, freq)]
    a, b, c = (_t(x, dev) for _ in range(3))
    be.apply_penalties(a, *args)
    be.apply_penalties(b, *args)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        be.apply_penalties(_t(x, dev), *args)  # warm-up: kernel attributes
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        be.apply_penalties(c, *args)
    c.copy_(_t(x, dev))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(a.view(torch.int16), c.view(torch.int16))


def test_penalty_argument_errors(dev):
    be = _backend()
    x = torch.zeros((2, 64), dtype=torch.half, device=dev)
    h = torch.zeros((2, 8), dtype=torch.int64, device=dev)
    ln = torch.full((2,), 4, dtype=torch.int32, device=dev)
    for bad in (dict(repetition=0.0), dict(repetition=2.5), dict(presence=2.1), dict(frequency=-2.1)):
        kw = dict(repetition=1.1, presence=0.0, frequency=0.0)
        kw.update(bad)
        with pytest.raises(RuntimeError):
            be.apply_penalties(x, h, ln, ln, **kw)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x, h.int(), ln, ln, 1.1, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x, h[:1], ln, ln, 1.1, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x, h, ln.long(), ln, 1.1, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x.float(), h, ln, ln, 1.1, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(torch.zeros((2, 60), dtype=torch.half, device=dev), h, ln, ln, 1.1, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x, h, ln, ln, torch.ones(3, device=dev), 0.0, 0.0)
    with pytest.raises(RuntimeError):
        be.apply_penalties(x.cpu(), h, ln, ln, 1.1, 0.0, 0.0)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. log-probabilities
# ---------------------------------------------------------------------------------------------------------------------------------
def _logit_rows(rng, R, V):
    x = (rng.standard_normal((R, V)) * 3).astype(np.float16)
    for r in range(R):
        kind = r % 8
        if kind == 1:
            x[r] = (rng.integers(-3, 4, V) * 1.25)  # heavy ties
        elif kind == 2:
            x[r, rng.integers(0, V, 3)] = np.inf
        elif kind == 3:
            x[r, rng.random(V) < 0.5] = -np.inf
            x[r, rng.integers(0, V, 5)] = np.nan
        elif kind == 4:
            x[r] = np.nan
            x[r, rng.integers(0, V, 3)] = [1.0, -np.inf, 1.0]  # fewer than n non-NaN logits
        elif kind == 5:
            x[r] = -np.inf if r % 16 == 5 else np.nan  # no weight
        elif kind == 6:
            x[r, : V // 2] = 0.0
            x[r, V // 2:] = -0.0
    return x


def _check_logprobs(x, tok, n, got):
    lp, ids, tlp = (g.cpu().numpy() for g in got)
    wlp, wids, wtlp = opl.logprobs_rows(x, tok, n)
    assert np.array_equal(ids, wids)
    np.testing.assert_allclose(lp, wlp, rtol=1e-6, atol=1e-5, equal_nan=True)
    np.testing.assert_allclose(tlp, wtlp, rtol=1e-6, atol=1e-5, equal_nan=True)


@pytest.mark.parametrize("V", [1024, 32000, 128256, 152064])
@pytest.mark.parametrize("n", [0, 1, 5, 20])
def test_logprobs_match_oracle(dev, V, n):
    be = _backend()
    rng = np.random.default_rng(V + n)
    R = 24
    x = _logit_rows(rng, R, V)
    tok = rng.integers(0, V, R)
    tok[0], tok[9] = -1, V
    xd = _t(x, dev)
    got = be.logprobs_rows(xd, _t(tok, dev), n)
    torch.cuda.synchronize()
    _check_logprobs(x, tok, n, got)
    if n:
        xf = x.astype(np.float32)
        rows = ~np.isnan(xf).any(axis=1) & (xf != -np.inf).any(axis=1)  # no NaN, some weight
        am = be.argmax_rows(xd).cpu().numpy()
        assert rows.sum() >= R // 2 and np.array_equal(got[1].cpu().numpy()[rows, 0], am[rows])


def test_prompt_logprobs_shape(dev):
    """prompt_logprobs: one row per prompt position (2048 rows), the next prompt token as the chosen token."""
    be = _backend()
    rng = np.random.default_rng(5)
    R, V, n = 2048, 32000, 5
    x = (rng.standard_normal((R, V)) * 2).astype(np.float16)
    tok = rng.integers(0, V, R)
    got = be.logprobs_rows(_t(x, dev), _t(tok, dev), n)
    torch.cuda.synchronize()
    assert got[0].shape == (R,) and got[1].shape == (R, n) and got[2].shape == (R, n)
    _check_logprobs(x, tok, n, got)


def test_logprobs_deterministic_and_graph_replay(dev):
    be = _backend()
    rng = np.random.default_rng(9)
    R, V, n = 64, 128256, 20
    x = _t(_logit_rows(rng, R, V), dev)
    tok = _t(rng.integers(0, V, R), dev)
    a = be.logprobs_rows(x, tok, n)
    b = be.logprobs_rows(x, tok, n)
    outs = (torch.empty(R, device=dev), torch.empty((R, n), dtype=torch.int64, device=dev), torch.empty((R, n), device=dev))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        be.logprobs_rows(x, tok, n, *outs)
    g.replay()
    torch.cuda.synchronize()
    for u, v, w in zip(a, b, outs):
        assert torch.equal(_bits(u), _bits(v)) and torch.equal(_bits(u), _bits(w))


def test_logprob_argument_errors(dev):
    be = _backend()
    x = torch.zeros((4, 64), dtype=torch.half, device=dev)
    tok = torch.zeros(4, dtype=torch.int64, device=dev)
    for bad in ((x, tok, 21), (x, tok, -1), (x, tok.int(), 5), (x, tok[:3], 5), (x.float(), tok, 5), (x[:, :60].contiguous(), tok, 5),
                (x.cpu(), tok, 5)):
        with pytest.raises(RuntimeError):
            be.logprobs_rows(*bad)
    with pytest.raises(RuntimeError):
        be.logprobs_rows(x, tok, 5, top_ids=torch.empty((4, 4), dtype=torch.int64, device=dev))
    with pytest.raises(RuntimeError):
        be.logprobs_rows(x, tok, 5, logprob=torch.empty(4, dtype=torch.float64, device=dev))


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. the decode runner
# ---------------------------------------------------------------------------------------------------------------------------------
def test_runner_neutral_penalties_change_nothing(dev):
    from qserve_b200.decode import DecodeRunner

    plain = DecodeRunner("tiny", "w4a8kv4", batch=5, ctx=130, device=dev, seed=3)
    run = DecodeRunner("tiny", "w4a8kv4", batch=5, ctx=130, device=dev, seed=3, max_new_tokens=4)
    assert torch.equal(plain.embed, run.embed) and torch.equal(plain.kpools[0], run.kpools[0])  # no extra generator draws
    run.s_history[:, :130] = torch.randint(0, run.cfg.vocab, (5, 130), device=dev)
    run.tokens_in.copy_(torch.arange(5, device=dev) * 7)
    run.s_temperature.fill_(0.9); run.s_top_k.fill_(-1); run.s_top_p.fill_(0.95)
    with torch.no_grad():
        greedy = run.forward(run.tokens_in).clone()
        greedy_p = run.forward(run.tokens_in, penalties=True).clone()
        run.s_offsets.zero_()
        sampled = run.forward(run.tokens_in, sample=True).clone()
        run.s_offsets.zero_()
        sampled_p = run.forward(run.tokens_in, sample=True, penalties=True, logprobs=3).clone()
    torch.cuda.synchronize()
    assert torch.equal(greedy, greedy_p) and torch.equal(sampled, sampled_p)
    assert torch.equal(run.s_seq_lens, torch.full((5,), 132, dtype=torch.int32, device=dev))
    assert torch.equal(run.s_history[:, 130], greedy) and torch.equal(run.s_history[:, 131], sampled)


@pytest.mark.parametrize("model,batch,layers", [("tiny", 5, None), ("llama-3-8b", 64, 1)])
def test_runner_replays_equal_the_eager_composition(dev, model, batch, layers):
    be = _backend()
    from qserve_b200.decode import DecodeRunner

    ctx, n = 130, 5
    run = DecodeRunner(model, "w4a8kv4", batch=batch, ctx=ctx, device=dev, seed=4, layers=layers, max_new_tokens=6)
    V = run.cfg.vocab
    g = torch.Generator(device=dev).manual_seed(1)
    run.s_history[:, :ctx] = torch.randint(0, 64, (batch, ctx), device=dev, generator=g)  # a small alphabet: many repeats
    run.s_prompt_lens.copy_(torch.randint(0, ctx, (batch,), device=dev, generator=g).int())
    run.s_repetition.copy_(torch.rand(batch, device=dev, generator=g) + 0.5)
    run.s_presence.copy_(torch.rand(batch, device=dev, generator=g) * 4 - 2)
    run.s_frequency.copy_(torch.rand(batch, device=dev, generator=g) * 4 - 2)
    run.s_temperature.fill_(0.8); run.s_top_k.fill_(-1); run.s_top_p.fill_(0.95)
    run.tokens_in.copy_(torch.randint(0, V, (batch,), device=dev, generator=g))
    run.capture(sample=True, penalties=True, logprobs=n)  # two eager warm-up steps append two tokens
    assert torch.equal(run.s_seq_lens, torch.full((batch,), ctx + 2, dtype=torch.int32, device=dev))
    for _ in range(3):
        hist, seq, off = run.s_history.clone(), run.s_seq_lens.clone(), run.s_offsets.clone()
        with torch.no_grad():
            logits = run._forward_fused(run.tokens_in, True).clone()
        be.apply_penalties(logits, hist, run.s_prompt_lens, seq, run.s_repetition, run.s_presence, run.s_frequency)
        tok = be.sample_rows(logits, run.s_temperature, run.s_top_k, run.s_top_p, run.s_seed, off.clone())
        lp, ids, tlp = be.logprobs_rows(logits, tok, n)
        hist[torch.arange(batch, device=dev), seq.long()] = tok
        run.step((True, True, n))
        torch.cuda.synchronize()
        ids_g, tlp_g = run.top_logprobs_view(n)
        assert torch.equal(run.tokens_out, tok)
        assert torch.equal(_bits(run.s_logprob), _bits(lp))
        assert torch.equal(ids_g, ids) and torch.equal(_bits(tlp_g), _bits(tlp))
        assert torch.equal(run.s_history, hist) and torch.equal(run.s_seq_lens, seq + 1) and torch.equal(run.s_offsets, off + 1)
        assert bool((lp <= 0).all()) and bool(torch.isfinite(lp).all())
