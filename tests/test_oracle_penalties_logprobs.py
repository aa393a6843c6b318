"""CPU: the penalty and log-probability oracles (tests/penalty_logprob_oracle.py) against independent torch restatements.

  * penalties: vLLM's sampler code (bin counts by scatter_add with padding id V, repetition by torch.where over the prompt | output mask,
    then logits -= frequency * counts and logits -= presence * mask) in fp32, then .half().  vLLM also subtracts 0 * penalty from tokens
    that were never generated, which can only flip the sign of a zero, so logits are compared by value, and bitwise where a token was
    generated;
  * log-probabilities: torch.log_softmax in float64 (NaN as -inf; a row with +inf logits as 0 there and -inf elsewhere) and a stable
    descending sort over the non-NaN logits.
"""
import numpy as np
import pytest
import torch

from tests import penalty_logprob_oracle as opl


def _vllm_penalties(logits, history, prompt_lens, seq_lens, rep, pres, freq):
    x = torch.from_numpy(logits).float()
    R, V = x.shape
    H = history.shape[1]
    prompt = torch.full((R, H), V, dtype=torch.int64)
    output = torch.full((R, H), V, dtype=torch.int64)
    for r in range(R):
        hl = min(max(int(seq_lens[r]), 0), H)
        pl = min(max(int(prompt_lens[r]), 0), hl)
        ids = torch.from_numpy(history[r, :hl].copy())
        ids = torch.where((ids >= 0) & (ids < V), ids, torch.full_like(ids, V))
        prompt[r, :pl] = ids[:pl]
        output[r, : hl - pl] = ids[pl:]

    def bins(tokens):
        b = torch.zeros((R, V + 1), dtype=torch.int64)
        b.scatter_add_(1, tokens, torch.ones_like(tokens))
        b = b[:, :V]
        return b, b > 0

    _, prompt_mask = bins(prompt)
    counts, output_mask = bins(output)
    rp = torch.from_numpy(np.asarray(rep, np.float32))[:, None].repeat(1, V)
    rp[~(prompt_mask | output_mask)] = 1.0
    x = torch.where(x > 0, x / rp, x * rp)
    x -= torch.from_numpy(np.asarray(freq, np.float32))[:, None] * counts
    x -= torch.from_numpy(np.asarray(pres, np.float32))[:, None] * output_mask
    return x.half().numpy(), counts.numpy()


def _history(rng, R, H, V):
    h = rng.integers(0, min(V, 40), (R, H))  # heavy duplication
    h[rng.random((R, H)) < 0.1] = -1
    h[rng.random((R, H)) < 0.05] = V + 3
    return h


@pytest.mark.parametrize("V", [64, 1024])
def test_penalty_oracle_is_vllm(V):
    rng = np.random.default_rng(V)
    R, H = 24, 96
    x = (rng.standard_normal((R, V)) * 3).astype(np.float16)
    x[0, :40:3] = np.nan
    x[1, :40:2] = np.inf
    x[2, :40:2] = -np.inf
    x[3, :40] = 0.0
    x[4, :40] = -0.0
    h = _history(rng, R, H, V)
    seq = rng.integers(0, H + 1, R).astype(np.int32)
    prompt = np.minimum(rng.integers(0, H + 1, R), seq).astype(np.int32)
    seq[5], prompt[5] = 0, 0      # empty history
    seq[6], prompt[6] = 50, 50    # prompt only
    seq[7], prompt[7] = 50, 0     # output only
    rep = rng.choice([0.01, 0.5, 1.0, 1.3, 2.0], R).astype(np.float32)
    pres = rng.choice([-2.0, -0.5, 0.0, 0.7, 2.0], R).astype(np.float32)
    freq = rng.choice([-2.0, -0.3, 0.0, 1.1, 2.0], R).astype(np.float32)
    rep[8], pres[8], freq[8] = 1.0, 0.0, 0.0
    got = opl.apply_penalties(x, h, prompt, seq, rep, pres, freq)
    want, counts = _vllm_penalties(x, h, prompt, seq, rep, pres, freq)
    assert np.array_equal(got.astype(np.float32), want.astype(np.float32), equal_nan=True)
    gen = counts > 0
    assert np.array_equal(got.view(np.uint16)[gen], want.view(np.uint16)[gen])
    assert np.array_equal(got[8].view(np.uint16), x[8].view(np.uint16))  # neutral row untouched
    assert not np.array_equal(got.view(np.uint16), x.view(np.uint16))


def test_penalty_oracle_clamps_lengths_and_ignores_bad_ids():
    x = np.arange(16, dtype=np.float16).reshape(1, 16) - 8
    h = np.array([[3, -1, 40, 3, 5, 12]])
    got = opl.apply_penalties(x, h, [-4], [99], 2.0, 0.5, 1.0)  # clamped to prompt 0, seq 6: every valid id is output
    want = x.copy()
    for t, c in ((3, 2), (5, 1), (12, 1)):
        v = np.float32(x[0, t])
        v = v / np.float32(2) if v > 0 else v * np.float32(2)
        want[0, t] = np.float16(np.float32(np.float32(v - np.float32(c)) - np.float32(0.5)))
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))


def _torch_logprobs(x16, tokens, n):
    x = torch.from_numpy(x16.astype(np.float64))
    R, V = x.shape
    nan = torch.isnan(x)
    z = torch.where(nan, torch.full_like(x, -np.inf), x)
    pinf = (z == np.inf).any(dim=1, keepdim=True)
    z = torch.where(pinf, torch.where(z == np.inf, torch.zeros_like(z), torch.full_like(z, -np.inf)), z)
    lsm = torch.log_softmax(z, dim=-1)
    lsm = torch.where(nan, torch.full_like(lsm, np.nan), lsm)
    lp = np.array([lsm[r, t].item() if 0 <= t < V else np.nan for r, t in enumerate(tokens)])
    ids = np.full((R, n), -1, np.int64)
    tlp = np.full((R, n), np.nan)
    for r in range(R):
        if torch.isnan(lsm[r][~nan[r]]).all():  # no weight (or no non-NaN logit)
            lp[r] = np.nan
            continue
        cand = torch.nonzero(~nan[r]).flatten()
        order = cand[torch.sort(x[r, cand], descending=True, stable=True).indices][:n]
        ids[r, : order.numel()] = order.numpy()
        tlp[r, : order.numel()] = lsm[r, order].numpy()
        tlp[r, order.numel():] = -np.inf
    return lp, ids, tlp


@pytest.mark.parametrize("n", [0, 1, 5, 20])
def test_logprob_oracle_is_log_softmax_and_stable_topk(n):
    rng = np.random.default_rng(n)
    R, V = 12, 256
    x = (rng.standard_normal((R, V)) * 2).astype(np.float16)
    x[0] = (rng.integers(-2, 3, V) * 0.5).astype(np.float16)  # ties everywhere
    x[1, [5, 9, 200]] = np.inf                               # +inf shares the mass
    x[2, ::2] = -np.inf
    x[3, ::3] = np.nan
    x[4] = np.nan                                            # all masked
    x[5] = -np.inf
    x[6] = np.nan
    x[6, [3, 7]] = -np.inf                                   # no weight, two -inf
    x[7] = np.nan
    x[7, [10, 11, 12]] = [1.0, -np.inf, 1.0]                 # fewer than n non-NaN
    x[8, :10] = 0.0
    x[8, 10:20] = -0.0                                       # -0 ties with +0
    x[8, 20:] = -1.0
    tokens = rng.integers(0, V, R)
    tokens[9], tokens[10] = -1, V
    tokens[3] = 3  # a NaN logit
    got = opl.logprobs_rows(x, tokens, n)
    want = _torch_logprobs(x, tokens, n)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12, atol=1e-12, equal_nan=True)
    assert np.array_equal(got[1], want[1])
    np.testing.assert_allclose(got[2], want[2], rtol=1e-12, atol=1e-12, equal_nan=True)
    assert np.isnan(got[0][[4, 5, 6, 9, 10, 3]]).all()
    if n:
        assert (got[1][[4, 5, 6]] == -1).all() and np.isnan(got[2][[4, 5, 6]]).all()
        assert got[1][7, 0] == 10 and (n < 2 or got[1][7, 1] == 12)
        assert (got[1][7, 3:] == -1).all() and (got[2][7, 3:] == -np.inf).all()
        np.testing.assert_allclose(got[2][1, : min(n, 3)], -np.log(3.0))
        assert list(got[1][8, : min(n, 20)]) == list(range(min(n, 20)))
