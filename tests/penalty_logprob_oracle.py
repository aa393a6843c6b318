"""Oracle: repetition / presence / frequency penalties and top-n log-probabilities (TEST INFRASTRUCTURE, not product).

States the contract of qs_apply_penalties and qs_logprobs_rows:
  * `apply_penalties`: vLLM's penalty semantics in the kernel's exact fp32 step order (x / rep or x * rep, then x - (frequency * c), then
    x - presence, each an IEEE fp32 operation), one rounding to fp16; only history tokens whose value changes are written;
  * `logprobs_rows`: the T = 1 softmax with the sampler's conventions in float64 (NaN and -inf weigh 0, w = 1 at the maximum so +inf logits
    share the mass), the chosen token's log-probability and the top n by (logit descending, index ascending).
"""
from __future__ import annotations

import numpy as np

MAX_HISTORY = 32768
MAX_TOP = 20


def _per_row(a, R, dt):
    return np.broadcast_to(np.asarray(a, dt), (R,))


def apply_penalties(logits, history, prompt_lens, seq_lens, repetition, presence, frequency):
    """fp16 logits [R, V] -> the penalised copy.  history int64 [R, H]; prompt_lens / seq_lens [R]; parameters [R] or scalars."""
    x = np.array(logits, np.float16, copy=True)
    R, V = x.shape
    history = np.asarray(history, np.int64)
    H = history.shape[1]
    rep, pres, freq = (_per_row(a, R, np.float32) for a in (repetition, presence, frequency))
    pls, sls = np.asarray(prompt_lens, np.int64), np.asarray(seq_lens, np.int64)
    for r in range(R):
        if rep[r] == 1 and pres[r] == 0 and freq[r] == 0:
            continue
        hl = int(min(max(sls[r], 0), H))
        pl = int(min(max(pls[r], 0), hl))
        ids = history[r, :hl]
        ok = (ids >= 0) & (ids < V)
        out = np.arange(hl) >= pl
        counts = np.bincount(ids[ok & out], minlength=V)
        t = np.unique(ids[ok])
        if t.size == 0:
            continue
        old = x[r, t]
        xf = old.astype(np.float32)
        with np.errstate(invalid="ignore", over="ignore"):
            if rep[r] != 1:
                xf = np.where(xf > 0, xf / rep[r], xf * rep[r]).astype(np.float32)
            c = counts[t]
            pen = ((xf - freq[r] * c.astype(np.float32)).astype(np.float32) - pres[r]).astype(np.float32)
            xf = np.where(c > 0, pen, xf)
        new = xf.astype(np.float16)
        x[r, t] = np.where(np.isnan(old), old, new)
    return x


def logprobs_rows(logits, tokens, n: int):
    """fp16 logits [R, V], tokens [R] -> (logprob float64 [R], top_ids int64 [R, n], top_logprobs float64 [R, n])."""
    x = np.asarray(logits, np.float16).astype(np.float64)
    R, V = x.shape
    tokens = np.asarray(tokens, np.int64)
    lp = np.full(R, np.nan)
    ids = np.full((R, n), -1, np.int64)
    tlp = np.full((R, n), np.nan)
    for r in range(R):
        row = x[r]
        nan = np.isnan(row)
        valid = ~nan & (row != -np.inf)
        if not valid.any():
            continue
        m = row[valid].max()
        with np.errstate(invalid="ignore", over="ignore"):
            rel = np.where(row == m, 0.0, row - m)  # -inf below a +inf maximum and at -inf logits
        w = np.where(valid, np.exp(rel), 0.0)
        lrow = np.where(nan, np.nan, rel - np.log(w.sum()))
        t = int(tokens[r])
        lp[r] = lrow[t] if 0 <= t < V else np.nan
        cand = np.flatnonzero(~nan)
        order = cand[np.lexsort((cand, -row[cand]))][:n]  # logit descending, index ascending (-0 == +0)
        ids[r, : order.size] = order
        tlp[r, : order.size] = lrow[order]
        tlp[r, order.size:] = -np.inf
    return lp, ids, tlp
