"""Oracle: temperature / top-p / top-k sampling and sampled acceptance of draft trees, in float64 (TEST INFRASTRUCTURE, not product).

States the contract of qs_sample_rows and qs_tree_accept_sampling:
  * `philox4x32_10` / `uniform`: the counter-based draws, bit for bit (counter (lo(off), hi(off), row, j), key (lo(seed), hi(seed)),
    u = (x0 >> 8) * 2^-24, exact in float32 and float64);
  * `warp`: steps 1-5 -- greedy rows, z = float32(x) / float32(T), w = exp(z - max z) (NaN / -inf weigh 0), the kept set
    {z >= max(tau_p, tau_k)} with both thresholds computed on the full row;
  * `sample`: step 6, the inverse CDF in token-index order;
  * `tree_accept_sampling`: SpecInfer multi-step speculative sampling over a draft tree.
Each decision also reports its margin (how far it is from flipping), which the GPU tests use to excuse fp32 rounding.

The reference (qserve/modeling/layers/sampler.py) applies TopP then TopK in fp16 and draws with torch.multinomial: the distribution agrees
up to its fp16 rounding, the random stream does not.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from .tree import ancestors

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 on uint32 counters; ctr: 4 arrays (or ints), key: 2 arrays (or ints), broadcast together.  Returns 4 uint64 arrays."""
    c = [np.asarray(x, np.uint64) & MASK32 for x in ctr]
    k = [np.asarray(x, np.uint64) & MASK32 for x in key]
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & np.uint64(MASK32), (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & np.uint64(MASK32)]
        k = [(k[0] + np.uint64(W0)) & np.uint64(MASK32), (k[1] + np.uint64(W1)) & np.uint64(MASK32)]
    return c


def uniform(seed: int, offset, row, j):
    """The draw u in [0, 1 - 2^-24] (float64, exactly the kernel's float32 value); offset / row / j broadcast."""
    off = np.asarray(offset, np.int64).astype(np.uint64)
    seed = int(seed) & ((1 << 64) - 1)
    x0 = philox4x32_10((off & np.uint64(MASK32), off >> np.uint64(32), row, j), (seed & MASK32, seed >> 32))[0]
    return (x0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def is_greedy(temperature, top_p) -> bool:
    return bool(np.float32(temperature) < np.float32(1e-5) or np.float32(top_p) < np.float32(1e-8))


def argmax_row(x) -> int:
    """argmax_rows / torch.argmax: first maximal index, NaN counts as the maximum."""
    x = np.asarray(x, np.float32)
    nan = np.isnan(x)
    return int(np.argmax(nan)) if nan.any() else int(np.argmax(x))


def warp(x, temperature, top_k, top_p):
    """Steps 1-5 for one fp16 logit row.  Returns (w float64 [V], kept bool [V], info): w is the unnormalised kept weight (0 outside the
    kept set).  info: 'greedy' (True: w is one-hot at the argmax), 'top_p_margin' (min over distinct z of |W(> z) - top_p S| / S, inf if
    top-p is off), 'S' (sum of all weights)."""
    x = np.asarray(x, np.float16)
    V = x.size
    xf = x.astype(np.float32)
    valid = ~np.isnan(xf) & ~(xf == -np.inf)
    if is_greedy(temperature, top_p) or not valid.any():
        w = np.zeros(V)
        w[argmax_row(xf)] = 1.0
        return w, w > 0, {"greedy": True, "top_p_margin": np.inf, "S": 1.0}
    z = np.where(valid, xf / np.float32(temperature), np.float32(-np.inf)).astype(np.float32)
    mz = z[valid].max()
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.where(valid, np.where(z == mz, 1.0, np.exp(z.astype(np.float64) - np.float64(mz))), 0.0)
    S = w.sum()
    tau = -np.inf
    margin = np.inf
    zs, inv = np.unique(z[valid], return_inverse=True)
    group = np.bincount(inv, weights=w[valid], minlength=zs.size)[::-1]  # weight of each distinct z, descending z
    zs = zs[::-1]
    if top_k > 0:
        kk = min(int(top_k), int(valid.sum()))
        tau = max(tau, np.sort(z[valid])[::-1][kk - 1])
    if top_p < 1:
        # W(> z) for each distinct z: keep z iff W(> z) < top_p * S
        above = np.concatenate([[0.0], np.cumsum(group)[:-1]])
        keep = above < np.float64(np.float32(top_p)) * S
        tau_p = zs[keep].min()
        margin = float(np.min(np.abs(above - np.float64(np.float32(top_p)) * S)) / S)
        tau = max(tau, tau_p)
    kept = valid & (z >= tau)
    return np.where(kept, w, 0.0), kept, {"greedy": False, "top_p_margin": margin, "S": S}


def kept_topp_then_topk(x, temperature, top_k, top_p):
    """The kept set by the reference's order, applied one after the other (TopP on the full row, then TopK on what survives as -inf
    elsewhere); equals warp()'s {z >= max(tau_p, tau_k)}."""
    x = np.asarray(x, np.float16).astype(np.float32)
    z = (x / np.float32(temperature)).astype(np.float64)
    keep = np.ones(z.size, bool)
    if top_p < 1:
        w = np.exp(z - z.max())
        S = w.sum()
        above = np.array([w[z > z[i]].sum() for i in range(z.size)])
        keep &= above < np.float64(np.float32(top_p)) * S
    if top_k > 0:
        zk = np.where(keep, z, -np.inf)
        kth = np.sort(zk)[::-1][min(int(top_k), z.size) - 1]
        keep &= zk >= kth
    return keep


def sample(w, u: float):
    """Step 6: the smallest index t with sum_{j <= t} w_j > u * sum w.  Returns (t, cdf float64 [V])."""
    c = np.cumsum(np.asarray(w, np.float64))
    t = int(np.searchsorted(c, u * c[-1], side="right"))
    return min(t, c.size - 1), c


def cdf_ok(token: int, w, u: float, rel: float = 4e-6) -> bool:
    """The bar for a token drawn by fp32 / fixed-point arithmetic: w[token] > 0 and its CDF interval [c_{t-1}, c_t] lies within
    rel * S of u * S."""
    w = np.asarray(w, np.float64)
    if not (0 <= token < w.size) or w[token] <= 0:
        return False
    c = np.cumsum(w)
    S, x = c[-1], u * c[-1]
    lo = c[token] - w[token]
    return lo - rel * S <= x <= c[token] + rel * S


def sample_rows(x, temperature, top_k, top_p, seed, offsets):
    """Reference answer of qs_sample_rows for fp16 logits [rows, V] and per-row parameters (arrays or scalars).  Returns (tokens int64
    [rows], w list of the kept weights, top-p margins [rows], u [rows])."""
    x = np.asarray(x, np.float16)
    R = x.shape[0]
    T, K, P = (np.broadcast_to(np.asarray(a), (R,)) for a in (temperature, top_k, top_p))
    u = uniform(seed, np.asarray(offsets, np.int64), np.arange(R), 0)
    toks, ws, margins = np.zeros(R, np.int64), [], np.zeros(R)
    for r in range(R):
        w, _, info = warp(x[r], float(T[r]), int(K[r]), float(P[r]))
        toks[r] = argmax_row(x[r]) if info["greedy"] else sample(w, u[r])[0]
        ws.append(w)
        margins[r] = info["top_p_margin"]
    return toks, ws, margins, u


def residual(p, q):
    """p <- max(p - q, 0) renormalised; p itself when the residual mass is 0."""
    r = np.maximum(np.asarray(p, np.float64) - np.asarray(q, np.float64), 0.0)
    s = r.sum()
    return r / s if s > 0 else np.asarray(p, np.float64)


def parents_of(tree_mask_row, n: int):
    return [-1] + [max(ancestors(tree_mask_row[c], c), default=-1) for c in range(1, n)]


def tree_accept_sampling(draft, tree_mask, logits, temperature, top_k, top_p, seed, offsets, draft_probs: Optional[np.ndarray] = None):
    """Reference answer of qs_tree_accept_sampling.  draft int64 [B, n], tree_mask int32 [B, n], logits fp16 [B, n, V], per-sequence
    parameters, draft_probs float [B, n, V] or None (one-hot at the draft).  Returns (accept_len int32 [B], path int32 [B, n], bonus int64
    [B], info) with info[b] = {'margin': the smallest |p(d) - u q(d)| over the acceptance decisions, 'bonus_p': the distribution the bonus
    was drawn from, 'u0': its draw, 'top_p_margin': the smallest top-p margin of the warped rows}."""
    draft, tree_mask, logits = np.asarray(draft), np.asarray(tree_mask), np.asarray(logits, np.float16)
    B, n, V = logits.shape
    T, K, P = (np.broadcast_to(np.asarray(a), (B,)) for a in (temperature, top_k, top_p))
    offsets = np.asarray(offsets, np.int64)
    accept_len, path, bonus = np.zeros(B, np.int32), np.full((B, n), -1, np.int32), np.zeros(B, np.int64)
    info = []
    for b in range(B):
        parent = parents_of(tree_mask[b], n)
        margin, pmargin = np.inf, np.inf

        def target(node):
            nonlocal pmargin
            w, _, inf = warp(logits[b, node], float(T[b]), int(K[b]), float(P[b]))
            pmargin = min(pmargin, inf["top_p_margin"])
            return w / w.sum()

        p = target(0)
        cur, walk = 0, [0]
        while True:
            nxt = None
            for c in range(cur + 1, n):
                if parent[c] != cur:
                    continue
                d = int(draft[b, c])
                if d < 0 or d >= V:
                    continue
                if draft_probs is None:
                    q = np.zeros(V)
                    q[d] = 1.0
                else:
                    q = np.asarray(draft_probs[b, c], np.float64)
                u = float(uniform(seed, offsets[b], b, c))
                lhs, rhs = u * q[d], p[d]
                margin = min(margin, abs(rhs - lhs))
                if lhs < rhs:
                    nxt = c
                    break
                p = residual(p, q)
            if nxt is None:
                break
            cur = nxt
            walk.append(cur)
            p = target(cur)
        u0 = float(uniform(seed, offsets[b], b, 0))
        accept_len[b] = len(walk)
        path[b, : len(walk)] = walk
        bonus[b] = sample(p, u0)[0]
        info.append({"margin": margin, "bonus_p": p, "u0": u0, "top_p_margin": pmargin})
    return accept_len, path, bonus, info
