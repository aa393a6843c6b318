"""Oracle of prompt-lookup speculative decoding (test infrastructure, not product): `ngram_propose` and `spec_commit` restated in plain
Python integers from the contract in include/qserve_b200.h, and a CPU speculative loop built from them and `oracle.tree.tree_accept_greedy`.
The GPU ops must match these bit for bit."""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np

from oracle.tree import tree_accept_greedy

PAD_TOKEN, PAD_MASK = -1, 1


def match_len(h, L: int, j: int, n_max: int) -> int:
    """m(j): the largest g <= min(n_max, j + 1) with h[j - g + 1 .. j] == h[L - g .. L - 1], every id of both windows >= 0."""
    g = 0
    while g < min(n_max, j + 1) and h[L - 1 - g] >= 0 and h[j - g] == h[L - 1 - g]:
        g += 1
    return g


def candidates(h, L: int, n_min: int, n_max: int, branches: int):
    """The first `branches` end positions j with m(j) >= n_min, by (m descending, j descending)."""
    c = [(match_len(h, L, j, n_max), j) for j in range(L - 1)]
    c = [x for x in c if x[0] >= n_min]
    c.sort(reverse=True)
    return [j for _, j in c[:branches]]


def propose_row(h, L: int, n: int, n_min: int, n_max: int, branches: int):
    """One row: (tokens [n], mask [n]) as Python int lists."""
    h = [int(x) for x in h]
    L = min(max(int(L), 0), len(h))
    toks = [h[L - 1] if L > 0 else -1] + [PAD_TOKEN] * (n - 1)
    mask = [0] + [PAD_MASK] * (n - 1)
    parent = [-1] * n
    cnt = 1
    if L >= 2:
        for j in candidates(h, L, n_min, n_max, branches):
            if cnt == n:
                break
            cur = 0
            for t in h[j + 1: min(j + n - 1, L - 1) + 1]:
                child = [i for i in range(1, cnt) if parent[i] == cur and toks[i] == t]
                if child:
                    cur = child[0]
                    continue
                if cnt == n:
                    break
                toks[cnt], parent[cnt], mask[cnt] = t, cur, mask[cur] | (1 << cur)
                cur, cnt = cnt, cnt + 1
    return toks, mask


def ngram_propose(history, seq_lens, n: int, n_min: int = 1, n_max: int = 4, branches: int = 1):
    """history int64 [B, H], seq_lens [B] -> (tokens int64 [B, n], tree_mask int32 [B, n])."""
    history = np.asarray(history, np.int64)
    B = history.shape[0]
    tokens = np.zeros((B, n), np.int64)
    mask = np.zeros((B, n), np.int32)
    for b in range(B):
        t, m = propose_row(history[b], int(seq_lens[b]), n, n_min, n_max, branches)
        tokens[b], mask[b] = t, m
    return tokens, mask


def spec_commit(draft, path, accept_len, bonus, history, seq_lens, prompt_lens, budget, eos, finished):
    """In place on copies: returns (history, seq_lens, finished, start_pos, context_lens, roots) after the commit.  start_pos / context_lens /
    roots of finished rows are None (the op leaves them untouched)."""
    draft, path = np.asarray(draft, np.int64), np.asarray(path, np.int64)
    history = np.array(history, np.int64)
    seq_lens, finished = np.array(seq_lens, np.int32), np.array(finished, np.int32)
    B, n = draft.shape
    H = history.shape[1]
    start, ctx, roots = [None] * B, [None] * B, [None] * B
    for b in range(B):
        if finished[b]:
            continue
        L = min(max(int(seq_lens[b]), 0), H)
        acc = min(max(int(accept_len[b]), 1), n)
        app = [int(draft[b, min(max(int(path[b, k]), 0), n - 1)]) for k in range(1, acc)] + [int(bonus[b])]
        hit = False
        e = int(eos[b])
        if e >= 0 and e in app:
            app = app[: app.index(e) + 1]
            hit = True
        room = max(int(budget[b]) - (L - int(prompt_lens[b])), 0)
        if len(app) > room:
            app, hit = app[:room], False
        for k, t in enumerate(app):
            if L + k < H:
                history[b, L + k] = t
        last = app[-1] if app else (int(history[b, L - 1]) if L > 0 else -1)
        L2 = L + len(app)
        seq_lens[b] = L2
        start[b], ctx[b], roots[b] = L2 - 1, L2, last
        if hit or L2 - int(prompt_lens[b]) >= int(budget[b]):
            finished[b] = 1
    return history, seq_lens, finished, start, ctx, roots


def speculative_generate(prompt, next_token: Callable, T: int, n: int, branches: int = 1, n_min: int = 1, n_max: int = 4, eos: Optional[int] = None):
    """The speculative loop on the CPU for one row: propose -> next_token of every node's root path -> tree_accept_greedy -> commit, until T
    tokens are generated or eos is appended.  next_token(seq) is the target model's greedy token after the token list seq.  Returns (the
    generated tokens, the number of steps)."""
    prompt = [int(x) for x in prompt]
    H = len(prompt) + T
    hist = np.full((1, H), -1, np.int64)
    hist[0, : len(prompt)] = prompt
    lens = np.array([len(prompt)], np.int32)
    fin = np.zeros(1, np.int32)
    steps = 0
    e = -1 if eos is None else int(eos)
    while not fin[0]:
        L = int(lens[0])
        toks, mask = ngram_propose(hist, lens, n, n_min, n_max, branches)
        seq = [int(x) for x in hist[0, :L]]
        target = np.zeros((1, n), np.int64)
        for i in range(n):
            if toks[0, i] < 0 and i > 0:
                target[0, i] = -1  # padding: never on an accepted path
                continue
            anc = [j for j in range(i) if (int(mask[0, i]) >> j) & 1]
            target[0, i] = next_token(seq + [int(toks[0, j]) for j in anc if j > 0] + ([int(toks[0, i])] if i > 0 else []))
        acc, path, bonus = tree_accept_greedy(toks, mask, target)
        hist, lens, fin, _, _, _ = spec_commit(toks, path, acc, bonus, hist, lens, [len(prompt)], [T], [e], fin)
        steps += 1
    return [int(x) for x in hist[0, len(prompt): int(lens[0])]], steps
