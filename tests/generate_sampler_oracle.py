"""Oracle of the generation loop's sampler ops (test infrastructure, not product): the contracts of qs_apply_penalties_tree,
qs_spec_commit_stops and the column placement of qs_logprobs_accepted, restated on top of tests/penalty_logprob_oracle.py and
tests/ngram_oracle.py.  The GPU ops must match these bit for bit."""
from __future__ import annotations

import numpy as np

from tests import penalty_logprob_oracle as plo


def path_nodes(mask_word: int, i: int) -> list:
    """The nodes whose tokens node i's expanded history appends: its ancestors j >= 1 in index order, then i itself (i >= 1)."""
    return [j for j in range(1, i) if (int(mask_word) >> j) & 1] + ([i] if i >= 1 else [])


def expand_histories(draft, tree_mask, history, prompt_lens, seq_lens):
    """Per-node expanded histories: (history int64 [B n, H + 16], prompt_lens [B n], seq_lens [B n]).  Row b n + i holds h[0 .. L) (L =
    seq_lens[b] clamped to [0, H]), then the tokens of path_nodes(tree_mask[b, i], i); unused columns are -1."""
    draft, tree_mask, history = np.asarray(draft, np.int64), np.asarray(tree_mask, np.int64), np.asarray(history, np.int64)
    B, n = draft.shape
    H = history.shape[1]
    out = np.full((B * n, H + 16), -1, np.int64)
    pl = np.zeros(B * n, np.int32)
    sl = np.zeros(B * n, np.int32)
    for b in range(B):
        L = min(max(int(seq_lens[b]), 0), H)
        for i in range(n):
            toks = [int(draft[b, j]) for j in path_nodes(tree_mask[b, i], i)]
            r = b * n + i
            out[r, :L] = history[b, :L]
            out[r, L:L + len(toks)] = toks
            pl[r], sl[r] = int(prompt_lens[b]), L + len(toks)
    return out, pl, sl


def apply_penalties_tree(logits, draft, tree_mask, history, prompt_lens, seq_lens, repetition, presence, frequency):
    """fp16 logits [B, n, V] -> the penalised copy: penalty_logprob_oracle.apply_penalties over the expanded histories, parameters per row."""
    x = np.asarray(logits, np.float16)
    B, n, V = x.shape
    per = lambda a: np.repeat(np.broadcast_to(np.asarray(a, np.float32), (B,)), n)
    h, pl, sl = expand_histories(draft, tree_mask, history, prompt_lens, seq_lens)
    return plo.apply_penalties(x.reshape(B * n, V), h, pl, sl, per(repetition), per(presence), per(frequency)).reshape(B, n, V)


def spec_commit_stops(draft, path, accept_len, bonus, history, seq_lens, prompt_lens, budget, eos, stop_ids, finished):
    """ngram_oracle.spec_commit where any token of {eos[b]} and stop_ids[b] (entries < 0 ignored) ends the row as eos does.  Same returns."""
    draft, path = np.asarray(draft, np.int64), np.asarray(path, np.int64)
    stop_ids = np.asarray(stop_ids, np.int64).reshape(len(draft), -1)
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
        stops = {int(t) for t in [eos[b], *stop_ids[b]] if int(t) >= 0}
        hit = False
        first = next((k for k, t in enumerate(app) if t in stops), None)
        if first is not None:
            app, hit = app[: first + 1], True
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


def accepted_entries(draft, path, accept_len, bonus, seq_lens, finished, W: int):
    """Where qs_logprobs_accepted writes: a list of (b, column, node row, token) for every unfinished row b and emitted token k < acc whose
    column min(max(seq_lens[b], 0), W) + k lies below W."""
    draft, path = np.asarray(draft, np.int64), np.asarray(path, np.int64)
    B, n = draft.shape
    out = []
    for b in range(B):
        if finished[b]:
            continue
        acc = min(max(int(accept_len[b]), 1), n)
        L = min(max(int(seq_lens[b]), 0), W)
        node = lambda k: min(max(int(path[b, k]), 0), n - 1)
        for k in range(acc):
            if L + k >= W:
                break
            tok = int(draft[b, node(k + 1)]) if k + 1 < acc else int(bonus[b])
            out.append((b, L + k, node(k), tok))
    return out

