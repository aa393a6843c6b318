"""Beam search as the decode runner implements it: vLLM 0.3's algorithm (llm_engine._process_sequence_group_outputs with the sampler's
_beam_search_sample), restated over arrays.  The C entries qs_beam_select / qs_beam_reorder and DecodeRunner.beam_* follow this contract.

Layout and parameters
  * R requests of W beams each, 1 <= W <= 8 (so 2 W <= 16 <= MAX_TOP_LOGPROBS).  Request r owns rows r W .. r W + W - 1; batch = R W.
  * Per request: length_penalty fp32, early_stopping int32 (0 = False, 1 = True, 2 = "never"), eos int64 (-1 = none), up to 8 stop ids
    (-1 pads) and budget = max_tokens (clamped to [1, T], T = the pool's tokens per hypothesis).
  * Per beam slot: live int32 and cum fp32 (the cumulative log-probability).
  * Every live beam of a request has the same length L = P0 + out_len: the prompt length P0 plus the generated tokens.

One step of request r (skipped when the request is done; its slots then only get parent -1):
  1. Candidates.  For each live slot j, logprobs_rows(logits_j, ., 2 W): ids and lp, ordered by logit descending, then index ascending.  Ids < 0
     are skipped.  The candidate score is s = fp32(cum_j + lp).
  2. Selection.  Sort all candidates of the request by (s descending, j ascending, rank ascending) and keep the first 2 W: the children, in
     that order.
  3. Finishing.  A child finishes if its token is eos, or one of the stop ids, or out_len + 1 >= budget.
  4. Scoring a finished child.  cum / len ** length_penalty with len = P0 + out_len + 1, minus 1 if the token is eos (only eos, as in vLLM's
     get_beam_search_score).
  5. Finished pool.  The stored hypotheses in stored order, then the new finished children in child order, sorted by score descending with a
     stable sort; the first W are stored in that order.  A hypothesis holds its generated tokens (the parent's, then the child's token), their
     count, cum and score.
  6. Running children: the children that did not finish, in child order.
  7. Stopping.  The request is done if no child is running; or the pool holds W hypotheses and early_stopping is 1; or the pool holds W,
     early_stopping is 0 and worst.score >= the best running child's score at its current length; or the pool holds W, early_stopping is 2 and
     worst.score >= the best running child's score at len = max(P0 + budget, max_model_len) (only when length_penalty > 0; otherwise at its
     current length as for 0).  max_model_len is a runner constant, ctx + max_new_tokens.
  8. New beams.  If the request is not done, running child i < W goes into slot r W + i with its parent slot, token and cum = s, live = 1.  The
     remaining slots die (live = 0, parent -1).  If the request is done, every slot dies.  Every slot of the request gets seq_len =
     context_len = L + 1 (cum and token of a dead slot are left as they are).

The first step runs on the prefill logits with only slot r W live and cum = 0: vLLM's prompt-phase topk(2 W) of the single sequence.

The reorder then gives every slot with a parent p != itself p's page-table entries below P / 64, the filled slots of p's tail page and history
columns [P0, P), P = L; every live slot appends its token at column P.  Here only the history part is modelled.

The results of a request are its pool, best first.

Numerics.  The cum and s sums are fp32 in a fixed order, so every running-beam decision is bitwise reproducible.  With length_penalty 1 (or 0)
a score is a correctly rounded fp32 division, so it is bitwise too.  With other penalties the GPU powf may differ from numpy's in the last
ulps: scores then agree within NEAR_TIE, and a request may decide differently only where a comparison that decided it was that close
(select's margins, mismatched).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def score(cum, length: int, length_penalty) -> np.float32:
    """cum / length ** length_penalty in fp32."""
    return F32(F32(cum) / np.power(F32(length), F32(length_penalty)))


def init_state(prompt_lens, beam_width: int, max_tokens: int, history_len: int, prompts=None) -> dict:
    """The state before the first step: slot r W live with cum 0, every slot of request r at length P0 = prompt_lens[r]; history holds the
    prompt (prompts[r], or zeros) and -1 after it."""
    R, W = len(prompt_lens), int(beam_width)
    B = R * W
    P0 = np.repeat(np.asarray(prompt_lens, np.int32), W)
    hist = np.full((B, history_len), -1, np.int64)
    for b in range(B):
        hist[b, : P0[b]] = 0 if prompts is None else np.asarray(prompts[b // W])[: P0[b]]
    live = np.zeros(B, np.int32)
    live[::W] = 1
    return dict(live=live, cum=np.zeros(B, F32), seq_lens=P0.copy(), context_lens=P0 + 1, tokens=np.zeros(B, np.int64),
                parents=np.full(B, -1, np.int32), prompt_lens=P0.copy(), history=hist, done=np.zeros(R, np.int32),
                pool_tokens=np.full((R, W, max_tokens), -1, np.int64), pool_len=np.zeros((R, W), np.int32), pool_cum=np.zeros((R, W), F32),
                pool_score=np.zeros((R, W), F32), pool_count=np.zeros(R, np.int32))


def params(R: int, max_tokens: int, max_model_len: int, length_penalty=1.0, early_stopping=0, eos=-1, stop_ids=None) -> dict:
    """Per-request parameters (scalars broadcast)."""
    stop = np.full((R, 8), -1, np.int64) if stop_ids is None else np.asarray(stop_ids, np.int64).reshape(R, -1)
    return dict(length_penalty=np.broadcast_to(np.asarray(length_penalty, F32), (R,)).copy(),
                early_stopping=np.broadcast_to(np.asarray(early_stopping, np.int32), (R,)).copy(),
                eos=np.broadcast_to(np.asarray(eos, np.int64), (R,)).copy(), stop_ids=stop,
                budget=np.full(R, max_tokens, np.int32), max_model_len=int(max_model_len))


# With length_penalty outside {0, 1} the GPU's powf and numpy's may differ by a few ulps.  A request whose outcome differs from the oracle's is
# explained only if a score comparison that decided it had two sides within this relative distance (select's `margins`).
NEAR_TIE = 2.0 ** -19


def _gap(a, b) -> float:
    """Relative distance of two scores that went through powf; inf where no rounding can move them (equal zeros or infinities, or one
    side infinite)."""
    a, b = float(a), float(b)
    if (a == b and (a == 0.0 or not np.isfinite(a))) or not (np.isfinite(a) and np.isfinite(b)):
        return float("inf")
    return abs(a - b) / max(abs(a), abs(b))


def select(st: dict, prm: dict, top_ids, top_lp, margins: list | None = None) -> dict:
    """One qs_beam_select: returns the new state (st is not modified).  top_ids int64 / top_lp fp32 [B, 2 W].  margins (a list) receives
    per request the smallest relative distance (_gap) between the two sides of a score comparison that decided it: adjacent entries of the
    sorted pool merge (not two stored hypotheses, nor two new ones from the same cum and length, whose bits cannot differ) and the stopping
    comparison of early_stopping 0 / 2; inf when no such comparison ran."""
    st = {k: v.copy() for k, v in st.items()}
    R, W, T = st["pool_tokens"].shape
    C, H = 2 * W, st["history"].shape[1]
    top_ids, top_lp = np.asarray(top_ids, np.int64), np.asarray(top_lp, F32)
    for r in range(R):
        base = r * W
        margin = float("inf")
        if st["done"][r]:
            st["parents"][base: base + W] = -1
            if margins is not None:
                margins.append(margin)
            continue
        L, P0 = int(st["seq_lens"][base]), int(st["prompt_lens"][base])
        out_len = L - P0
        budget = min(max(int(prm["budget"][r]), 1), T)
        lp, eos = F32(prm["length_penalty"][r]), int(prm["eos"][r])
        stops = [int(x) for x in prm["stop_ids"][r] if x >= 0]
        cands = []  # (s, j, rank, token)
        for j in range(W):
            if not st["live"][base + j]:
                continue
            for k in range(C):
                tok = int(top_ids[base + j, k])
                if tok >= 0:
                    cands.append((F32(st["cum"][base + j] + top_lp[base + j, k]), j, k, tok))
        cands.sort(key=lambda c: (-float(c[0]), c[1], c[2]))
        children = cands[:C]
        items = [(F32(st["pool_score"][r, q]), ("old", q)) for q in range(min(max(int(st["pool_count"][r]), 0), W))]
        running = []
        for c, (s, j, _, tok) in enumerate(children):
            fin = (eos >= 0 and tok == eos) or out_len + 1 >= budget or tok in stops
            if fin:
                flen = L + 1 - (1 if eos >= 0 and tok == eos else 0)
                items.append((score(s, flen, lp), ("new", c), (float(s), flen)))
            else:
                running.append(c)
        items = [it if len(it) == 3 else (it[0], it[1], None) for it in items]
        items.sort(key=lambda it: -float(it[0]))  # stable
        for (a, (ka, _), ia), (b, (kb, _), ib) in zip(items, items[1:]):
            if not (ka == kb == "old" or (ia is not None and ia == ib)):
                margin = min(margin, _gap(a, b))
        items = [it[:2] for it in items]
        kept = items[:W]
        old = (st["pool_tokens"][r].copy(), st["pool_len"][r].copy(), st["pool_cum"][r].copy())
        for q, (sc, (kind, i)) in enumerate(kept):
            if kind == "old":
                st["pool_tokens"][r, q], st["pool_len"][r, q], st["pool_cum"][r, q] = old[0][i], old[1][i], old[2][i]
            else:
                s, j, _, tok = children[i]
                n = min(max(out_len + 1, 0), T)
                row = st["pool_tokens"][r, q]  # entries past the hypothesis' length are unspecified
                gen = [int(st["history"][base + j, P0 + x]) if P0 + x < H else -1 for x in range(min(out_len, T))]
                row[: len(gen)] = gen
                if 0 <= out_len < T:
                    row[out_len] = tok
                st["pool_len"][r, q], st["pool_cum"][r, q] = n, s
            st["pool_score"][r, q] = sc
        count = len(kept)
        done = not running
        if not done and count == W:
            es = int(prm["early_stopping"][r])
            if es == 1:
                done = True
            else:
                best = children[running[0]][0]
                length = max(P0 + budget, prm["max_model_len"]) if es == 2 and lp > 0 else L + 1
                bound = score(best, length, lp)
                done = bool(st["pool_score"][r, W - 1] >= bound)
                margin = min(margin, _gap(st["pool_score"][r, W - 1], bound))
        for i in range(W):
            slot = base + i
            if not done and i < len(running):
                s, j, _, tok = children[running[i]]
                st["parents"][slot], st["tokens"][slot], st["cum"][slot], st["live"][slot] = base + j, tok, s, 1
            else:
                st["parents"][slot], st["live"][slot] = -1, 0
            st["seq_lens"][slot] = st["context_lens"][slot] = L + 1
        st["pool_count"][r], st["done"][r] = count, int(done)
        if margins is not None:
            margins.append(margin)
    return st


def mismatched(got: dict, want: dict, exact: bool = True) -> list:
    """The requests whose state differs between got and want: done, every slot's live / parent / lengths, the live slots' token and cum bits,
    the pool count and every valid pool entry (tokens up to its length, length, cum bits, and the score bits if exact, else within
    NEAR_TIE)."""
    R, W, _ = want["pool_tokens"].shape
    bad = []
    for r in range(R):
        rows = slice(r * W, r * W + W)
        live = want["live"][rows].astype(bool)
        ok = got["done"][r] == want["done"][r] and got["pool_count"][r] == want["pool_count"][r]
        ok = ok and all(np.array_equal(got[k][rows], want[k][rows]) for k in ("live", "parents", "seq_lens", "context_lens"))
        ok = ok and np.array_equal(got["tokens"][rows][live], want["tokens"][rows][live])
        ok = ok and np.array_equal(got["cum"][rows][live].view(np.uint32), want["cum"][rows][live].view(np.uint32))
        for q in range(int(want["pool_count"][r]) if ok else 0):
            n = int(want["pool_len"][r, q])
            a, b = F32(got["pool_score"][r, q]), F32(want["pool_score"][r, q])
            ok = ok and int(got["pool_len"][r, q]) == n and np.array_equal(got["pool_tokens"][r, q, :n], want["pool_tokens"][r, q, :n])
            ok = ok and F32(got["pool_cum"][r, q]).view(np.uint32) == F32(want["pool_cum"][r, q]).view(np.uint32)
            ok = ok and (a.view(np.uint32) == b.view(np.uint32) if exact else (a == b or _gap(a, b) <= NEAR_TIE))
        if not ok:
            bad.append(r)
    return bad


def reorder_history(st: dict) -> dict:
    """The history part of qs_beam_reorder, in place: with P = context_lens[r W] - 1 for request r, slots re-parented inside their request
    take the parent's columns [P0, P) and every slot whose parent lies in its request appends its token at P."""
    B, H = st["history"].shape
    W = st["pool_tokens"].shape[1]
    old = st["history"].copy()
    for s in range(B):
        p, base = int(st["parents"][s]), s - s % W
        if not base <= p < base + W:
            continue
        P, P0 = int(st["context_lens"][base]) - 1, max(int(st["prompt_lens"][s]), 0)  # one P per request: its first slot's
        if p != s and P > 0 and min(P, H) > P0:
            st["history"][s, P0: min(P, H)] = old[p, P0: min(P, H)]
        if 0 <= P < H:
            st["history"][s, P] = st["tokens"][s]
    return st


def same_pool(a: dict, b: dict) -> bool:
    """Equal pools: counts, and every valid entry's tokens (up to its length), length, cum and score bits."""
    if not np.array_equal(a["pool_count"], b["pool_count"]):
        return False
    for r, c in enumerate(a["pool_count"]):
        for q in range(int(c)):
            n = int(a["pool_len"][r, q])
            if n != int(b["pool_len"][r, q]) or not np.array_equal(a["pool_tokens"][r, q, :n], b["pool_tokens"][r, q, :n]):
                return False
            for k in ("pool_cum", "pool_score"):
                if np.float32(a[k][r, q]).view(np.uint32) != np.float32(b[k][r, q]).view(np.uint32):
                    return False
    return True


def step(st: dict, prm: dict, top_ids, top_lp) -> dict:
    """select followed by the history part of the reorder."""
    return reorder_history(select(st, prm, top_ids, top_lp))


def results(st: dict, n: int) -> list:
    """Per request, its best n hypotheses: (tokens, cum, score)."""
    out = []
    for r in range(st["pool_count"].shape[0]):
        c = min(int(st["pool_count"][r]), n)
        out.append([(st["pool_tokens"][r, q, : st["pool_len"][r, q]].tolist(), float(st["pool_cum"][r, q]), float(st["pool_score"][r, q]))
                    for q in range(c)])
    return out
