"""CPU tests of beam search: the array oracle (tests/beam_oracle.py) against a literal restatement of vLLM 0.3's list-of-Sequence algorithm over
random multi-step candidate streams, the exported C signatures, and the host checks of backend.beam_select / beam_reorder and of
DecodeRunner(beam_width=...)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import beam_oracle as bo

F32 = np.float32


class _Seq:
    """vLLM's Sequence, reduced to what beam search reads."""

    def __init__(self, prompt_len, tokens=(), cum=F32(0)):
        self.prompt_len, self.output, self.cum, self.finished = prompt_len, list(tokens), F32(cum), False

    def fork(self):
        return _Seq(self.prompt_len, self.output, self.cum)

    def append(self, tok, lp):
        self.output.append(tok)
        self.cum = F32(self.cum + F32(lp))

    def get_len(self):
        return self.prompt_len + len(self.output)

    def get_beam_search_score(self, length_penalty, seq_len=None, eos_token_id=None):  # sequence.py
        if seq_len is None:
            seq_len = self.get_len()
            if eos_token_id is not None and self.output and self.output[-1] == eos_token_id:
                seq_len -= 1
        return F32(self.cum / np.power(F32(seq_len), F32(length_penalty)))


class _Group:
    """One request: vLLM 0.3's _process_sequence_group_outputs for use_beam_search, with the sampler's top-2W selection in the contract's order."""

    def __init__(self, prompt_len, W, lp, es, eos, stops, budget, max_model_len):
        self.W, self.lp, self.es, self.eos, self.stops, self.budget, self.max_model_len = W, lp, es, eos, stops, budget, max_model_len
        self.running, self.finished, self.done = [_Seq(prompt_len)], [], False

    def _check_stop(self, seq):  # llm_engine._check_stop (stop strings are host work; the max_model_len cap never binds in the runner)
        tok = seq.output[-1]
        seq.finished = tok in self.stops or len(seq.output) == self.budget or (self.eos is not None and tok == self.eos)

    def _score(self, seq):
        return seq.get_beam_search_score(self.lp, eos_token_id=self.eos)

    def _early_stop(self, best_running, worst_finished):  # llm_engine._check_beam_search_early_stopping
        if self.es == 1:
            return True
        worst = self._score(worst_finished)
        if self.es == 0:
            best = self._score(best_running)
        elif self.lp > 0:
            best = best_running.get_beam_search_score(self.lp, seq_len=max(best_running.prompt_len + self.budget, self.max_model_len),
                                                      eos_token_id=self.eos)
        else:
            best = self._score(best_running)
        return worst >= best

    def step(self, cands):
        """cands[j] = (ids, lps) of running sequence j (slot order)."""
        if self.done:
            return
        flat = [(F32(seq.cum + F32(lp)), j, k, int(t), lp) for j, (seq, (ids, lps)) in enumerate(zip(self.running, cands))
                for k, (t, lp) in enumerate(zip(ids, lps)) if t >= 0]
        flat.sort(key=lambda c: (-float(c[0]), c[1], c[2]))
        child_seqs = []
        for _, j, _, t, lp in flat[: 2 * self.W]:
            child = self.running[j].fork()
            child.append(t, lp)
            self._check_stop(child)
            child_seqs.append(child)
        all_finished = self.finished + [c for c in child_seqs if c.finished]
        all_finished.sort(key=self._score, reverse=True)
        running = [c for c in child_seqs if not c.finished]
        running.sort(key=self._score, reverse=True)
        if not running:
            stop = True
        elif len(all_finished) < self.W:
            stop = False
        else:
            stop = self._early_stop(running[0], all_finished[self.W - 1])
        self.finished = all_finished[: self.W]
        self.running = [] if stop else running[: self.W]
        self.done = stop


def _candidates(rng, W, vocab, nan_p=0.1, short_p=0.2):
    """One slot's logprobs_rows(n = 2 W) output: distinct ids ordered by lp descending (coarse values, so ties occur), NaN rows all -1,
    short rows padded with -1."""
    C = 2 * W
    if rng.random() < nan_p:
        return np.full(C, -1, np.int64), np.full(C, np.nan, F32)
    ids = rng.choice(vocab, size=C, replace=False).astype(np.int64)
    lps = -(rng.integers(0, 12, C) * F32(0.25) + F32(0.03125) * rng.integers(0, 2, C)).astype(F32)
    order = np.lexsort((ids, -lps))  # lp descending, equal logits by index ascending
    ids, lps = ids[order], lps[order]
    if rng.random() < short_p:
        k = int(rng.integers(1, C))
        ids[k:], lps[k:] = -1, -np.inf
    return ids, lps


def _run(seed, W, lp, es, eos_mode, R=3, steps=14, vocab=12):
    rng = np.random.default_rng(seed)
    vocab = max(vocab, 2 * W + 4)
    P0 = [int(x) for x in rng.integers(1, 40, R)]
    T = int(rng.integers(2, 10))
    max_model_len = 60
    eos = {"none": -1, "eos": int(rng.integers(0, vocab))}[eos_mode if eos_mode != "stop" else "none"]
    stops = np.full((R, 8), -1, np.int64)
    if eos_mode == "stop":
        stops[:, :2] = rng.choice(vocab, 2, replace=False)
    prm = bo.params(R, T, max_model_len, lp, es, eos, stops)
    prm["budget"] = rng.integers(1, T + 1, R).astype(np.int32)
    groups = [_Group(P0[r], W, F32(lp), es, None if eos < 0 else eos, [int(x) for x in stops[r] if x >= 0], int(prm["budget"][r]), max_model_len)
              for r in range(R)]
    st = bo.init_state(P0, W, T, max(P0) + T + 2)
    for _ in range(steps):
        top_ids = np.full((R * W, 2 * W), -1, np.int64)
        top_lp = np.full((R * W, 2 * W), np.nan, F32)
        for b in range(R * W):
            top_ids[b], top_lp[b] = _candidates(rng, W, vocab)
        for r, g in enumerate(groups):
            g.step([(top_ids[r * W + j], top_lp[r * W + j]) for j in range(len(g.running))])
        st = bo.step(st, prm, top_ids, top_lp)
        for r, g in enumerate(groups):
            base = r * W
            assert bool(st["done"][r]) == g.done, (r, st["done"][r], g.done)
            live = [j for j in range(W) if st["live"][base + j]]
            assert live == list(range(len(g.running))), (live, len(g.running))
            for j, seq in enumerate(g.running):
                L = int(st["seq_lens"][base + j])
                assert st["history"][base + j, P0[r]:L].tolist() == seq.output
                assert F32(st["cum"][base + j]).view(np.uint32) == seq.cum.view(np.uint32)
            assert int(st["pool_count"][r]) == len(g.finished)
            for q, seq in enumerate(g.finished):
                n = int(st["pool_len"][r, q])
                assert st["pool_tokens"][r, q, :n].tolist() == seq.output
                assert F32(st["pool_score"][r, q]).view(np.uint32) == g._score(seq).view(np.uint32)
        if all(g.done for g in groups):
            break
    return st, groups


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("lp", [1.0, 0.5, 2.0, 0.0, -1.0])
@pytest.mark.parametrize("es", [0, 1, 2])
@pytest.mark.parametrize("eos_mode", ["none", "eos", "stop"])
def test_oracle_matches_vllm_restatement(W, lp, es, eos_mode):
    for seed in range(4):
        _run(1000 * W + 17 * seed + es, W, lp, es, eos_mode)


def test_all_children_finish_at_once():
    """Every candidate is eos (all 2 W children finish): the pool takes the best W, the request is done and every slot dies."""
    W, R, T = 2, 1, 8
    prm = bo.params(R, T, 40, 1.0, 0, eos=5)
    st = bo.init_state([10], W, T, 20)
    ids = np.array([[5, -1, -1, -1], [-1, -1, -1, -1]], np.int64)
    st = bo.step(st, prm, ids, np.array([[-0.5, np.nan, np.nan, np.nan], [np.nan] * 4], F32))
    assert st["done"][0] == 1 and st["live"].tolist() == [0, 0] and st["parents"].tolist() == [-1, -1]
    assert st["pool_count"][0] == 1 and st["pool_tokens"][0, 0, :1].tolist() == [5]
    assert st["pool_score"][0, 0] == F32(-0.5) / F32(10)  # eos does not count in the length
    st2 = bo.step(st, prm, ids, np.zeros((2, 4), F32))
    assert st2["parents"].tolist() == [-1, -1] and bo.same_pool(st, st2)


def test_budget_ends_the_search():
    W, R, T = 2, 1, 3
    prm = bo.params(R, T, 40, 1.0, 1)
    st = bo.init_state([4], W, T, 12)
    ids = np.array([[1, 2, 3, 4], [5, 6, 7, 8]], np.int64)
    lps = np.array([[-0.1, -0.2, -0.3, -0.4], [-0.15, -0.25, -0.35, -0.45]], F32)
    for _ in range(3):
        st = bo.step(st, prm, ids, lps)
    assert st["done"][0] == 1 and st["pool_count"][0] == 2
    assert [len(h[0]) for h in bo.results(st, 2)[0]] == [3, 3]


def guard_case():
    """One request, W = 1, a full pool and early_stopping 2 at length_penalty -1, where the "never" bound at max(P0 + budget, max_model_len)
    would stop the search and the current-length bound (the rule for length_penalty <= 0) does not.  Returns (state, params, ids, lps)."""
    st = bo.init_state([10], 1, 64, 80)
    st["seq_lens"][:] = st["context_lens"][:] = 12
    st["history"][0, 10:12] = [3, 4]
    st["cum"][:] = F32(-0.75)
    st["pool_count"][0], st["pool_len"][0, 0], st["pool_cum"][0, 0], st["pool_score"][0, 0] = 1, 2, F32(-1.5), F32(-20.0)
    prm = bo.params(1, 64, 40, -1.0, 2)
    ids = np.array([[5, 6]], np.int64)
    lps = np.array([[-0.25, -0.5]], F32)
    return st, prm, ids, lps


def test_near_tie_rule_can_fail():
    """The near-tie rule excuses a differing request only where a deciding comparison was within NEAR_TIE: a kernel that applied the "never"
    bound at length_penalty <= 0 decides this case differently with a margin far above it, and the rule reports it."""
    st, prm, ids, lps = guard_case()
    margins = []
    want = bo.select(st, prm, ids, lps, margins)
    assert want["done"][0] == 0 and want["live"][0] == 1
    s = F32(F32(-0.75) + F32(-0.25))
    assert F32(-20.0) < bo.score(s, 13, -1.0) and F32(-20.0) >= bo.score(s, 74, -1.0)  # current length: go on; max(10 + 64, 40): stop
    wrong = {k: v.copy() for k, v in want.items()}
    wrong["done"][0], wrong["live"][0], wrong["parents"][0] = 1, 0, -1
    assert bo.mismatched(wrong, want, exact=False) == [0]
    assert margins[0] > bo.NEAR_TIE
    assert bo.mismatched(want, want, exact=False) == []


def test_c_entries_are_exported():
    from qserve_b200 import _lib

    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("qs_beam_select", "qs_beam_reorder"):
        assert name in _lib.SIGNATURES and hasattr(raw, name)


def test_backend_rejects_bad_arguments():
    from qserve_b200 import backend

    R, W, T = 2, 4, 8
    B = R * W
    i32 = lambda *s: torch.zeros(s, dtype=torch.int32)
    i64 = lambda *s: torch.zeros(s, dtype=torch.int64)
    f32 = lambda *s: torch.zeros(s, dtype=torch.float32)
    pool = backend.beam_pool(R, W, T, "cpu")

    def select(**kw):
        a = dict(top_ids=i64(B, 2 * W), top_logprobs=f32(B, 2 * W), live=i32(B), cum=f32(B), seq_lens=i32(B), context_lens=i32(B), tokens=i64(B),
                 parents=i32(B), prompt_lens=i32(B), history=i64(B, 16), length_penalty=f32(R), early_stopping=i32(R), eos=i64(R), stop_ids=i64(R, 8),
                 budget=i32(R), done=i32(R), pool=pool, max_model_len=64)
        a.update(kw)
        backend.beam_select(**a)

    with pytest.raises(RuntimeError, match="beam width"):
        select(top_ids=i64(18 * 2, 2 * 9), top_logprobs=f32(36, 18), done=i32(2))  # W = 18
    with pytest.raises(RuntimeError, match="multiple"):
        select(top_ids=i64(7, 2 * W))
    with pytest.raises(RuntimeError, match="candidates"):
        select(top_ids=i64(B, W))
    with pytest.raises(RuntimeError, match="stop tokens"):
        select(stop_ids=i64(R, 9))
    with pytest.raises(RuntimeError, match="CUDA"):  # well-formed: the device check comes first
        select()

    def reorder(**kw):
        a = dict(kv_pointers=i64(2, B, 2, 3), parents=i32(B), context_lens=i32(B), prompt_lens=i32(B), tokens=i64(B), history=i64(B, 16),
                 beam_width=W, num_kv_heads=2, tokens_per_block=64, size_per_token=128, int4_kv_cache=True)
        a.update(kw)
        backend.beam_reorder(**a)

    with pytest.raises(RuntimeError, match="CUDA"):
        reorder()
    for w in (0, 9):
        with pytest.raises(RuntimeError, match="beam_width"):
            reorder(beam_width=w)
    with pytest.raises(RuntimeError, match="multiple"):
        reorder(kv_pointers=i64(2, 6, 2, 3))


def test_runner_constructor_rejects_bad_beam_arguments():
    from qserve_b200.decode import DecodeRunner

    cases = [(dict(beam_width=9), "beam_width"), (dict(beam_width=3, batch=8), "multiple"), (dict(beam_width=2, generate=True), "generate"),
             (dict(beam_width=2, verify_len=2), "verify_len"), (dict(beam_width=2, max_new_tokens=0), "max_new_tokens"),
             (dict(beam_width=2, prompt_tokens=0), "prompt_tokens"), (dict(beam_width=2, fused=False), "fused"),
             (dict(beam_width=2, max_new_tokens=8000), "positions")]
    for kw, msg in cases:
        args = dict(model="tiny", batch=8, ctx=200, max_new_tokens=16, prompt_tokens=1600)
        args.update(kw)
        with pytest.raises(RuntimeError, match=msg):
            DecodeRunner(**args)
