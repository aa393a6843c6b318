"""CPU tests of the prompt-lookup oracle (tests/ngram_oracle.py): every drafting rule on hand-built histories, the commit's truncations, and
the CPU speculative loop, which must emit exactly the sequential greedy tokens."""
import numpy as np
import pytest

from tests import ngram_oracle as ng


def propose(h, n, n_min=1, n_max=4, branches=1, L=None):
    return ng.propose_row(h, len(h) if L is None else L, n, n_min, n_max, branches)


def test_no_match_gives_root_and_padding():
    toks, mask = propose([1, 2, 3, 4, 5], 4)
    assert toks == [5, -1, -1, -1] and mask == [0, 1, 1, 1]


def test_longest_match_beats_more_recent_shorter():
    # key ... 7 8 9; "7 8 9" at j = 2 (m = 3), "8 9" alone at j = 6 (m = 2, more recent)
    h = [7, 8, 9, 100, 5, 8, 9, 200, 7, 8, 9]
    assert ng.candidates(h, len(h), 1, 4, 2) == [2, 6]
    toks, mask = propose(h, 3)
    assert toks == [9, 100, 5] and mask == [0, 1, 3]


def test_most_recent_wins_at_equal_length():
    h = [3, 4, 10, 3, 4, 20, 3, 4]
    toks, _ = propose(h, 2)
    assert toks == [4, 20]
    assert ng.candidates(h, len(h), 1, 4, 8) == [4, 1]


def test_overlapping_periodic_match():
    h = [5, 5, 5, 5, 5]
    # j = 3 overlaps the key window; m(3) = 4 (capped by n_max), m(2) = 3, ...
    assert [ng.match_len(h, 5, j, 4) for j in range(4)] == [1, 2, 3, 4]
    toks, mask = propose(h, 4)
    assert toks == [5, 5, -1, -1] and mask == [0, 1, 1, 1]  # the continuation of j = 3 is cut at L - 1
    h = [1, 2, 1, 2, 1, 2]
    toks, mask = propose(h, 5)
    assert toks == [2, 1, 2, -1, -1] and mask == [0, 1, 3, 1, 1]


def test_continuation_cut_at_last_token():
    h = [9, 1, 2, 9]
    toks, mask = propose(h, 8)
    assert toks == [9, 1, 2, 9] + [-1] * 4 and mask == [0, 1, 3, 7] + [1] * 4


def test_n_min_threshold():
    h = [1, 2, 50, 3, 2]  # only a one-token match
    assert propose(h, 3, n_min=1)[0] == [2, 50, 3]
    assert propose(h, 3, n_min=2)[0] == [2, -1, -1]


def test_negative_ids_never_match():
    h = [-1, 7, 1, -1, 7]
    # the key's last id matches at j = 1; the windows would extend into -1 == -1, which does not count
    assert ng.match_len(h, 5, 1, 4) == 1
    assert propose(h, 3, n_min=2)[0] == [7, -1, -1]
    h = [-1, 4, -1]
    assert propose(h, 3)[0] == [-1, -1, -1]  # a root < 0 matches nothing


@pytest.mark.parametrize("L", [0, 1, 2])
def test_short_histories(L):
    h = [4, 4, 0, 0]
    toks, mask = propose(h, 4, L=L)
    root = -1 if L == 0 else 4
    if L == 2:  # j = 0 matches the root: continuation h[1] only
        assert toks == [4, 4, -1, -1] and mask == [0, 1, 1, 1]
    else:
        assert toks == [root, -1, -1, -1] and mask == [0, 1, 1, 1]


def test_two_branches_share_a_prefix():
    h = [1, 2, 3, 4, 9, 1, 2, 3, 5, 9, 1, 2]
    # the key "9 1 2" ends at j = 6 (m = 3) and "1 2" at j = 1 (m = 2)
    assert ng.candidates(h, len(h), 1, 4, 2) == [6, 1]
    toks, mask = propose(h, 6, branches=2)
    # j = 6 drafts 3 5 9 1 2 and spends the budget; j = 1's 3 would be shared, its 4 has no node left
    assert toks == [2, 3, 5, 9, 1, 2] and mask == [0, 1, 3, 7, 15, 31]
    toks, mask = propose(h, 6, branches=2, n_max=2)
    assert toks[:2] == [2, 3]
    toks, mask = ng.propose_row(h, len(h), 5, 1, 4, 2)
    assert toks == [2, 3, 5, 9, 1]
    toks, mask = ng.propose_row([1, 2, 3, 4, 9, 1, 2, 3, 5, 9, 1, 2], 12, 4, 1, 4, 2)
    assert toks == [2, 3, 5, 9]


def test_branches_share_then_split():
    h = [8, 1, 2, 8, 1, 3, 8]
    toks, mask = propose(h, 5, branches=2)
    # j = 3 (most recent "8"): 1 3 8; j = 0: 1 (shared) 2 -> a sibling of 3
    assert toks == [8, 1, 3, 8, 2] and mask == [0, 1, 3, 7, 3]


def test_node_budget_exhausted_mid_branch():
    h = [8, 1, 2, 8, 4, 5, 8]
    toks, mask = propose(h, 4, branches=2)
    # j = 3: 4 5 8 fills the budget (3 nodes); j = 0 gets nothing
    assert toks == [8, 4, 5, 8] and mask == [0, 1, 3, 7]
    toks, mask = propose(h, 5, branches=2)
    # one node left: j = 0's first token 1 becomes a child of the root, its second token 2 does not fit
    assert toks == [8, 4, 5, 8, 1] and mask == [0, 1, 3, 7, 1]


def _check_tree(toks, mask):
    n = len(toks)
    for i in range(1, n):
        if toks[i] == -1 and mask[i] == 1:
            continue
        anc = [j for j in range(n) if (mask[i] >> j) & 1]
        assert anc and max(anc) < i and anc[0] == 0  # topological, rooted
        parent = max(anc)
        assert mask[i] == mask[parent] | (1 << parent)
        assert bin(mask[i]).count("1") == bin(mask[parent]).count("1") + 1  # depth = popcount


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_are_topological(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        L = int(rng.integers(0, 60))
        h = list(rng.integers(-1, 4, L))
        n = int(rng.integers(1, 17))
        toks, mask = propose(h, n, n_min=int(rng.integers(1, 3)), n_max=int(rng.integers(2, 9)), branches=int(rng.integers(1, 9)))
        assert len(toks) == n and mask[0] == 0
        _check_tree(toks, mask)
        chain, cm = propose(h, n, branches=1)
        drafted = [i for i in range(1, n) if not (chain[i] == -1 and cm[i] == 1)]
        assert all(cm[i] == (1 << i) - 1 for i in drafted)


def _commit1(app_draft, path, acc, bonus, hist, L, P, budget, eos, fin=0):
    out = ng.spec_commit(np.array([app_draft]), np.array([path]), [acc], [bonus], np.array([hist]), [L], [P], [budget], [eos], [fin])
    return out[0][0].tolist(), int(out[1][0]), int(out[2][0]), out[3][0], out[4][0], out[5][0]


def test_commit_appends_path_and_bonus():
    h = [5, 6, 7, -1, -1, -1, -1]
    hist, L, fin, sp, cl, root = _commit1([7, 1, 2, 3], [0, 2, 3, -1], 3, 9, h, 3, 2, 10, -1)
    assert hist == [5, 6, 7, 2, 3, 9, -1] and L == 6 and fin == 0 and sp == 5 and cl == 6 and root == 9


def test_commit_eos_inside_block():
    h = [5, 6, 7] + [-1] * 5
    hist, L, fin, sp, _, root = _commit1([7, 1, 2, 3], [0, 1, 2, 3], 4, 9, h, 3, 2, 10, eos=2)
    assert hist[:6] == [5, 6, 7, 1, 2, -1] and L == 5 and fin == 1 and sp == 4 and root == 2


def test_commit_budget_inside_block():
    h = [5, 6, 7] + [-1] * 5
    hist, L, fin, _, _, root = _commit1([7, 1, 2, 3], [0, 1, 2, 3], 4, 9, h, 3, 2, 3, eos=9)  # generated 1, room 2: eos (bonus) cut off
    assert hist[:6] == [5, 6, 7, 1, 2, -1] and L == 5 and fin == 1 and root == 2
    hist, L, fin, _, _, root = _commit1([7, 1], [0, -1], 1, 4, h, 3, 3, 0, -1)  # no room: nothing appended, finished
    assert L == 3 and fin == 1 and root == 7


def test_commit_finished_rows_unchanged():
    h = [5, 6, 7, -1]
    hist, L, fin, sp, cl, root = _commit1([7, 1], [0, 1], 2, 9, h, 3, 2, 10, -1, fin=1)
    assert hist == h and L == 3 and fin == 1 and sp is None and cl is None and root is None


def test_commit_drops_columns_past_history():
    h = [5, 6, 7]
    hist, L, fin, sp, _, root = _commit1([7, 1, 2], [0, 1, 2], 3, 9, h, 2, 0, 100, -1)
    assert hist == [5, 6, 1] and L == 5 and sp == 4 and root == 9


def _toy_next(vocab, seed):
    """A deterministic toy target: the next token depends on the last two tokens."""
    rng = np.random.default_rng(seed)
    table = rng.integers(0, vocab, (vocab + 1, vocab + 1))
    return lambda seq: int(table[seq[-2] if len(seq) > 1 else vocab, seq[-1]])


def _sequential(prompt, f, T):
    seq = list(prompt)
    for _ in range(T):
        seq.append(f(seq))
    return seq[len(prompt):]


@pytest.mark.parametrize("n,branches", [(1, 1), (4, 1), (8, 1), (8, 2), (16, 4)])
@pytest.mark.parametrize("planted", [False, True])
def test_speculative_loop_emits_greedy_tokens(n, branches, planted):
    for seed in range(4):
        vocab = 1000 if planted else 12  # a small vocabulary makes many (mostly wrong) drafts; a large one keeps the output aperiodic
        f = _toy_next(vocab, seed)
        rng = np.random.default_rng(100 + seed)
        prompt = [int(x) for x in rng.integers(0, vocab, 20)]
        T = 24
        want = _sequential(prompt, f, T)
        if planted:  # the toy target reads the last two tokens: after "... a b" + want + "a b" the continuation is want again
            prompt = prompt + want + prompt[-2:]
            assert _sequential(prompt, f, T) == want
        got, steps = ng.speculative_generate(prompt, f, T, n, branches)
        assert got == want
        if n == 1:
            assert steps == T
        elif planted:
            assert steps <= -(-T // (n - 1)) + 2


def test_speculative_loop_stops_at_eos():
    f = _toy_next(6, 3)
    prompt = [1, 2, 3, 4, 5, 0, 1, 2]
    want = _sequential(prompt, f, 30)
    eos = want[5]
    cut = want[: want.index(eos) + 1]
    for n in (1, 4, 8):
        got, _ = ng.speculative_generate(prompt, f, 30, n, 2, eos=eos)
        assert got == cut
