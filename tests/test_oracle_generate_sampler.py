"""CPU: the generation loop's sampler oracle (tests/generate_sampler_oracle.py) on hand-made cases: the per-node expanded histories of the
tree penalties, the stop-set commit against ngram_oracle.spec_commit, and the history columns of the accepted tokens' log-probabilities."""
import numpy as np

from tests import generate_sampler_oracle as gso
from tests import ngram_oracle as ng
from tests import penalty_logprob_oracle as plo

V = 16


def _one(draft, mask, hist, L, prompt):
    h, pl, sl = gso.expand_histories(np.array([draft]), np.array([mask]), np.array([hist]), [prompt], [L])
    return [list(h[i, : sl[i]]) for i in range(len(draft))], list(pl)


def test_expansion_chain():
    rows, pl = _one([5, 6, 7, 8], [0, 1, 3, 7], [1, 2, 3, 5, -1], 4, 2)
    assert rows == [[1, 2, 3, 5], [1, 2, 3, 5, 6], [1, 2, 3, 5, 6, 7], [1, 2, 3, 5, 6, 7, 8]]
    assert pl == [2] * 4


def test_expansion_star_and_padding():
    # root with three children; node 4 is padding (token -1, mask 1)
    rows, _ = _one([9, 4, 5, 6, -1], [0, 1, 1, 1, 1], [9, 9], 2, 1)
    assert rows == [[9, 9], [9, 9, 4], [9, 9, 5], [9, 9, 6], [9, 9, -1]]


def test_expansion_tree_ancestors_in_index_order():
    # 0 -> 1 -> 2 -> 4, 0 -> 3; the mask's bits below i are the ancestors (bit 0, the root, is in the history already)
    rows, _ = _one([3, 10, 11, 12, 13], [0, 1, 3, 1, 7], [3], 1, 0)
    assert rows == [[3], [3, 10], [3, 10, 11], [3, 12], [3, 10, 11, 13]]


def test_expansion_is_not_clipped_at_the_history_width():
    rows, _ = _one([2, 3, 4], [0, 1, 3], [1, 2], 5, 0)  # seq_lens 5 > H = 2: L = 2
    assert rows == [[1, 2], [1, 2, 3], [1, 2, 3, 4]]


def _logits(rng, B, n):
    return rng.standard_normal((B, n, V)).astype(np.float16)


def test_tree_penalties_repeated_tokens_along_a_path():
    rng = np.random.default_rng(0)
    x = _logits(rng, 1, 4)
    # token 7 occurs on the path twice (nodes 1 and 3) and once in the generated history; token 9 is only on the path
    draft, mask = np.array([[2, 7, 9, 7]]), np.array([[0, 1, 3, 7]])
    hist = np.array([[1, 2, 3, 7, 2]])  # prompt = 3 tokens, generated 7, 2 (the root)
    got = gso.apply_penalties_tree(x, draft, mask, hist, [3], [5], 1.3, 0.25, 0.5)
    f32 = lambda v: np.float32(v)
    for i, (c7, in9) in enumerate([(1, 0), (2, 0), (2, 1), (3, 1)]):
        x7 = f32(x[0, i, 7])
        x7 = f32(x7 / f32(1.3)) if x7 > 0 else f32(x7 * f32(1.3))
        assert got[0, i, 7] == np.float16(f32(f32(x7 - f32(f32(0.5) * f32(c7))) - f32(0.25)))
        if in9:
            x9 = f32(x[0, i, 9])
            x9 = f32(x9 / f32(1.3)) if x9 > 0 else f32(x9 * f32(1.3))
            assert got[0, i, 9] == np.float16(f32(f32(x9 - f32(0.5)) - f32(0.25)))
        else:
            assert got[0, i, 9] == x[0, i, 9]
        assert got[0, i, 5] == x[0, i, 5]  # in neither


def test_tree_penalties_prompt_only_row_and_neutral_row():
    rng = np.random.default_rng(1)
    x = _logits(rng, 2, 3)
    draft, mask = np.array([[4, 1, 6], [4, 1, 6]]), np.array([[0, 1, 3], [0, 1, 3]])
    hist = np.array([[1, 4, 0, 0], [1, 4, 0, 0]])
    got = gso.apply_penalties_tree(x, draft, mask, hist, [2, 2], [2, 2], [1.0, 1.0], [0.5, 0.0], [0.0, 0.0])
    # row 0, prompt only: the root's row sees no output token; node 1 sees token 1 once as output (presence applies to the prompt's 1 too)
    assert np.array_equal(got[0, 0], x[0, 0])
    assert got[0, 1, 1] == np.float16(np.float32(x[0, 1, 1]) - np.float32(0.5))
    assert got[0, 2, 6] == np.float16(np.float32(x[0, 2, 6]) - np.float32(0.5))
    assert got[0, 1, 4] == x[0, 1, 4]  # a prompt token: no presence penalty without repetition
    assert np.array_equal(got[1], x[1])  # neutral row


def test_tree_penalties_root_row_is_apply_penalties():
    rng = np.random.default_rng(2)
    B, n, H = 3, 5, 12
    x = _logits(rng, B, n)
    hist = rng.integers(-1, V, (B, H))
    L = np.array([12, 6, 0])
    pl = np.array([4, 6, 0])
    draft, mask = ng.ngram_propose(hist, L, n, 1, 4, 2)
    got = gso.apply_penalties_tree(x, draft, mask, hist, pl, L, 1.2, 0.3, -0.4)
    want = plo.apply_penalties(x[:, 0], hist, pl, L, 1.2, 0.3, -0.4)
    assert np.array_equal(got[:, 0], want)


def _commit_case(rng, B, n, H):
    draft = rng.integers(0, 12, (B, n))
    acc = rng.integers(1, n + 1, B).astype(np.int32)
    path = np.zeros((B, n), np.int32)
    for b in range(B):
        path[b, 1: acc[b]] = np.sort(rng.choice(np.arange(1, n), acc[b] - 1, replace=False)) if acc[b] > 1 else []
    return (draft, path, acc, rng.integers(0, 12, B), rng.integers(0, 12, (B, H)), rng.integers(H // 2, H, B).astype(np.int32),
            np.full(B, H // 2, np.int32), rng.integers(0, 8, B).astype(np.int32), np.where(rng.random(B) < 0.5, rng.integers(0, 12, B), -1),
            (rng.random(B) < 0.2).astype(np.int32))


def test_stop_commit_with_empty_sets_is_spec_commit():
    rng = np.random.default_rng(3)
    for n in (1, 4, 16):
        draft, path, acc, bonus, hist, L, prompt, budget, eos, fin = _commit_case(rng, 32, n, 40)
        want = ng.spec_commit(draft, path, acc, bonus, hist, L, prompt, budget, eos, fin)
        for S in (0, 3):
            got = gso.spec_commit_stops(draft, path, acc, bonus, hist, L, prompt, budget, eos, np.full((32, S), -1), fin)
            assert all(np.array_equal(np.asarray(a, dtype=object), np.asarray(b, dtype=object)) for a, b in zip(got, want))


def test_stop_commit_hand_cases():
    draft = np.array([[0, 5, 6, 7]] * 4)
    path = np.array([[0, 1, 2, 3]] * 4, np.int32)
    acc = np.array([4, 4, 4, 4], np.int32)
    bonus = np.array([8, 8, 8, 8])
    hist = np.full((4, 10), -1)
    L = np.array([2, 2, 2, 2], np.int32)
    prompt = np.array([2, 2, 2, 2], np.int32)
    budget = np.array([8, 8, 2, 8], np.int32)
    eos = np.array([7, -1, -1, 5])
    stops = np.array([[6, -1], [7, 8], [6, -1], [-1, -1]])
    h, sl, fin, _, _, roots = gso.spec_commit_stops(draft, path, acc, bonus, hist, L, prompt, budget, eos, stops, np.zeros(4, np.int32))
    # row 0: the stop 6 comes before eos 7; row 1: stop 7 first of {7, 8}; row 2: the budget cut (2 tokens) falls before the stop;
    # row 3: eos alone
    assert list(sl) == [4, 5, 4, 3] and list(fin) == [1, 1, 1, 1] and list(roots) == [6, 7, 6, 5]
    assert list(h[0, 2:5]) == [5, 6, -1] and list(h[1, 2:6]) == [5, 6, 7, -1]


def test_logprob_columns_hand_cases():
    draft = np.array([[3, 4, 5, 6], [3, 4, 5, 6], [3, 4, 5, 6]])
    path = np.array([[0, 2, 3, -1], [0, 1, -1, -1], [0, 1, 2, 3]], np.int32)
    acc = np.array([3, 9, 4], np.int32)  # row 1: clamped to n = 4 (path -1 entries clamp to node 0)
    bonus = np.array([10, 11, 12])
    got = gso.accepted_entries(draft, path, acc, bonus, [5, 2, 8], [0, 0, 0], 10)
    assert got[:3] == [(0, 5, 0, 5), (0, 6, 2, 6), (0, 7, 3, 10)]
    assert got[3:7] == [(1, 2, 0, 4), (1, 3, 1, 3), (1, 4, 0, 3), (1, 5, 0, 11)]
    assert got[7:] == [(2, 8, 0, 4), (2, 9, 1, 5)]  # columns >= W = 10 are dropped
    assert gso.accepted_entries(draft, path, acc, bonus, [5, 2, 8], [1, 1, 0], 10) == got[7:]  # finished rows write nothing
