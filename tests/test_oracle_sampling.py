"""CPU checks of the sampling oracle (oracle/sampling.py): Philox known answers, the warpers against Hugging Face's, the max(tau_p, tau_k)
identity, and losslessness of the sampled tree acceptance rule, integrated over u in closed form."""
import itertools

import numpy as np
import pytest

from oracle import sampling as os_
from oracle import tree as ot


def test_philox_known_answers():
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        assert tuple(int(v) for v in os_.philox4x32_10(ctr, key)) == want


def test_uniform_is_exact_in_float32_and_counter_layout():
    u = os_.uniform(0x123456789ABCDEF, np.arange(1000) + (5 << 32), np.arange(1000) % 7, 3)
    assert np.array_equal(u, u.astype(np.float32).astype(np.float64))
    assert u.min() >= 0 and u.max() <= 1 - 2.0 ** -24
    # counter (lo(off), hi(off), row, j), key (lo(seed), hi(seed))
    x0 = os_.philox4x32_10((7, 5, 2, 3), (0x89ABCDEF, 0x01234567))[0]
    assert os_.uniform(0x0123456789ABCDEF, (5 << 32) | 7, 2, 3) == float(int(x0) >> 8) * 2.0 ** -24


def _tie_free_row(rng, V, scale):
    while True:
        x = (rng.standard_normal(V) * scale).astype(np.float16)
        if np.unique(x).size == V:
            return x


@pytest.mark.parametrize("T", [0.3, 0.7, 1.0, 1.5])
def test_warp_matches_transformers_warpers(T):
    tr = pytest.importorskip("transformers")
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(int(T * 10))
    for top_k, top_p in itertools.product([-1, 1, 2, 7, 50, 300], [1.0, 0.95, 0.8, 0.5, 0.1]):
        x = _tie_free_row(rng, 256, 2.0)
        w, kept, info = os_.warp(x, T, top_k, top_p)
        if info["top_p_margin"] < 1e-9:
            continue  # a crossing within float64 rounding of HF's cumsum
        z = torch.from_numpy((x.astype(np.float32) / np.float32(T)).astype(np.float64))[None]
        if top_p < 1:
            z = tr.TopPLogitsWarper(top_p=float(np.float32(top_p)))(None, z)
        if top_k > 0:
            z = tr.TopKLogitsWarper(top_k=top_k)(None, z)
        assert np.array_equal(kept, np.isfinite(z[0].numpy())), (T, top_k, top_p)


def test_threshold_identity_with_ties():
    """TopP then TopK (each with the tie-independent rule) keeps exactly {z >= max(tau_p, tau_k)}, on rows with heavy ties."""
    rng = np.random.default_rng(1)
    for _ in range(300):
        V = int(rng.integers(8, 64))
        x = (rng.integers(-4, 4, V) * 0.5).astype(np.float16)
        T, top_k, top_p = float(rng.choice([0.5, 1.0, 2.0])), int(rng.choice([-1, 1, 2, 3, 5, 100])), float(rng.choice([1.0, 0.9, 0.6, 0.3]))
        _, kept, _ = os_.warp(x, T, top_k, top_p)
        assert np.array_equal(kept, os_.kept_topp_then_topk(x, T, top_k, top_p))
        zs = x.astype(np.float32)[kept]
        assert kept[np.isin(x, x[kept])].all()  # tie groups are kept or dropped together
        assert zs.size >= 1


def test_warp_special_rows():
    x = np.array([1, np.nan, 3, 3, -np.inf, 2, 0, 0], np.float16)
    assert os_.warp(x, 0.0, -1, 1.0)[2]["greedy"] and os_.warp(x, 0.0, -1, 1.0)[0][1] == 1  # NaN counts as the maximum
    assert os_.warp(x, 1.0, -1, 1e-9)[0].argmax() == 1
    w, kept, _ = os_.warp(x, 1.0, -1, 1.0)
    assert w[1] == 0 and w[4] == 0 and kept[[0, 2, 3, 5, 6, 7]].all()
    w, _, _ = os_.warp(x, 1.0, 1, 1.0)  # top_k = 1 keeps the tied maxima
    assert np.array_equal(np.nonzero(w)[0], [2, 3]) and w[2] == w[3] == 1
    w, _, _ = os_.warp(x, 1.0, 3, 1.0)  # the third largest is 2: kept with both 3s
    assert np.array_equal(np.nonzero(w)[0], [2, 3, 5])
    only = np.full(8, -np.inf, np.float16)
    only[5] = -3
    assert np.array_equal(np.nonzero(os_.warp(only, 0.7, -1, 0.5)[0])[0], [5])
    none = np.full(8, -np.inf, np.float16)
    assert os_.warp(none, 1.0, -1, 1.0)[2]["greedy"] and os_.warp(none, 1.0, -1, 1.0)[0][0] == 1
    t, _ = os_.sample(np.array([0, 1.0, 0, 1.0]), 0.5)
    assert t == 3 and os_.sample(np.array([0, 1.0, 0, 1.0]), 0.49)[0] == 1 and os_.sample(np.array([0, 1.0, 0, 1.0]), 0.0)[0] == 1


# ------------------------------------------------------------------------------------------------
# losslessness: the acceptance probability of child c given that it is tried is P(u q_c(d) < p(d)) = min(1, p(d) / q_c(d))
# ------------------------------------------------------------------------------------------------
def _accept(p, q, d):
    return min(1.0, p[d] / q[d])


def _siblings(p, drafts, qs):
    """Distribution of the first emitted token for a star: children tried in order, bonus from the final residual."""
    out, reach = np.zeros_like(p), 1.0
    for d, q in zip(drafts, qs):
        a = _accept(p, q, d)
        out[d] += reach * a
        reach *= 1.0 - a
        p = os_.residual(p, q)
    return out + reach * p


def _targets(rng, V, settings):
    for T, k, tp in settings:
        for _ in range(3):
            x = (rng.standard_normal(V) * 1.5).astype(np.float16)
            w = os_.warp(x, T, k, tp)[0]
            yield w / w.sum()


SETTINGS = [(1.0, -1, 1.0), (0.7, 3, 0.9), (1.3, -1, 0.8), (0.0, -1, 1.0)]


@pytest.mark.parametrize("V", [4, 5])
@pytest.mark.parametrize("k", [2, 3])
def test_lossless_iid_star(V, k):
    rng = np.random.default_rng(V * 10 + k)
    for p in _targets(rng, V, SETTINGS):
        q = rng.dirichlet(np.ones(V) * 0.7)
        dist = np.zeros(V)
        for drafts in itertools.product(range(V), repeat=k):
            dist += np.prod(q[list(drafts)]) * _siblings(p, drafts, [q] * k)
        assert np.abs(dist - p).max() < 1e-12


@pytest.mark.parametrize("V", [4, 5])
@pytest.mark.parametrize("k", [2, 3])
def test_lossless_without_replacement_star(V, k):
    rng = np.random.default_rng(100 + V * 10 + k)
    for p in _targets(rng, V, SETTINGS):
        q0 = rng.dirichlet(np.ones(V))
        dist = np.zeros(V)
        for drafts in itertools.permutations(range(V), k):
            qs, prob, q = [], 1.0, q0.copy()
            for d in drafts:
                qs.append(q)
                prob *= q[d]
                q = q.copy()
                q[d] = 0
                q /= q.sum()
            dist += prob * _siblings(p, drafts, qs)
        assert np.abs(dist - p).max() < 1e-12


@pytest.mark.parametrize("V", [4, 5])
def test_lossless_deterministic_candidates(V):
    rng = np.random.default_rng(200 + V)
    for p in _targets(rng, V, SETTINGS):
        for k in (1, 2, 3):
            for drafts in itertools.permutations(range(V), k):
                qs = [np.eye(V)[d] for d in drafts]
                assert np.abs(_siblings(p, drafts, qs) - p).max() < 1e-12


@pytest.mark.parametrize("V", [4, 5])
def test_lossless_chain_joint_of_two_tokens(V):
    """Depth-2 chain: node 1 ~ q1, node 2 ~ q2(. | node 1); target p1 and p2(. | t1).  If node 1 is rejected, the second token comes from
    the next step, exactly p2(. | t1).  The joint of the first two emitted tokens must be p1(t1) p2(t2 | t1)."""
    rng = np.random.default_rng(300 + V)
    for T, k, tp in SETTINGS:
        rows = (rng.standard_normal((V + 1, V)) * 1.5).astype(np.float16)
        w = [os_.warp(r, T, k, tp)[0] for r in rows]
        p1, p2 = w[V] / w[V].sum(), np.array([x / x.sum() for x in w[:V]])
        q1 = rng.dirichlet(np.ones(V))
        q2 = rng.dirichlet(np.ones(V), size=V)
        joint = np.zeros((V, V))
        for d1, d2 in itertools.product(range(V), repeat=2):
            prob = q1[d1] * q2[d1, d2]
            a1 = _accept(p1, q1, d1)
            a2 = _accept(p2[d1], q2[d1], d2)
            joint[d1, d2] += prob * a1 * a2
            joint[d1] += prob * a1 * (1 - a2) * os_.residual(p2[d1], q2[d1])
            joint += prob * (1 - a1) * os_.residual(p1, q1)[:, None] * p2
        assert np.abs(joint - p1[:, None] * p2).max() < 1e-12


def _mask(parents):
    m = [0] * len(parents)
    for i, pp in enumerate(parents):
        m[i] = (m[pp] | (1 << pp)) if pp >= 0 else 0
    return np.array(m, np.int32)


def test_oracle_walk_uses_the_rule():
    """The oracle's walk accepts child c iff u_c q_c(d) < p(d); greedy rows reduce to tree_accept_greedy of the argmax targets."""
    rng = np.random.default_rng(5)
    parents = [-1, 0, 0, 1, 1, 2, 3]
    mask = np.tile(_mask(parents), (6, 1))
    V, n = 16, len(parents)
    logits = (rng.standard_normal((6, n, V)) * 2).astype(np.float16)
    draft = rng.integers(-1, V, (6, n))
    q = rng.dirichlet(np.ones(V), size=(6, n))
    alen, path, bonus, _ = os_.tree_accept_sampling(draft, mask, logits, 0.0, -1, 1.0, 9, np.arange(6), q)
    target = logits.astype(np.float32).argmax(-1)
    want = ot.tree_accept_greedy(draft, mask, target)
    assert np.array_equal(alen, want[0]) and np.array_equal(path, want[1]) and np.array_equal(bonus, want[2])
    # q_c = the warped target of c's parent and p(d) > 0 for every draft: the first child is always accepted
    draft = rng.integers(0, V, (6, n))
    qp = np.zeros((6, n, V))
    for b in range(6):
        for c in range(1, n):
            w = os_.warp(logits[b, parents[c]], 1.0, -1, 1.0)[0]
            qp[b, c] = w / w.sum()
    alen, path, _, _ = os_.tree_accept_sampling(draft, mask, logits, 1.0, -1, 1.0, 3, np.arange(6), qp)
    assert (alen == 4).all() and (path[:, :4] == [0, 1, 3, 6]).all()
