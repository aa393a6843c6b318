"""CPU: the oracle of tree-structured draft verification (oracle/tree.py) against the chain oracle it generalises (oracle/multi_token.py):
a chain mask is the multi-token verify, every node of a random tree is the chain verify of its root path once that path has been
compacted, and the greedy acceptance walks a hand-worked tree as stated."""
import numpy as np
import pytest

from oracle import kv
from oracle import multi_token as om
from oracle import prefix as op
from oracle import tree as ot

ROPE = 500000.0
D = 128
PREFIX = [0, 1, 63, 64, 65, 200]
NODES = [5, 16, 1, 2, 3, 16]


def _setup(rng, hq, hkv, bits, P, N):
    B = len(P)
    nb = (max(p + n for p, n in zip(P, N)) + 63) // 64
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    kp, vp = kv.PagePool(B * nb + 1, hkv, D, bits, rng), kv.PagePool(B * nb + 1, hkv, D, bits, rng)
    cu = np.concatenate([[0], np.cumsum(N)]).astype(np.int64)
    qkv = rng.standard_normal((sum(N), (hq + 2 * hkv) * D)).astype(np.float16)
    return bt, kp, vp, cu, qkv


def _copy(pool):
    p = kv.PagePool(pool.data.shape[0], pool.Hkv, pool.D, pool.bits)
    p.data[:] = pool.data
    return p


def _split(rot, hq, hkv):
    T = rot.shape[0]
    return rot[:, : hq * D].reshape(T, hq, D), rot[:, hq * D: (hq + hkv) * D].reshape(T, hkv, D), rot[:, (hq + hkv) * D:].reshape(T, hkv, D)


def random_tree_mask(rng, n):
    """Node i > 0 gets a random earlier parent; its word is the parent's word plus the parent's bit."""
    m = np.zeros(n, np.int64)
    for i in range(1, n):
        p = int(rng.integers(0, i))
        m[i] = m[p] | (1 << p)
    return m.astype(np.int32)


@pytest.mark.parametrize("bits", [4, 8])
def test_chain_mask_is_the_multi_token_verify(rng, bits):
    hq, hkv = 8, 2
    bt, kp, vp, cu, qkv = _setup(rng, hq, hkv, bits, PREFIX, NODES)
    kp2, vp2 = _copy(kp), _copy(vp)
    T, mx = sum(NODES), max(NODES)
    pad = kv.compute_padding_offsets(cu, mx, T)
    mask = np.concatenate([ot.chain_mask(n) for n in NODES])
    rot_c = op.prefill_rope_append_at(qkv.copy(), NODES, pad, PREFIX, kp, vp, bt, hq, hkv, mx, ROPE, 8192)
    rot_t = ot.tree_rope_append(qkv.copy(), NODES, pad, PREFIX, mask, kp2, vp2, bt, hq, hkv, mx, ROPE, 8192)
    assert np.array_equal(rot_c, rot_t) and np.array_equal(kp.data, kp2.data) and np.array_equal(vp.data, vp2.data)
    want = om.multi_token_decode_attention(*_split(rot_c, hq, hkv), cu, PREFIX, kp, vp, bt)
    got = ot.tree_decode_attention(*_split(rot_t, hq, hkv), cu, PREFIX, mask, kp2, vp2, bt)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("bits", [4, 8])
def test_every_node_is_the_chain_verify_of_its_compacted_root_path(rng, bits):
    hq, hkv = 4, 1
    bt, kp, vp, cu, qkv = _setup(rng, hq, hkv, bits, PREFIX, NODES)
    T, mx = sum(NODES), max(NODES)
    mask = np.concatenate([random_tree_mask(rng, n) for n in NODES])
    rot = ot.tree_rope_append(qkv.copy(), NODES, kv.compute_padding_offsets(cu, mx, T), PREFIX, mask, kp, vp, bt, hq, hkv, mx, ROPE, 8192)
    q, k, v = _split(rot, hq, hkv)
    got = ot.tree_decode_attention(q, k, v, cu, PREFIX, mask, kp, vp, bt)
    for b, (P, n) in enumerate(zip(PREFIX, NODES)):
        for i in range(n):
            path = ot.root_path(mask[cu[b]: cu[b + 1]], i)
            kc, vc = _copy(kp), _copy(vp)
            full = np.full((len(PREFIX), max(NODES)), -1, np.int32)
            full[b, : len(path)] = path
            alen = np.zeros(len(PREFIX), np.int32)
            alen[b] = len(path)
            ot.kv_compact(kc, vc, bt, PREFIX, full, alen)
            rows = [int(cu[b]) + j for j in path]
            # the chain verify of the path, with the nodes' rotated rows (node path[k] was rotated at depth k = its chain position)
            want = om.multi_token_decode_attention(q[rows], k[rows], v[rows], [0, len(path)], [P], kc, vc, bt[b: b + 1])
            assert np.allclose(got[cu[b] + i], want[-1], rtol=0, atol=1e-12), (b, i, path)


def test_compaction_moves_overlapping_slots_across_a_page():
    """path [0, 2, 3] behind P = 62: slot 64 -> 63 (across the page boundary) and 65 -> 64, read before written."""
    rng = np.random.default_rng(7)
    kp, vp = kv.PagePool(4, 2, D, 4, rng), kv.PagePool(4, 2, D, 4, rng)
    bt = np.array([[1, 2]])
    before = kp.data.copy()
    ot.kv_compact(kp, vp, bt, [62], np.array([[0, 2, 3, -1]], np.int32), np.array([3], np.int32))
    c0 = kv.PagePool(4, 2, D, 4)
    c0.data[:] = before
    assert np.array_equal(kp.codes()[1, :, 63], c0.codes()[2, :, 0]) and np.array_equal(kp.codes()[2, :, 0], c0.codes()[2, :, 1])
    assert np.array_equal(kp.scales()[2, :, 0], c0.scales()[2, :, 1]) and np.array_equal(kp.zeros()[1, :, 63], c0.zeros()[2, :, 0])
    assert np.array_equal(kp.codes()[1, :, :63], c0.codes()[1, :, :63]) and np.array_equal(kp.codes()[2, :, 2:], c0.codes()[2, :, 2:])


def test_greedy_acceptance_hand_worked():
    """Tree (node: parent, draft):  0 root;  1: 0, 'a';  2: 0, 'b';  3: 2, 'c';  4: 2, 'c' (duplicate sibling);  5: 3, 'd';  6: 1, 'e'.
    Targets after each node: 0 -> 'b', 2 -> 'c', 3 -> 'x' (no child 'x'): accepted path 0, 2, 3 (node 3 beats its duplicate 4), bonus 'x'."""
    a, b_, c, d, e, x = 10, 11, 12, 13, 14, 99
    parents = [-1, 0, 0, 2, 2, 3, 1]
    mask = np.zeros(7, np.int64)
    for i in range(1, 7):
        mask[i] = mask[parents[i]] | (1 << parents[i])
    draft = np.array([[5, a, b_, c, c, d, e]])
    target = np.array([[b_, 0, c, x, 0, 0, 0]])
    alen, path, bonus = ot.tree_accept_greedy(draft, mask[None].astype(np.int32), target)
    assert alen.tolist() == [3] and path.tolist() == [[0, 2, 3, -1, -1, -1, -1]] and bonus.tolist() == [x]
    # no child matches: only the root, bonus = the target after the root
    alen, path, bonus = ot.tree_accept_greedy(draft, mask[None].astype(np.int32), np.array([[x, 0, 0, 0, 0, 0, 0]]))
    assert alen.tolist() == [1] and path[0, 0] == 0 and bonus.tolist() == [x]
    # the full depth: 0 -> 2 -> 3 -> 5
    alen, path, bonus = ot.tree_accept_greedy(draft, mask[None].astype(np.int32), np.array([[b_, 0, c, d, 0, 7, 0]]))
    assert alen.tolist() == [4] and path[0, :4].tolist() == [0, 2, 3, 5] and bonus.tolist() == [7]
