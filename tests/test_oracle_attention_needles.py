"""The needle inputs of test_gpu_attention_needles.py have the power to see one wrong read (float64 oracle, no GPU).

For the needle inputs the GPU tests use, each corruption below is applied to the cache the way a kernel bug would read it, and the exact
output must move by at least 10x the bar (oracle/needles.py `exact`) at the affected heads:
  * token t read as t + 1 (t - 1 at the end of the cache);
  * t's V scale, V zero or K scale taken from the neighbouring slot (lane ^ 1 of the 32-token slice);
  * the zero points of t's page rotated by one slot;
  * the split that holds t dropped;
  * a non-ancestor tree node unmasked;
  * the last prefix slot dropped.
"""
import numpy as np
import pytest

from oracle import needles as nd
from oracle.kv import TOKENS_PER_PAGE, PagePool

D = 128
DECODE = [  # (B, Hq, Hkv, lens): the configurations of the GPU decode sweep
    (2, 64, 64, [2048, 1985]),
    (2, 32, 8, [1087, 96]),
    (2, 64, 4, [575, 33]),
]


def _copy(p):
    q = PagePool(p.data.shape[0], p.Hkv, p.D, p.bits)
    q.data[:] = p.data
    return q


def _loc(bt_row, t):
    return int(bt_row[t // TOKENS_PER_PAGE]), t % TOKENS_PER_PAGE


def _moved(base, corrupt):
    """Largest |change| / bar over the elements of the affected heads."""
    (o, bar), (o2, _) = base, corrupt
    return float((np.abs(o2 - o) / bar).max())


def _decode_corruptions(c, b, hk, t, L=None):
    """(name, kpool, vpool, drop) for the corruptions of cached position t of (b, hk); L - 1 cached tokens."""
    L = L or c.lens[b]
    row = c.bt[b]
    pg, sl = _loc(row, t)
    nb = t + 1 if t + 1 < L - 1 else t - 1
    pn, sn = _loc(row, nb)
    ps, ss = _loc(row, t ^ 1 if (t ^ 1) < L - 1 else nb)
    out = []
    kp, vp = _copy(c.kp), _copy(c.vp)
    for src, dst in ((c.kp, kp), (c.vp, vp)):
        dst.codes()[pg, hk, sl] = src.codes()[pn, hk, sn]
        dst.scales()[pg, hk, sl] = src.scales()[pn, hk, sn]
        dst.zeros()[pg, hk, sl] = src.zeros()[pn, hk, sn]
    out.append(("token read as its neighbour", kp, vp, None))
    for name, which, field in (("V scale of lane ^ 1", "v", "scales"), ("V zero of lane ^ 1", "v", "zeros"), ("K scale of lane ^ 1", "k", "scales")):
        kp, vp = _copy(c.kp), _copy(c.vp)
        p = vp if which == "v" else kp
        getattr(p, field)()[pg, hk, sl] = getattr(p, field)()[ps, hk, ss]
        out.append((name, kp, vp, None))
    kp, vp = _copy(c.kp), _copy(c.vp)
    n_in_page = min(TOKENS_PER_PAGE, L - 1 - (t // TOKENS_PER_PAGE) * TOKENS_PER_PAGE)
    if n_in_page > 1:
        vp.zeros()[pg, hk, :n_in_page] = np.roll(c.vp.zeros()[pg, hk, :n_in_page], -1)
        out.append(("page zeros rotated", kp, vp, None))
    return out


def _positions(L, nsplit):
    """Needle positions that sit on every kind of boundary: slices, warps, pages, splits and the ends of the cache."""
    pos = {0, 1, 31, 32, 33, 63, 64, 65, 127, 128, L // 2, L - 3, L - 2}
    n_pages = (L - 1 + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE
    pps = (n_pages + nsplit - 1) // nsplit
    for s in range(1, nsplit):
        pos |= {s * pps * TOKENS_PER_PAGE - 1, s * pps * TOKENS_PER_PAGE}
    return sorted(t for t in pos if 0 <= t < L - 1)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode_needles_see_one_wrong_read(bits, B, Hq, Hkv, lens):
    nsplit = nd.decode_splits(B, Hq, Hkv, max(lens), sms=132)
    for t in _positions(lens[0], nsplit):
        c = nd.DecodeCase(7 + t, B, Hq, Hkv, lens, bits, {(0, 0): t})
        base = c.exact_head(0, 0)
        for name, kp, vp, drop in _decode_corruptions(c, 0, 0, t):
            assert _moved(base, c.exact_head(0, 0, kp, vp)) >= 10, (name, t)
        if nsplit > 1:
            s = nd.split_of(t, lens[0] - 1, nsplit)
            pps = -(-((lens[0] - 1 + 63) // 64) // nsplit)
            drop = range(s * pps * 64, min((s + 1) * pps * 64, lens[0] - 1))
            assert _moved(base, c.exact_head(0, 0, drop=drop)) >= 10, ("split dropped", t)


@pytest.mark.parametrize("bits", [4, 8])
def test_decode_two_needles_see_a_wrong_merge(bits):
    """Two needles a logit gap of ln 3 apart in different splits: dropping either split, or losing the gap (a merge weight without its
    max rescale), moves the 3:1 mix by O(|v|).  These are checks beyond the single-needle corruptions above, and the margin is smaller:
    in a mix the logit-error term of the bar grows with sum_t p_t |v_t - exact|, so at KV4 (the larger needle K scale) the bar is about
    0.08 and the moves are 8.4x to 25x it (KV8: 19x to 58x).  Still an order of magnitude above any error the kernels showed (err / bar
    at most 0.27 on the GPU two-needle test)."""
    B, Hq, Hkv, lens = 2, 32, 8, [1087, 96]
    c = nd.DecodeCase(3, B, Hq, Hkv, lens, bits, {(0, 0): 10}, second={(0, 0): (1000, np.log(3))})
    base = c.exact_head(0, 0)
    assert _moved(base, c.exact_head(0, 0, drop=range(0, 64))) >= 5
    assert _moved(base, c.exact_head(0, 0, drop=range(960, 1024))) >= 5
    equal = nd.DecodeCase(3, B, Hq, Hkv, lens, bits, {(0, 0): 10}, second={(0, 0): (1000, 0.0)})
    assert _moved(base, equal.exact_head(0, 0)) >= 5


def _rows(c, qkv):
    T = qkv.shape[0]
    G, hkv = c.G, c.hkv
    q = qkv[:, : c.hq * D].reshape(T, c.hq, D)
    k = qkv[:, c.hq * D: (c.hq + hkv) * D].reshape(T, hkv, D)
    v = qkv[:, (c.hq + hkv) * D:].reshape(T, hkv, D)
    return q, k, v


@pytest.mark.parametrize("bits", [4, 8])
def test_verify_needles_see_one_wrong_read(bits):
    c = nd.ChunkCase(5, "chain", [1000, 63], [16, 16], 32, 8, bits, {(0, 0): 999, (0, 1): 1003, (1, 2): 31})
    qkv, kp, vp = c.append()
    q, k, v = _rows(c, qkv)
    for (b, hk), t in c.needles.items():
        base = c.exact_head(b, hk, q, k, v, kp, vp)
        j = max(t - c.P[b], 0)
        drop = {i: [t] for i in range(c.N[b])}
        moved = np.abs(c.exact_head(b, hk, q, k, v, kp, vp, drop=drop)[0] - base[0]) / base[1]
        assert moved.reshape(c.N[b], -1)[j + 1:].max(axis=1).min() >= 10, (b, hk, t)
        # a causal mask one position late lets row j - 1 see draft needle j
        if t >= c.P[b] and j > 0:
            late = c.exact_head(b, hk, q, k, v, kp, vp, extra={j - 1: [t]})
            assert _moved(base, late) >= 10


@pytest.mark.parametrize("bits", [4, 8])
def test_tree_needle_on_a_non_ancestor_is_visible_if_unmasked(bits):
    from tests.test_gpu_tree_verify import tree
    masks = [tree("binary"), tree("random", 16, seed=4), tree("medusa")]
    from oracle.tree import ancestors
    for b, node in ((0, 4), (1, 9), (2, 2)):
        c = nd.ChunkCase(11 + node, "tree", [300, 64, 1], [len(m) for m in masks], 8, 2, bits, {(b, 0): [300, 64, 1][b] + node}, masks=masks,
                         logit=16.0)
        qkv, kp, vp = c.append()
        q, k, v = _rows(c, qkv)
        base = c.exact_head(b, 0, q, k, v, kp, vp)
        others = [i for i in range(len(masks[b])) if i != node and node not in ancestors(masks[b][i], i)]
        for i in others:
            opened = c.exact_head(b, 0, q, k, v, kp, vp, extra={i: [c.P[b] + node]})
            moved = np.abs(opened[0] - base[0]) / base[1]
            assert moved.reshape(len(masks[b]), -1)[i].max() >= 10, (b, node, i)


@pytest.mark.parametrize("bits", [4, 8])
def test_prefix_needle_on_the_last_slot_is_missed_if_dropped(bits):
    c = nd.ChunkCase(9, "prefix", [191, 128, 1], [66, 64, 130], 16, 8, bits, {(0, 0): 190, (1, 3): 127, (2, 5): 0})
    qkv, kp, vp = c.append()
    q, k, v = _rows(c, qkv)
    for (b, hk), t in c.needles.items():
        base = c.exact_head(b, hk, q, k, v, kp, vp)
        dropped = c.exact_head(b, hk, q, k, v, kp, vp, drop={i: [t] for i in range(c.N[b])})
        moved = np.abs(dropped[0] - base[0]) / base[1]
        assert moved.reshape(c.N[b], -1).max(axis=1).min() >= 10, (b, hk, t)


@pytest.mark.parametrize("kind,P,N,hq,hkv", [
    ("chain", [700, 1, 64], [2, 1, 2], 32, 8),
    ("chain", [1000, 63], [16, 16], 32, 8),
    ("prefix", [191, 128, 1], [66, 64, 130], 16, 8),
])
@pytest.mark.parametrize("bits", [4, 8])
def test_chunk_needles_see_one_wrong_read(bits, kind, P, N, hq, hkv):
    """The decode corruptions (neighbour token, lane ^ 1 scale / zero, page zeros) on prefix needles of the verify and prefix inputs."""
    b = 0
    for t in (0, 31, 32, 63, 64, P[b] // 2, P[b] - 2):
        c = nd.ChunkCase(21 + t, kind, P, N, hq, hkv, bits, {(b, 1): t})
        qkv, kp, vp = c.append()
        q, k, v = _rows(c, qkv)
        base = c.exact_head(b, 1, q, k, v, kp, vp)
        for name, kp2, vp2, _ in _decode_corruptions(c, b, 1, t, L=P[b] + 1):
            for src, dst in ((kp, kp2), (vp, vp2)):  # the appended rows stay as the append left them
                for i in range(N[b]):
                    pg, sl = _loc(c.bt[b], P[b] + i)
                    dst.codes()[pg, :, sl], dst.scales()[pg, :, sl], dst.zeros()[pg, :, sl] = (src.codes()[pg, :, sl], src.scales()[pg, :, sl],
                                                                                               src.zeros()[pg, :, sl])
            assert _moved(base, c.exact_head(b, 1, q, k, v, kp2, vp2)) >= 10, (name, t)
