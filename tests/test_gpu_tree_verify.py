"""GPU: verification of tree-structured drafts over the paged INT4 / INT8 KV cache (qs_apply_bias_rope_update_kv_cache_tree,
qs_tree_decode_attention, qs_tree_accept_greedy, qs_kv_cache_compact).

Bars, as for the chain verify (test_gpu_multi_token_attention.py): |out - exact| <= 3e-3 * max(1, max|exact|) against the float64 oracle
(oracle/tree.py) over the pages the kernels wrote, and, against sequential decoding, a per-token error of at most 1.5x the decode kernel's
error on that token plus 2.5e-4 (half an fp16 ulp at |x| < 1: both kernels round their result to fp16 once).  The first bar is not a bound
of the decode kernel itself: on random KV8 pages (values up to 0.1 * 255) single_query_attention exceeds it on some tokens, with the very
error the tree kernel has there.  So the oracle-parity tests hold a token that misses the first bar to the second one.  Page slots at or beyond
P_b + n_b hold NaN scales, so a read of a slot the op must not touch shows up as NaN.
"""
import numpy as np
import pytest
import torch

from oracle import kv
from oracle import prefix as oprefix
from oracle import tree as ot
from tests.test_gpu_multi_token_attention import DRAFT, PREFIX, Case, _bar, _check
from tests.util import GpuPool, kv_pointer_table, np_of

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128


def mask_of(parents):
    m = [0] * len(parents)
    for i, p in enumerate(parents):
        if p >= 0:
            m[i] = m[p] | (1 << p)
    return m


def tree(shape, n=16, seed=0):
    """Ancestor words of one draft tree of the named shape (n nodes where the shape allows)."""
    if shape == "chain":
        return mask_of([i - 1 for i in range(n)])
    if shape == "star":
        return mask_of([-1] + [0] * (n - 1))
    if shape == "binary":
        return mask_of([-1] + [(i - 1) // 2 for i in range(1, 15)])
    if shape == "medusa":  # 1 + 3 + 3 x 3: three candidates for the next token, three for the one after each
        return mask_of([-1, 0, 0, 0] + [1 + (i - 4) // 3 for i in range(4, 13)])
    rng = np.random.default_rng(seed)
    return mask_of([-1] + [int(rng.integers(0, i)) for i in range(1, n)])


class TreeCase(Case):
    """Case with the nodes of per-sequence draft trees: masks[b] holds the ancestor words of sequence b's nodes."""

    def __init__(self, dev, P, masks, hq, hkv, bits, seed, n_blocks=None):
        self.mask_h = np.concatenate([np.asarray(m, np.int64) for m in masks]).astype(np.int32) if masks else np.zeros(0, np.int32)
        self.mask_d = torch.from_numpy(self.mask_h).to(dev)
        super().__init__(dev, P, [len(m) for m in masks], hq, hkv, bits, seed, n_blocks)

    def append(self):
        from qserve_b200 import backend
        backend.apply_bias_rope_update_kv_cache_at(self.qkv, self.lens_d, self.pad, self.prefix_d, self.table, self.hq, self.hkv, self.max_n, 64,
                                                   self.spt, D, ROPE, 8192, True, self.bits == 4, True, tree_mask=self.mask_d)

    def attend(self, **kw):
        return super().attend(tree_mask=self.mask_d, **kw)

    def exact(self, softmax_scale=None):
        kg, vg = self.host_pools()
        return ot.tree_decode_attention(np_of(self.q), np_of(self.k), np_of(self.v), self.cu, self.P, self.mask_h, kg, vg, self.bt, softmax_scale)


def _decode_along_root_path(c, b, node):
    """single_query_attention steps along the root path of node `node` of sequence b on a copy of the pages before the append: returns the
    last step's output [Hq, D] (the decode step of that node) and the copies of the pages the steps wrote."""
    from qserve_b200 import backend
    dev = c.qkv.device
    hq, hkv = c.hq, c.hkv
    path = ot.root_path(c.mask_h[c.cu[b]: c.cu[b + 1]], node)
    gk, gv = GpuPool(c.kp, dev), GpuPool(c.vp, dev)  # the host pools still hold the pages before the append
    table = kv_pointer_table(gk, gv, c.bt[b: b + 1], dev)
    raw = torch.from_numpy(c.raw).to(dev)
    P = c.P[b]
    for k, nd in enumerate(path):  # decode step k at position P + k = P + depth(nd)
        row = int(c.cu[b]) + nd
        q, kk, vv = (t.reshape(1, -1, D) for t in raw[row: row + 1].split([hq * D, hkv * D, hkv * D], dim=-1))
        lens = torch.tensor([P + k + 1], dtype=torch.int32, device=dev)
        dec = backend.single_query_attention(q, kk, vv, table, lens, None, 8192, 64, c.spt, P + k + 1, D, ROPE, True, c.bits == 4, True)
    torch.cuda.synchronize()
    return np_of(dec)[0].astype(np.float64), gk, gv


def _check_tree(c, out, exact):
    """The oracle bar, or for a token that misses it, no further from the truth than 1.5x the decode kernel on that token + 2.5e-4."""
    got = np_of(out).astype(np.float64)
    assert np.isfinite(got).all()
    err = np.abs(got - exact).reshape(len(exact), -1).max(axis=1)
    for t in np.nonzero(err > _bar(exact))[0]:
        b = int(np.searchsorted(c.cu, t, side="right") - 1)
        dec, _, _ = _decode_along_root_path(c, b, int(t - c.cu[b]))
        err_dec = np.abs(dec - exact[t]).max()
        assert err[t] <= 1.5 * err_dec + 2.5e-4, (int(t), err[t], err_dec, _bar(exact))


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. a chain mask is the chain verify, bit for bit (pages, rotated q / k and attention output)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("hq,hkv", [(32, 8), (8, 8), (4, 1)])
def test_chain_mask_is_bitwise_the_chain_verify(dev, bits, hq, hkv):
    seed = 70 + bits + hq
    chain = Case(dev, PREFIX, DRAFT, hq, hkv, bits, seed=seed)
    tc = TreeCase(dev, PREFIX, [tree("chain", n) for n in DRAFT], hq, hkv, bits, seed=seed)
    o_chain, o_tree = chain.attend(), tc.attend()
    torch.cuda.synchronize()
    assert torch.equal(chain.qkv, tc.qkv)
    assert torch.equal(chain.gk.t, tc.gk.t) and torch.equal(chain.gv.t, tc.gv.t)
    assert torch.equal(o_chain, o_tree)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. parity with the float64 oracle: tree shapes x head layouts, prefixes on both sides of a page boundary, KV4 / KV8
# ---------------------------------------------------------------------------------------------------------------------------------
SHAPES = ["chain", "star", "binary", "medusa", "random"]


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("hq,hkv", [(1, 1), (4, 1), (8, 2), (32, 8), (64, 64)])
@pytest.mark.parametrize("shape", SHAPES)
def test_matches_oracle(dev, shape, hq, hkv, bits):
    P = [0, 63, 64, 65]
    masks = [tree(shape, 16, seed=b) for b in range(len(P))]
    if shape == "random":  # ragged: 16, 9, 1 and 5 nodes
        masks = [tree("random", n, seed=b) for b, n in enumerate([16, 9, 1, 5])]
    c = TreeCase(dev, P, masks, hq, hkv, bits, seed=hq * 10 + hkv + bits + len(shape))
    out = c.attend()
    torch.cuda.synchronize()
    assert out.shape == c.q.shape and out.dtype == torch.half
    _check_tree(c, out, c.exact())


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. every node equals sequential decoding along its root path; compacting that path gives the decode steps' bytes
# ---------------------------------------------------------------------------------------------------------------------------------
def _slot_bytes(pool_np, nkv, bits, bt_row, positions):
    p = kv.PagePool(pool_np.shape[0], nkv, D, bits)
    p.data[:] = pool_np
    return [(p.codes()[bt_row[t // 64], :, t % 64].copy(), p.scales()[bt_row[t // 64], :, t % 64].copy(), p.zeros()[bt_row[t // 64], :, t % 64].copy())
            for t in positions]


@pytest.mark.parametrize("bits", [4, 8])
def test_every_node_equals_sequential_decode(dev, bits):
    from qserve_b200 import backend
    hq, hkv = 32, 8
    P = [1, 63, 1000, 130]
    masks = [tree("medusa"), tree("binary"), tree("random", 16, seed=5), tree("star", 6)]
    c = TreeCase(dev, P, masks, hq, hkv, bits, seed=80 + bits)
    new = c.attend()
    torch.cuda.synchronize()
    exact = c.exact()
    got = np_of(new).astype(np.float64)
    assert np.isfinite(got).all()
    err_new = np.abs(got - exact).reshape(len(exact), -1).max(axis=1)
    tree_k, tree_v = c.gk.download(), c.gv.download()
    for b, m in enumerate(masks):
        n = len(m)
        for node in range(n):
            row = int(c.cu[b]) + node
            dec, gk, gv = _decode_along_root_path(c, b, node)
            err_dec = np.abs(dec - exact[row]).max()
            assert err_new[row] <= 1.5 * err_dec + 2.5e-4, (b, node, err_new[row], err_dec)
            if any((m[j] >> node) & 1 for j in range(n)):
                continue  # not a leaf: its path is a prefix of a leaf's
            # compact the leaf's root path on a copy of the tree pages: slots P .. P + len - 1 must be the decode steps' bytes
            path = ot.root_path(m, node)
            ck, cv = GpuPool(c.kp, dev), GpuPool(c.vp, dev)
            ck.t.copy_(torch.from_numpy(tree_k)); cv.t.copy_(torch.from_numpy(tree_v))
            B = len(P)
            path_d = torch.full((B, 16), -1, dtype=torch.int32, device=dev)
            path_d[:, 0] = 0
            path_d[b, : len(path)] = torch.tensor(path, dtype=torch.int32)
            acc = torch.ones(B, dtype=torch.int32, device=dev)
            acc[b] = len(path)
            backend.kv_cache_compact(kv_pointer_table(ck, cv, c.bt, dev), c.prefix_d, path_d, acc, hkv, 64, c.spt, bits == 4)
            torch.cuda.synchronize()
            pos = range(P[b] + len(path))
            for got_pool, want_pool in ((ck, gk), (cv, gv)):
                g_ = _slot_bytes(got_pool.download(), hkv, bits, c.bt[b], pos)
                w_ = _slot_bytes(want_pool.download(), hkv, bits, c.bt[b], pos)
                for t, (x, y) in enumerate(zip(g_, w_)):
                    assert all(np.array_equal(u, v) for u, v in zip(x, y)), (b, node, t)


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. greedy acceptance against the Python reference
# ---------------------------------------------------------------------------------------------------------------------------------
def _accept(dev, draft, mask, target):
    from qserve_b200 import backend
    t = lambda a, dt: torch.tensor(np.asarray(a), dtype=dt, device=dev)
    acc, path, bonus = backend.tree_accept_greedy(t(draft, torch.int64), t(mask, torch.int32), t(target, torch.int64))
    torch.cuda.synchronize()
    want = ot.tree_accept_greedy(np.asarray(draft), np.asarray(mask, np.int32), np.asarray(target))
    assert np.array_equal(np_of(acc), want[0]) and np.array_equal(np_of(path), want[1]) and np.array_equal(np_of(bonus), want[2])
    return want


def test_acceptance_cases(dev):
    m = tree("medusa")  # nodes 1..3 children of 0; 4..6 of 1, 7..9 of 2, 10..12 of 3
    draft = [7, 20, 21, 22, 30, 31, 32, 33, 34, 33, 36, 37, 38]
    tgt_none = [99] + [0] * 12                      # no child matches
    tgt_full = [22, 0, 0, 38] + [5] * 9              # 0 -> 3 -> 12, bonus 5
    tgt_dup = [21, 0, 33, 0] + [6] * 9               # node 2's children 7 and 9 both carry 33: node 7 wins
    acc, path, bonus = _accept(dev, [draft] * 3, [m] * 3, [tgt_none, tgt_full, tgt_dup])
    assert acc.tolist() == [1, 3, 3] and bonus.tolist() == [99, 5, 6]
    assert path[1, :3].tolist() == [0, 3, 12] and path[2, :3].tolist() == [0, 2, 7]
    # ragged: a 4-node chain padded with -1 drafts to 13 chained nodes accepts all of its nodes and none of the padding
    acc, path, bonus = _accept(dev, [[1, 2, 3, 4] + [-1] * 9], [tree("chain", 13)], [[2, 3, 4, 9] + [0] * 9])
    assert acc.tolist() == [4] and bonus.tolist() == [9]


def test_acceptance_random(dev):
    """64 random trees over a 3-token vocabulary (many matches and duplicate siblings), ragged node counts padded with -1."""
    rng = np.random.default_rng(3)
    B, n = 64, 16
    draft = rng.integers(0, 3, (B, n))
    mask = np.zeros((B, n), np.int64)
    for b in range(B):
        nb = int(rng.integers(1, n + 1))
        mask[b, :nb] = tree("random", nb, seed=b)
        draft[b, nb:] = -1
    target = rng.integers(0, 3, (B, n))
    acc, _, _ = _accept(dev, draft, mask, target)
    assert acc.max() > 3  # the cases reach some depth


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. compaction: expected bytes, nothing else touched, 3-D and 4-D page tables
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
def test_compaction(dev, bits):
    from qserve_b200 import backend
    rng = np.random.default_rng(11 + bits)
    L, hkv, nb = 3, 4, 3
    P = [62, 0, 100, 50]
    B = len(P)
    paths = [[0, 2, 3], [0, 5, 9, 12], [0], list(range(16))]  # overlapping moves across a page (62: 64 -> 63, 65 -> 64); identity
    path_h = np.full((B, 16), -1, np.int32)
    for b, p in enumerate(paths):
        path_h[b, : len(p)] = p
    acc_h = np.array([len(p) for p in paths], np.int32)
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    pools = [[kv.PagePool(B * nb + 1, hkv, D, bits, rng) for _ in range(2)] for _ in range(L)]
    gpools = [[GpuPool(p, dev) for p in lp] for lp in pools]
    table = torch.stack([kv_pointer_table(gk, gv, bt, dev) for gk, gv in gpools]).contiguous()  # [L, B, 2, nb]
    spt = hkv * D * bits // 8
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    # 3-D form: layer 1 only
    backend.kv_cache_compact(table[1].contiguous(), t(np.array(P, np.int32)), t(path_h), t(acc_h), hkv, 64, spt, bits == 4)
    torch.cuda.synchronize()
    ot.kv_compact(pools[1][0], pools[1][1], bt, P, path_h, acc_h)
    for li in range(L):
        for g, p in zip(gpools[li], pools[li]):
            assert np.array_equal(g.download(), p.data), li
    # 4-D form: every layer in one launch
    backend.kv_cache_compact(table, t(np.array(P, np.int32)), t(path_h), t(acc_h), hkv, 64, spt, bits == 4)
    torch.cuda.synchronize()
    for li in range(L):
        ot.kv_compact(pools[li][0], pools[li][1], bt, P, path_h, acc_h)
        for g, p in zip(gpools[li], pools[li]):
            assert np.array_equal(g.download(), p.data), li


# ---------------------------------------------------------------------------------------------------------------------------------
# 6. context splits and column parts; determinism, graph replay and workspace reuse
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,shapes,hq,hkv", [
    ([8000], ["random"], 32, 8),                       # one sequence: many splits, 4 x 16 columns per KV head
    ([7999, 0, 64], ["binary", "star", "medusa"], 8, 8),  # G = 1: splits, ragged trees
])
def test_splits_and_column_parts(dev, P, shapes, hq, hkv):
    c = TreeCase(dev, P, [tree(s, 16, seed=i) for i, s in enumerate(shapes)], hq, hkv, 4, seed=sum(P))
    out = c.attend()
    torch.cuda.synchronize()
    _check_tree(c, out, c.exact())


def test_deterministic_graph_and_workspace_reuse(dev):
    from qserve_b200 import backend
    a = TreeCase(dev, [7999], [tree("random", 16, seed=1)], 32, 8, 4, seed=21)
    a.attend()
    c = TreeCase(dev, [65, 1000, 0, 300], [tree("medusa"), tree("binary"), tree("star", 4), tree("chain", 2)], 32, 8, 4, seed=22)
    pristine = torch.from_numpy(c.raw).to(dev)
    o1, o2 = c.attend(), c.attend()
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    _check_tree(c, o1, c.exact())
    B = 4
    draft = torch.randint(0, 3, (B, 13), device=dev)
    target = torch.randint(0, 3, (B, 13), device=dev)
    mask2 = torch.zeros((B, 13), dtype=torch.int32, device=dev)
    mask2[:, :13] = torch.tensor(tree("medusa"), dtype=torch.int32)
    acc_e, path_e, bonus_e = (x.clone() for x in backend.tree_accept_greedy(draft, mask2, target))
    pages_k, pages_v = c.gk.t.clone(), c.gv.t.clone()
    acc, path, bonus = torch.zeros_like(acc_e), torch.zeros_like(path_e), torch.zeros_like(bonus_e)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c.qkv.copy_(pristine)
        c.append()
        c.attend()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.qkv.copy_(pristine)
        c.append()
        og = c.attend()
        backend.tree_accept_greedy(draft, mask2, target, acc, path, bonus)
    c.qkv.zero_()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, o1)
    assert torch.equal(c.gk.t, pages_k) and torch.equal(c.gv.t, pages_v)
    assert torch.equal(acc, acc_e) and torch.equal(path, path_e) and torch.equal(bonus, bonus_e)


# ---------------------------------------------------------------------------------------------------------------------------------
# 7. full size: Llama-3-8B heads, 64 x (1024 prefix + a 16-node tree), KV4, against a float32 torch reference on the device
# ---------------------------------------------------------------------------------------------------------------------------------
def test_llama3_8b_full_size(dev):
    B, P, n, hq, hkv = 64, 1024, 16, 32, 8
    masks = [tree("random", n, seed=b) for b in range(B)]
    c = TreeCase(dev, [P] * B, masks, hq, hkv, 4, seed=3)
    out = c.attend()
    kg, vg = c.host_pools()
    G = hq // hkv
    worst = 0.0
    for b in range(B):
        allowed = torch.zeros((n, P + n - 1), dtype=torch.bool, device=dev)
        allowed[:, :P] = True
        for i in range(n):
            for j in ot.ancestors(masks[b][i], i):
                allowed[i, P + j] = True
        s = slice(int(c.cu[b]), int(c.cu[b + 1]))
        kc = torch.from_numpy(oprefix.dequant_prefix(kg, c.bt[b], P + n - 1)).to(dev).float().repeat_interleave(G, dim=1)
        vc = torch.from_numpy(oprefix.dequant_prefix(vg, c.bt[b], P + n - 1)).to(dev).float().repeat_interleave(G, dim=1)
        q = c.q[s].float()
        ko, vo = c.k[s].float().repeat_interleave(G, dim=1), c.v[s].float().repeat_interleave(G, dim=1)
        sc = torch.einsum("ihd,thd->hit", q, kc).masked_fill(~allowed[None], float("-inf"))
        own = (q * ko).sum(-1).transpose(0, 1)[..., None]
        p = torch.softmax(torch.cat([sc, own], dim=-1) * D ** -0.5, dim=-1)
        ref = torch.einsum("hit,thd->ihd", p[..., :-1], vc) + p[..., -1].transpose(0, 1)[..., None] * vo
        worst = max(worst, float((out[s].float() - ref).abs().max()))
    assert worst <= 3e-3, worst


# ---------------------------------------------------------------------------------------------------------------------------------
# 8. argument errors
# ---------------------------------------------------------------------------------------------------------------------------------
def test_argument_errors(dev):
    from qserve_b200 import backend
    c = TreeCase(dev, [70, 3], [tree("star", 5), tree("chain", 2)], 4, 2, 4, seed=1)
    base = dict(q=c.q, k=c.k, v=c.v, cu_seqlens=c.cu_d, max_seqlen=5, prefix_lens=c.prefix_d, max_prefix_len=70, kv_pointers=c.table,
                tokens_per_block=64, size_per_token=c.spt, int4_kv_cache=True, tree_mask=c.mask_d)
    backend.multi_token_decode_attention(**base)  # valid

    def bad(fn=backend.multi_token_decode_attention, kw=base, **over):
        with pytest.raises(RuntimeError):
            fn(**{**kw, **over})

    bad(tree_mask=c.mask_d.long())
    bad(tree_mask=c.mask_d[:-1].clone())
    bad(tree_mask=c.mask_d.cpu())
    bad(tree_mask=torch.stack([c.mask_d, c.mask_d], 1)[:, 0])  # not contiguous
    bad(max_seqlen=17)
    bad(max_prefix_len=c.n_blocks * 64)
    ap = dict(qkv=c.qkv, seq_lens=c.lens_d, padding_offset=c.pad, start_pos=c.prefix_d, kv_pointers=c.table, head_num=4, kv_head_num=2, seq_len=5,
              tokens_per_block=64, size_per_token=c.spt, rotary_embedding_dim=D, rotary_embedding_base=ROPE, rotary_embedding_max_positions=8192,
              neox_rotary_style=True, int4_kv_cache=True, kv_cache_with_zeros=True, tree_mask=c.mask_d)
    bad(backend.apply_bias_rope_update_kv_cache_at, ap, tree_mask=c.mask_d.long())
    bad(backend.apply_bias_rope_update_kv_cache_at, ap, seq_len=17)
    d = torch.zeros((2, 5), dtype=torch.int64, device=dev)
    m = torch.zeros((2, 5), dtype=torch.int32, device=dev)
    acc = dict(draft_tokens=d, tree_mask=m, target_tokens=d)
    backend.tree_accept_greedy(**acc)  # valid
    bad(backend.tree_accept_greedy, acc, draft_tokens=d.int())
    bad(backend.tree_accept_greedy, acc, tree_mask=m.long())
    bad(backend.tree_accept_greedy, acc, target_tokens=d[:, :4].contiguous())
    bad(backend.tree_accept_greedy, acc, draft_tokens=torch.zeros((2, 17), dtype=torch.int64, device=dev), tree_mask=torch.zeros((2, 17), dtype=torch.int32,
        device=dev), target_tokens=torch.zeros((2, 17), dtype=torch.int64, device=dev))
    bad(backend.tree_accept_greedy, acc, draft_tokens=d.cpu())
    bad(backend.tree_accept_greedy, acc, accept_len=torch.zeros(3, dtype=torch.int32, device=dev))
    path = torch.zeros((2, 5), dtype=torch.int32, device=dev)
    alen = torch.ones(2, dtype=torch.int32, device=dev)
    cp = dict(kv_pointers=c.table, start_pos=c.prefix_d, path=path, accept_len=alen, num_kv_heads=2, tokens_per_block=64, size_per_token=c.spt,
              int4_kv_cache=True)
    backend.kv_cache_compact(**cp)  # valid
    bad(backend.kv_cache_compact, cp, path=path.long())
    bad(backend.kv_cache_compact, cp, path=torch.zeros((3, 5), dtype=torch.int32, device=dev))
    bad(backend.kv_cache_compact, cp, accept_len=alen.long())
    bad(backend.kv_cache_compact, cp, start_pos=c.prefix_d.cpu())
    bad(backend.kv_cache_compact, cp, size_per_token=c.spt * 2)
    bad(backend.kv_cache_compact, cp, kv_pointers=c.table[:, 0].contiguous())
    bad(backend.kv_cache_compact, cp, path=torch.zeros((2, 17), dtype=torch.int32, device=dev))


# ---------------------------------------------------------------------------------------------------------------------------------
# 9. the decode runner: one tree step against sequential decoding
# ---------------------------------------------------------------------------------------------------------------------------------
def _cache_slots(runner, pools, upto):
    """(codes, scales / zeros) of cache positions 0 .. upto - 1 of every sequence of one layer's pool."""
    B, bps, cb = runner.batch, runner.blocks_per_seq, 64 * runner.size_per_token
    p = pools.view(B, bps, -1)
    codes = p[:, :, :cb].reshape(B, bps, runner.Hkv, 64, -1).permute(0, 2, 1, 3, 4).reshape(B, runner.Hkv, bps * 64, -1)[:, :, :upto]
    meta = p[:, :, cb:].reshape(B, bps, 2, runner.Hkv, 64, 2).permute(0, 2, 3, 1, 4, 5).reshape(B, 2, runner.Hkv, bps * 64, 2)[:, :, :, :upto]
    return codes, meta


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
def test_runner_tree_step_equals_sequential_decode(dev, precision):
    """The tree holds the first two greedy tokens of sequential decoding on one branch (nodes 0 -> 2 -> 3), a wrong third token below them
    (node 4) and wrong siblings (nodes 1, 5).  The step must accept 3 nodes and return the third greedy token as the bonus.  Layer 0's K / V
    depend only on the tokens, so its compacted slots are byte-identical to sequential decoding; deeper layers see attention outputs that
    differ from the decode kernel's in fp32 summation order, so for every layer the compacted slots are checked to be the accepted nodes'
    bytes, and the next decode step at ctx + accept_len against sequential decoding's logits."""
    from qserve_b200.decode import DecodeRunner
    B, ctx, n = 5, 130, 6
    seq = DecodeRunner("tiny", precision, batch=B, ctx=ctx, device=dev, seed=3, verify_len=n)
    tre = DecodeRunner("tiny", precision, batch=B, ctx=ctx, device=dev, seed=3, verify_len=n)
    V = seq.cfg.vocab
    root = (torch.arange(B, device=dev) * 37 + 11) % V
    with torch.no_grad():
        greedy, tok = [], root
        for i in range(3):  # decode steps at ctx, ctx + 1, ctx + 2
            seq.context_lens.fill_(ctx + 1 + i)
            seq.max_seq_len = ctx + 1 + i
            tok = seq._forward_fused(tok.contiguous())
            greedy.append(tok.clone())
        seq_slots = [_cache_slots(seq, pool, ctx + 3) for pool in seq.kpools + seq.vpools]
        seq.context_lens.fill_(ctx + 4)
        seq.max_seq_len = ctx + 4
        want_next = seq._forward_fused(greedy[2].contiguous(), return_logits=True).float()
        g1, g2, g3 = greedy
        parents = [-1, 0, 0, 2, 3, 0]
        tokens = torch.stack([root, (g1 + 1) % V, g1, g2, (g3 + 1) % V, (g1 + 2) % V], dim=1)
        mask = torch.tensor(mask_of(parents), dtype=torch.int32, device=dev).repeat(B, 1)
        target = tre.verify_forward(tokens, tree_mask=mask)
        before = [pool.clone() for pool in tre.kpools + tre.vpools]
        acc, path, bonus = tre.accept_and_compact(tokens, mask, target)
        acc, path, bonus = acc.clone(), path.clone(), bonus.clone()
    torch.cuda.synchronize()
    assert acc.tolist() == [3] * B and path[:, :3].tolist() == [[0, 2, 3]] * B and torch.equal(bonus, g3)
    L = tre.L
    for li, (pool, old) in enumerate(zip(tre.kpools + tre.vpools, before)):
        got_c, got_m = _cache_slots(tre, pool, ctx + 3)
        old_c, old_m = _cache_slots(tre, old, ctx + 6)
        src = [ctx + j for j in (0, 2, 3)]
        assert torch.equal(got_c[:, :, :ctx], old_c[:, :, :ctx]) and torch.equal(got_m[:, :, :, :ctx], old_m[:, :, :, :ctx]), li
        assert torch.equal(got_c[:, :, ctx:], old_c[:, :, src]) and torch.equal(got_m[:, :, :, ctx:], old_m[:, :, :, src]), li
        if li % L == 0:  # layer 0 (K and V)
            assert torch.equal(got_c, seq_slots[li][0]) and torch.equal(got_m, seq_slots[li][1]), li
    with torch.no_grad():
        tre.context_lens.fill_(ctx + 4)
        tre.max_seq_len = ctx + 4
        got_next = tre._forward_fused(bonus.contiguous(), return_logits=True).float()
    torch.cuda.synchronize()
    assert torch.isfinite(got_next).all()
    assert float((got_next - want_next).abs().max()) <= 1e-2 * float(want_next.abs().max())
    # the captured tree step replays bitwise what the eager step computes (every draft slot is rewritten by the step's own append)
    with torch.no_grad():
        e_target = tre.verify_forward(tokens, tree_mask=mask).clone()
        e_acc, e_path, e_bonus = (x.clone() for x in tre.accept_and_compact(tokens, mask, e_target))
    e_pages = [pool.clone() for pool in tre.kpools + tre.vpools]
    tre.v_tokens_in[:, :n].copy_(tokens)
    tre.v_tree_mask[:, :n].copy_(mask)
    tre.capture_verify(n, tree=True)
    tre.v_tokens_out.zero_(); tre.v_accept_len.zero_(); tre.v_path.zero_(); tre.v_bonus.zero_()
    tre.verify_step(n, tree=True)
    torch.cuda.synchronize()
    assert torch.equal(tre.v_tokens_out[:, :n], e_target)
    assert torch.equal(tre.v_accept_len, e_acc) and torch.equal(tre.v_path[: B * n].view(B, n), e_path) and torch.equal(tre.v_bonus, e_bonus)
    assert all(torch.equal(p, e) for p, e in zip(tre.kpools + tre.vpools, e_pages))
