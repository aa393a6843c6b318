"""GPU: shared-prefix decode attention (backend.shared_prefix_decode_attention) against the float64 oracle and the decode kernel.

Rows of a group share the pages 0 .. S - 1 of the group's first row; the op reads them once per group, then every row's own pages from page
S on.  Bars (DESIGN.md 4, the decode bar): max |out - exact| <= 3e-3 * max(1, max |exact|), where `exact` is oracle/kv.decode_attention with
faithful=False over the same quantised cache, and the op is never further from `exact` than 1.5x single_query_attention on the same inputs
(plus 2^-12 * max(1, max |exact|), one fp16 ulp at 4: both kernels round to fp16).  Pages: byte-identical to single_query_attention's; the
shared pages are not written.  Needles (oracle/needles.py): one key in each group's shared region and one in a member's own suffix make
a wrong page read move the output by O(1).  Children's table entries below S point at a NaN-poisoned page: the op reads the shared pages
through the group's first row only.
"""
import numpy as np
import pytest
import torch

from oracle import kv
from oracle import needles as nd
from tests.util import GpuPool, kv_pointer_table, np_of, to_dev

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128
HKV = 2

# (groups, S per group, batch): non-contiguous rows, groups of 1, 2, 3, 4, 5, 8, 16 and 33 rows, and rows in no group
_perm = np.random.default_rng(7).permutation(80).tolist()
_sizes = [1, 2, 3, 4, 5, 8, 16, 33]
_cut = np.cumsum([0] + _sizes).tolist()
MIXED = ([_perm[a:b] for a, b in zip(_cut, _cut[1:])], [1, 16, 0, 1, 16, 1, 16, 1], 80)
LONG = ([[3, 0, 5], [1, 4]], [64, 16], 7)  # S = 64: context splits in the shared pass and in the row pass
CASES = {"mixed": MIXED, "long": LONG}
SUFFIX = [1, 2, 37, 64, 100]  # a member's length is 64 S + suffix: 1 = the own token only, past the shared pages


def _build(seed, G, bits, groups, pages, batch, needles=True):
    """Pools, the true tables, the tables with the children's shared entries poisoned, q / k / v, lengths, and the layout lists."""
    rng = np.random.default_rng(seed)
    hq = G * HKV
    S_of = {r: s for g, s in zip(groups, pages) for r in g}
    lens = []
    for b in range(batch):
        s = S_of.get(b, int(rng.integers(0, 20)))
        lens.append(64 * s + SUFFIX[b % len(SUFFIX)])
    blocks = max((L + 63) // 64 for L in lens)
    n_pages = batch * blocks + 1
    kp, vp = kv.PagePool(n_pages, HKV, D, bits, rng), kv.PagePool(n_pages, HKV, D, bits, rng)
    for p in (kp, vp):  # page 0: NaN scales (what a poisoned table entry points at)
        p.scales()[0] = np.float16(np.nan)
    bt = 1 + np.arange(batch * blocks).reshape(batch, blocks)
    for g, s in zip(groups, pages):
        for r in g[1:]:
            bt[r, :s] = bt[g[0], :s]
    poisoned = bt.copy()
    for g, s in zip(groups, pages):
        for r in g[1:]:
            poisoned[r, :s] = 0
    q = rng.standard_normal((batch, hq, D)).astype(np.float16)
    k = rng.standard_normal((batch, HKV, D)).astype(np.float16)
    v = rng.standard_normal((batch, HKV, D)).astype(np.float16)
    if needles:
        for g, s in zip(groups, pages):
            if s == 0:
                continue
            tgt, own = g[-1], g[0]
            qr = kv.rope_neox(q[tgt], lens[tgt] - 1, ROPE)[:G]  # the query heads of kv head 0 of the group's last member
            t = int(rng.integers(0, 64 * s))
            nd.write_row(kp, bt[own, t // 64], t % 64, 0, nd.needle_key(qr, bits))
            if lens[own] - 1 > 64 * s:  # a needle in the first member's own suffix
                t = int(rng.integers(64 * s, lens[own] - 1))
                qo = kv.rope_neox(q[own], lens[own] - 1, ROPE)[G:2 * G]
                nd.write_row(kp, bt[own, t // 64], t % 64, 1, nd.needle_key(qo, bits))
    return kp, vp, bt, poisoned, q, k, v, lens


class _Dev:
    """Device copies of one case; every call runs on fresh copies of the pools unless `pools` is given."""

    def __init__(self, dev, c, groups, pages, bits):
        self.dev, self.bits = dev, bits
        self.kp, self.vp, self.bt, self.poisoned, q, k, v, self.lens = c
        B, Hq, _ = q.shape
        self.B, self.Hq = B, Hq
        qkv = torch.from_numpy(np.concatenate([q.reshape(B, -1), k.reshape(B, -1), v.reshape(B, -1)], axis=1)).to(dev)
        qd, kd, vd = qkv.split([Hq * D, HKV * D, HKV * D], dim=-1)
        self.q, self.k, self.v = qd.reshape(B, Hq, D), kd.reshape(B, HKV, D), vd.reshape(B, HKV, D)
        self.lens_d = torch.tensor(self.lens, dtype=torch.int32, device=dev)
        from qserve_b200 import backend as ext
        self.layout = ext.shared_prefix_layout(groups, pages, B, device=dev)

    def pools(self):
        return GpuPool(self.kp, self.dev), GpuPool(self.vp, self.dev)

    def args(self):
        return (64, HKV * D * self.bits // 8, max(self.lens), D, ROPE, self.bits == 4, True)

    def shared(self, gk, gv, table="bt", **kw):
        from qserve_b200 import backend as ext
        t = kv_pointer_table(gk, gv, getattr(self, table), self.dev)
        return ext.shared_prefix_decode_attention(self.q, self.k, self.v, t, self.lens_d, self.layout, *self.args(), **kw)

    def decode(self, gk, gv):
        import qserve_backend.fused_attention as fa
        t = kv_pointer_table(gk, gv, self.bt, self.dev)
        return fa.single_query_attention(self.q, self.k, self.v, t, self.lens_d, None, 8192, 64, HKV * D * self.bits // 8, max(self.lens), D,
                                         ROPE, True, self.bits == 4, True)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("case", list(CASES))
def test_shared_prefix_attention(dev, bits, G, case):
    groups, pages, batch = CASES[case]
    c = _build(100 * G + bits + len(case), G, bits, groups, pages, batch)
    d = _Dev(dev, c, groups, pages, bits)
    shared_pages = sorted({int(d.bt[g[0], j]) for g, s in zip(groups, pages) for j in range(s)})
    gk, gv = d.pools()
    before = (gk.t[shared_pages].clone(), gv.t[shared_pages].clone())
    out = np_of(d.shared(gk, gv, table="poisoned")).astype(np.float64)
    torch.cuda.synchronize()
    assert torch.equal(gk.t[shared_pages], before[0]) and torch.equal(gv.t[shared_pages], before[1]), "the op wrote into shared pages"
    dk, dv = d.pools()
    ref = np_of(d.decode(dk, dv)).astype(np.float64)
    assert torch.equal(gk.t, dk.t) and torch.equal(gv.t, dv.t), "pages differ from single_query_attention's"
    # the poisoned children's entries are never read: the same bits as with the true tables
    gk2, gv2 = d.pools()
    assert np.array_equal(np_of(d.shared(gk2, gv2)).view(np.uint16), out.astype(np.float16).view(np.uint16))
    kp2, vp2 = kv.PagePool(d.kp.data.shape[0], HKV, D, bits), kv.PagePool(d.vp.data.shape[0], HKV, D, bits)
    kp2.data[:], vp2.data[:] = d.kp.data, d.vp.data
    exact = kv.decode_attention(c[4], c[5], c[6], kp2, vp2, d.bt, d.lens, ROPE, faithful=False).astype(np.float64)
    scale = max(1.0, float(np.abs(exact).max()))
    assert np.isfinite(out).all()
    err, err_dec = np.abs(out - exact).max(), np.abs(ref - exact).max()
    print(f"\nSHARED-PREFIX {case} G={G} KV{bits}: err {err:.3e}, decode kernel {err_dec:.3e}, scale {scale:.2f}")
    assert err <= 3e-3 * scale, (err, scale)
    assert err <= 1.5 * err_dec + 2.0 ** -12 * scale, (err, err_dec)


@pytest.mark.parametrize("bits", [4, 8])
def test_fused_quant_equals_fp16_then_quant(dev, bits):
    from qserve_b200 import backend as ext
    groups, pages, batch = MIXED
    c = _build(31 + bits, 4, bits, groups, pages, batch)
    d = _Dev(dev, c, groups, pages, bits)
    gk, gv = d.pools()
    out = d.shared(gk, gv).reshape(batch, -1)
    want_q = torch.empty((batch, d.Hq * D), dtype=torch.int8, device=dev)
    want_s = torch.empty(batch, dtype=torch.half, device=dev)
    want_sum = torch.empty(batch, dtype=torch.half, device=dev)
    ext.invoke_quant_fuse_sum(want_q, out, want_sum, want_s)
    for with_sum in (True, False):
        gk, gv = d.pools()
        oq = torch.empty_like(want_q)
        sc = torch.empty_like(want_s)
        sm = torch.empty_like(want_sum) if with_sum else None
        assert d.shared(gk, gv, out_q=oq, out_scale=sc, out_sum=sm) is None
        assert torch.equal(oq, want_q) and torch.equal(sc.view(torch.int16), want_s.view(torch.int16))
        if with_sum:
            assert torch.equal(sm.view(torch.int16), want_sum.view(torch.int16))


def test_equal_members_calls_and_graph_replay_give_equal_bits(dev):
    """Members with equal q / k / v, lengths and own-page contents get equal bits wherever they sit in the group (another column of the
    n8 tile, another column part); two calls and a graph replay give the eager bits."""
    G, bits = 4, 4
    groups, pages, batch = [[0, 2, 5, 6, 7], [1, 3]], [16, 16], 8
    c = list(_build(5, G, bits, groups, pages, batch, needles=False))
    kp, vp, bt, _, q, k, v, lens = c
    twins = [0, 6, 7]  # members 0, 3 and 4 of the first group: columns 0, 12 and 16 (column part 1)
    lens[0] = 64 * pages[0] + 37
    for r in twins[1:]:
        q[r], k[r], v[r], lens[r] = q[0], k[0], v[0], lens[0]
        for j in range(pages[0], (lens[0] + 63) // 64):
            for p in (kp, vp):
                p.data[bt[r, j]] = p.data[bt[0, j]]
    d = _Dev(dev, c, groups, pages, bits)
    gk, gv = d.pools()
    a = d.shared(gk, gv)
    b = d.shared(gk, gv)  # the append rewrites the same bytes; the new token's slot is never read
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for r in twins[1:]:
        assert torch.equal(a[r].view(torch.int16), a[0].view(torch.int16)), f"row {r} differs from its twin row 0"
    from qserve_b200 import backend as ext
    table = kv_pointer_table(gk, gv, d.bt, dev)
    out = torch.empty_like(a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        out.copy_(ext.shared_prefix_decode_attention(d.q, d.k, d.v, table, d.lens_d, d.layout, *d.args()))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out.copy_(ext.shared_prefix_decode_attention(d.q, d.k, d.v, table, d.lens_d, d.layout, *d.args()))
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), a.view(torch.int16))


def test_argument_errors(dev):
    from qserve_b200 import backend as ext
    groups, pages, batch = LONG
    c = _build(3, 2, 4, groups, pages, batch, needles=False)
    d = _Dev(dev, c, groups, pages, 4)
    gk, gv = d.pools()
    table = kv_pointer_table(gk, gv, d.bt, dev)
    with pytest.raises(RuntimeError):
        ext.shared_prefix_decode_attention(d.q, d.k, d.v, table, d.lens_d.long(), d.layout, *d.args())
    with pytest.raises(RuntimeError):
        bad = d.layout._replace(row_pages=d.layout.row_pages[:-1])
        ext.shared_prefix_decode_attention(d.q, d.k, d.v, table, d.lens_d, bad, *d.args())
    with pytest.raises(RuntimeError):  # more shared pages than the page table holds
        bad = d.layout._replace(max_pages=table.size(-1) + 1)
        ext.shared_prefix_decode_attention(d.q, d.k, d.v, table, d.lens_d, bad, *d.args())
