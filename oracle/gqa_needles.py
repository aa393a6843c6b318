"""Oracle: head-tagged needle inputs for the paged-attention kernels at any GQA group size (TEST INFRASTRUCTURE, not product).

The needles of oracle/needles.py give every query head of a KV head the same direction and one shared needle, so all G heads of a group
return the same V and a kernel that mixes up the heads of a group (column c -> (token, head) at an n8-tile or column-part seam, the first
head of a decode head group, the KV head of a query head) is invisible.  Here every COLUMN (query head x row or member) of a KV head has its
own needle:
  * queries: the rotated queries of the columns of one KV head are mutually orthogonal with norm sqrt(128) (at most 128 columns per KV
    head), and the op is fed their `unrotate`d form;
  * visible needles: each column gets its own key (`needle_key` of that column's query alone, logit 14) at its own cache position, on
    the boundaries `boundary_positions` lists (slices, pages, splits, the last cached slot);
  * draft keys (chain / tree verify): the key of row r carries a logit of 14 for its own last column, for the first column of each child
    of r (chain: row r + 1), which sees it, and for the last column of row r - 1, which must not: only a wrong causal limit or ancestor
    word lets it in;
  * prompt kernels: rows span many positions, so each query head of a KV head has its own base direction in the low-frequency RoPE pairs
    (which barely rotate across a chunk), orthogonal across the heads of the KV head.
The oracle and its bar are those of oracle/needles.py (`exact`, `paged_exact`); only the inputs are new.
"""
from __future__ import annotations

import numpy as np

from . import needles as nd
from .kv import TOKENS_PER_PAGE, rope_neox
from .tree import ancestors

D = nd.D
LOGIT = nd.NEEDLE_LOGIT
LOW_FREQ_DIMS = np.r_[48:64, 112:128]  # RoPE pairs (i, i + 64), i >= 48: at rope base 5e5 they turn by < 0.11 rad over 2k positions
# dim 0 of every draft row's V: sets the row's quantisation range, so that its cached (quantised) V differs from the fp16 own V by up to
# half a step (KV4 about 1.5, KV8 about 0.08) -- a column whose causal limit lets in its own cache slot reads that copy
OWN_V_OUTLIER = 40.0


def orthogonal_rows(rng, n: int):
    """n <= 128 mutually orthogonal rows of norm sqrt(D) (float64 [n, D])."""
    assert n <= D, "at most 128 orthogonal columns per KV head"
    Q, _ = np.linalg.qr(rng.standard_normal((D, n)))
    return Q.T * np.sqrt(D)


def boundary_positions(n_cached: int, nsplit: int, count: int, shift: int = 0):
    """`count` distinct cache positions < n_cached: the slice, page, split and end-of-cache boundaries first (as in
    test_oracle_attention_needles._positions), then evenly spread fill.  `shift` rotates the order, so that the KV heads of a sequence put
    their first columns on different boundaries."""
    if n_cached <= 0:
        return []
    L = n_cached + 1
    edges = {0, 1, 31, 32, 33, 63, 64, 65, 127, 128, L // 2, L - 3, L - 2}
    n_pages = (n_cached + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE
    pps = (n_pages + nsplit - 1) // max(nsplit, 1)
    for s in range(1, nsplit):
        edges |= {s * pps * TOKENS_PER_PAGE - 1, s * pps * TOKENS_PER_PAGE}
    first = sorted(t for t in edges if 0 <= t < n_cached)
    if first:
        k = shift % len(first)
        first = first[k:] + first[:k]
    rest = [t for t in np.linspace(0, n_cached - 1, num=min(n_cached, max(count, 1) * 3)).astype(int).tolist() if t not in set(first)]
    out = []
    for t in first + rest + list(range(n_cached)):
        if t not in out:
            out.append(t)
        if len(out) == count:
            break
    return out


def _key(queries, bits, quant=True):
    return nd.needle_key(np.asarray(queries, np.float64).reshape(-1, D), bits, LOGIT, quant=quant)


# ----------------------------------------------------------------------------------------------------------------------------------------
# decode: single_query_attention
# ----------------------------------------------------------------------------------------------------------------------------------------
def decode_case(seed, B, hq, hkv, lens, bits, sms: int = 132, rope: float = 500000.0):
    """A nd.DecodeCase whose query heads are orthogonal within each KV head; heads 0 .. G-2 of (b, hk) have their own needle in the cache
    (boundary positions), head G-1 has the new token's key aligned with it.  `c.needle_at[(b, h)]` is query head h's needle position."""
    c = nd.DecodeCase(seed, B, hq, hkv, lens, bits, {}, rope=rope)
    rng = np.random.default_rng(seed + 7919)
    G = c.G
    nsplit = nd.decode_splits(B, hq, hkv, max(lens), sms)
    c.needle_at = {}
    for b, L in enumerate(lens):
        for hk in range(hkv):
            c.q[b, hk * G:(hk + 1) * G] = nd.unrotate(orthogonal_rows(rng, G), L - 1, rope)
        c.qr[b] = rope_neox(c.q[b], L - 1, rope)
        for hk in range(hkv):
            pos = boundary_positions(L - 1, nsplit, G - 1, shift=hk + b)
            for h, t in zip(range(G - 1), pos):
                nd.write_row(c.kp, c.bt[b, t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE, hk, _key(c.qr[b, hk * G + h], bits))
                c.needle_at[(b, hk * G + h)] = t
            last = hk * G + G - 1
            c.k[b, hk] = nd.unrotate(_key(c.qr[b, last], bits, quant=False), L - 1, rope)
            c.needle_at[(b, last)] = L - 1
    return c


def decode_head(c, b: int, hk: int, q=None):
    """(out, bar) [G, D] of kv head hk of sequence b, optionally for other rotated query rows q [G, D] (a mis-mapped head group)."""
    L = c.lens[b]
    n = L - 1
    qs = c.qr[b, hk * c.G:(hk + 1) * c.G] if q is None else q
    C = qs.shape[0]
    kr = rope_neox(c.k[b, hk], n, c.rope).astype(np.float64)
    own_k = np.repeat(kr[None], C, 0)
    own_v = np.repeat(c.v[b, hk][None].astype(np.float64), C, 0)
    n_acc = (n + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE + 2
    return nd.paged_exact(qs, c.kp, c.vp, c.bt[b], n, hk, own_k, own_v, None, n_acc=n_acc, rope_rel=2.0 ** -10)


def decode_exact(c):
    out = np.zeros((c.B, c.hq, D))
    bar = np.zeros_like(out)
    for b in range(c.B):
        for hk in range(c.hkv):
            s = slice(hk * c.G, (hk + 1) * c.G)
            out[b, s], bar[b, s] = decode_head(c, b, hk)
    return out, bar


# ----------------------------------------------------------------------------------------------------------------------------------------
# chain / tree verify: multi_token_decode_attention
# ----------------------------------------------------------------------------------------------------------------------------------------
def children(c, b: int, r: int):
    """The direct children of row r of sequence b (chain: row r + 1)."""
    n = c.N[b]
    if c.kind == "chain":
        return [r + 1] if r + 1 < n else []
    return [j for j in range(r + 1, n) if ancestors(c.masks[b][j], j)[-1:] == [r]]


def chunk_case(seed, kind, P, N, hq, hkv, bits, masks=None, rope: float = 500000.0):
    """A nd.ChunkCase ("chain" / "tree") with head-tagged needles: the n_b G columns of each (b, hk) have orthogonal rotated queries; every
    column but the last of a row has a visible needle in the prefix (while the prefix has room); the key of row r is aligned with its own
    last column, with the first column of each direct child of r (visible) and with the last column of row r - 1 (forbidden).  Records
    `c.probe_visible[(b, hk)] = [(row r, (row, head))]` and `c.probe_forbidden` likewise."""
    assert kind in ("chain", "tree")
    c = nd.ChunkCase(seed, kind, P, N, hq, hkv, bits, {}, masks=masks, rope=rope)
    rng = np.random.default_rng(seed + 7919)
    G, T = c.G, c.qkv.shape[0]
    q = c.qkv[:, : hq * D].reshape(T, hq, D)
    k = c.qkv[:, hq * D: (hq + hkv) * D].reshape(T, hkv, D)
    c.probe_visible, c.probe_forbidden = {}, {}
    for b, n in enumerate(N):
        s = int(c.cu[b])
        for hk in range(hkv):
            Q = orthogonal_rows(rng, n * G).reshape(n, G, D)
            for i in range(n):
                q[s + i, hk * G:(hk + 1) * G] = nd.unrotate(Q[i], int(c.pos[s + i]), rope)
    qr = np.stack([rope_neox(q[t], int(c.pos[t]), rope) for t in range(T)]) if T else q.astype(np.float64)
    c.qr = qr
    v = c.qkv[:, (hq + hkv) * D:].reshape(T, hkv, D)
    v[:, :, 0] = OWN_V_OUTLIER
    c.cache_needle = {}
    for b, n in enumerate(N):
        s = int(c.cu[b])
        for hk in range(hkv):
            cols = [(i, h) for i in range(n) for h in range(G - 1)]
            for (i, h), t in zip(cols, boundary_positions(P[b], 1, len(cols), shift=hk + b)):
                nd.write_row(c.kp, c.bt[b, t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE, hk, _key(qr[s + i, hk * G + h], bits))
                c.cache_needle[(b, hk, i, h)] = t
            vis, forb = [], []
            for r in range(n):
                seen = [(j, 0) for j in children(c, b, r)]
                unseen = [(r - 1, G - 1)] if r >= 1 else []
                vis += [(r, col) for col in seen]
                forb += [(r, col) for col in unseen]
                cols = [(r, G - 1)] + seen + unseen
                k[s + r, hk] = nd.unrotate(_key(np.stack([qr[s + i, hk * G + h] for i, h in cols]), bits), int(c.pos[s + r]), rope)
            c.probe_visible[(b, hk)], c.probe_forbidden[(b, hk)] = vis, forb
    return c


def chunk_allowed(c, b: int):
    """[n_b, P_b + n_b - 1] bool: the cache positions row i reads (its own key aside)."""
    n, P = c.N[b], c.P[b]
    al = np.zeros((n, P + n - 1), bool)
    for i in range(n):
        al[i, c.allowed(b, i)] = True
    return al


def chunk_head(c, b: int, hk: int, q, k, v, kpool, vpool, allowed=None, qcols=None, cols=None):
    """(out, bar) [n_b G, D] of kv head hk of sequence b, columns c = i G + h: ChunkCase.exact_head with a per-COLUMN allowed matrix
    allowed [n_b G, P_b + n_b - 1] and per-column rotated queries qcols [n_b G, D] (default: the op's); `cols`: only these columns."""
    n, P, G = c.N[b], c.P[b], c.G
    s = int(c.cu[b])
    cached = P + n - 1
    qs = np.asarray(q[s:s + n, hk * G:(hk + 1) * G], np.float64).reshape(n * G, D) if qcols is None else qcols
    al = np.repeat(chunk_allowed(c, b), G, 0) if allowed is None else allowed
    own_k = np.repeat(np.asarray(k[s:s + n, hk], np.float64), G, 0)
    own_v = np.repeat(np.asarray(v[s:s + n, hk], np.float64), G, 0)
    if cols is not None:
        qs, al, own_k, own_v = qs[cols], al[cols], own_k[cols], own_v[cols]
    n_acc = (cached + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE + 2
    # the mistakes re-evaluate a head many times over the same pools: dequantise its cache once
    memo = c.__dict__.setdefault("_rows", {})
    key = (b, hk, id(kpool), id(vpool))
    if key not in memo:
        memo[key] = (kpool, vpool, nd.cached_rows(kpool, vpool, c.bt[b], cached, hk))  # the pools are held so their ids stay unique
    return nd.paged_exact(qs, kpool, vpool, c.bt[b], cached, hk, own_k, own_v, al, n_acc=n_acc, rows=memo[key][2])


# ----------------------------------------------------------------------------------------------------------------------------------------
# prompt kernels: prefix_prefill_attention and flash_attn_varlen_func
# ----------------------------------------------------------------------------------------------------------------------------------------
def prompt_case(seed, P, N, hq, hkv, bits, rope: float = 500000.0):
    """A nd.ChunkCase ("prefix") whose query head h of kv head hk has its own base direction in the low-frequency RoPE pairs (orthogonal
    across the heads of hk, norm sqrt(128)) plus 0.2 noise on every dim; each head has a needle in the prefix (P_b > 0) and one on a chunk
    row (the chunk keys are used un-quantised), both aligned with that head's rows alone.  `c.chunk_needle[(b, h)]` is the chunk row."""
    c = nd.ChunkCase(seed, "prefix", P, N, hq, hkv, bits, {}, rope=rope)
    rng = np.random.default_rng(seed + 7919)
    G, T = c.G, c.qkv.shape[0]
    assert G <= len(LOW_FREQ_DIMS)
    q = c.qkv[:, : hq * D].reshape(T, hq, D)
    k = c.qkv[:, hq * D: (hq + hkv) * D].reshape(T, hkv, D)
    c.chunk_needle = {}
    for b, n in enumerate(N):
        s = int(c.cu[b])
        if n == 0:
            continue
        for hk in range(hkv):
            Qb, _ = np.linalg.qr(rng.standard_normal((len(LOW_FREQ_DIMS), G)))
            base = np.zeros((G, D))
            base[:, LOW_FREQ_DIMS] = Qb.T * np.sqrt(D)
            q[s:s + n, hk * G:(hk + 1) * G] = (base[None] + 0.2 * rng.standard_normal((n, G, D))).astype(np.float16)
    qr = np.stack([rope_neox(q[t], int(c.pos[t]), rope) for t in range(T)])
    edges = [0, 1, 63, 64, 65, 127, 128, 129]
    for b, n in enumerate(N):
        s = int(c.cu[b])
        if n == 0:
            continue
        for hk in range(hkv):
            ppos = boundary_positions(P[b], 1, G, shift=hk + b)
            rows = [j for j in edges + np.linspace(0, n - 1, num=G + 2).astype(int).tolist() if j < n]
            rows = list(dict.fromkeys(rows))[(hk + b) % 3:] + list(dict.fromkeys(rows))[:(hk + b) % 3]
            for h in range(G):
                mine = qr[s:s + n, hk * G + h]
                if h < len(ppos):
                    t = ppos[h]
                    nd.write_row(c.kp, c.bt[b, t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE, hk, _key(mine, bits))
                if h < len(rows):
                    j = rows[h]
                    k[s + j, hk] = nd.unrotate(_key(mine[j:], bits, quant=False), int(c.pos[s + j]), rope)
                    c.chunk_needle[(b, hk * G + h)] = j
    return c


def prompt_head(c, b: int, hk: int, q, k, v, kpool, vpool, kv_head=None, qcols=None):
    """(out, bar) [n_b G, D] (rows major) of the query heads of kv head hk of sequence b, read through kv head `kv_head` (default hk);
    qcols [n_b g, D]: other rotated queries, g per row."""
    from .prefix import dequant_prefix
    n, P, G = c.N[b], c.P[b], c.G
    s = int(c.cu[b])
    kh = hk if kv_head is None else kv_head
    qs = np.asarray(q[s:s + n, hk * G:(hk + 1) * G], np.float64).reshape(n * G, D) if qcols is None else qcols
    pk = dequant_prefix(kpool, c.bt[b], P)[:, kh].astype(np.float64)
    pv = dequant_prefix(vpool, c.bt[b], P)[:, kh].astype(np.float64)
    keys = np.concatenate([pk, np.asarray(k[s:s + n, kh], np.float64)])
    vals = np.concatenate([pv, np.asarray(v[s:s + n, kh], np.float64)])
    g = qs.shape[0] // n
    allowed = np.concatenate([np.ones((n * g, P), bool), np.repeat(np.tril(np.ones((n, n), bool)), g, 0)], axis=1)
    vmag = np.abs(vals).max(axis=1)
    n_blk = (P + 127) // 128 + (n + 127) // 128 + 2
    return nd.exact(qs, keys, vals, allowed, v_op=vmag, acc_mag=vmag, n_acc=8 * n_blk, rope_rel=2.0 ** -18)


def prompt_exact(c, q, k, v, kpool, vpool):
    out = np.zeros((sum(c.N), c.hq, D))
    bar = np.zeros_like(out)
    G = c.G
    for b, n in enumerate(c.N):
        s = int(c.cu[b])
        for hk in range(c.hkv):
            if n:
                o, r = prompt_head(c, b, hk, q, k, v, kpool, vpool)
                out[s:s + n, hk * G:(hk + 1) * G], bar[s:s + n, hk * G:(hk + 1) * G] = o.reshape(n, G, D), r.reshape(n, G, D)
    return out, bar


# ----------------------------------------------------------------------------------------------------------------------------------------
# shared-prefix decode: shared_prefix_decode_attention
# ----------------------------------------------------------------------------------------------------------------------------------------
class SharedCase:
    """Rows of groups that share the first S_g pages of the group's first row, and rows in no group; lengths count the new token and a row's
    own pages are background with NaN scales at and beyond its new token.  Per kv head, the (member, query head) columns of a group have
    orthogonal rotated queries (each member rotated at its own position lengths[row] - 1) and a needle each in the shared pages; rows in no
    group get decode_case's needles (heads 0 .. G-2 in the cache, head G-1 on the new token).  `table` is the true page table, `poisoned`
    the one whose children's entries below S_g point at page 0 (NaN scales)."""

    def __init__(self, seed, hq, hkv, bits, groups, pages, suffix, rope: float = 500000.0):
        rng = np.random.default_rng(seed)
        self.hq, self.hkv, self.bits, self.rope = hq, hkv, bits, rope
        self.G = G = hq // hkv
        self.groups, self.pages = [list(g) for g in groups], list(pages)
        B = len(suffix)
        self.B = B
        S_of = {r: s for g, s in zip(groups, pages) for r in g}
        self.lens = [64 * S_of.get(b, 1) + suffix[b] for b in range(B)]
        blocks = max((L + 63) // 64 for L in self.lens)
        self.kp, self.vp = nd.background_pools(rng, B * blocks + 1, hkv, bits)
        for p in (self.kp, self.vp):
            p.scales()[0] = np.float16("nan")
        self.bt = 1 + np.arange(B * blocks).reshape(B, blocks)
        for b, L in enumerate(self.lens):
            for p in (self.kp, self.vp):
                nd.poison(p, self.bt[b], L - 1, blocks)
        for g, s in zip(groups, pages):
            for r in g[1:]:
                self.bt[r, :s] = self.bt[g[0], :s]
        self.poisoned = self.bt.copy()
        for g, s in zip(groups, pages):
            for r in g[1:]:
                self.poisoned[r, :s] = 0
        self.q = np.zeros((B, hq, D), np.float16)
        self.k = (0.02 * rng.standard_normal((B, hkv, D))).astype(np.float16)
        self.v = (1.5 * rng.standard_normal((B, hkv, D))).astype(np.float16)
        in_group = set(S_of)
        for g, s in zip(groups, pages):
            for hk in range(hkv):
                Q = orthogonal_rows(rng, len(g) * G).reshape(len(g), G, D)
                for j, r in enumerate(g):
                    self.q[r, hk * G:(hk + 1) * G] = nd.unrotate(Q[j], self.lens[r] - 1, rope)
        for b in range(B):
            if b not in in_group:
                for hk in range(hkv):
                    self.q[b, hk * G:(hk + 1) * G] = nd.unrotate(orthogonal_rows(rng, G), self.lens[b] - 1, rope)
        self.qr = np.stack([rope_neox(self.q[b], L - 1, rope) for b, L in enumerate(self.lens)])
        for g, s in zip(groups, pages):
            for hk in range(hkv):
                pos = boundary_positions(64 * s, 1, len(g) * G, shift=hk)
                for col, t in enumerate(pos):
                    j, h = divmod(col, G)
                    nd.write_row(self.kp, self.bt[g[0], t // 64], t % 64, hk, _key(self.qr[g[j], hk * G + h], bits))
        for b in range(B):
            if b in in_group:
                continue
            for hk in range(hkv):
                for h, t in zip(range(G - 1), boundary_positions(self.lens[b] - 1, 1, G - 1, shift=hk)):
                    nd.write_row(self.kp, self.bt[b, t // 64], t % 64, hk, _key(self.qr[b, hk * G + h], bits))
                self.k[b, hk] = nd.unrotate(_key(self.qr[b, hk * G + G - 1], bits, quant=False), self.lens[b] - 1, rope)

    def head(self, b: int, hk: int, q=None):
        """(out, bar) [G, D] of row b, kv head hk, optionally for other rotated query rows q."""
        n = self.lens[b] - 1
        qs = self.qr[b, hk * self.G:(hk + 1) * self.G] if q is None else q
        C = qs.shape[0]
        kr = rope_neox(self.k[b, hk], n, self.rope).astype(np.float64)
        n_acc = (n + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE + 2
        return nd.paged_exact(qs, self.kp, self.vp, self.bt[b], n, hk, np.repeat(kr[None], C, 0),
                              np.repeat(self.v[b, hk][None].astype(np.float64), C, 0), None, n_acc=n_acc, rope_rel=2.0 ** -10)

    def exact(self):
        out = np.zeros((self.B, self.hq, D))
        bar = np.zeros_like(out)
        for b in range(self.B):
            for hk in range(self.hkv):
                s = slice(hk * self.G, (hk + 1) * self.G)
                out[b, s], bar[b, s] = self.head(b, hk)
        return out, bar
