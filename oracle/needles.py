"""Oracle: "needle" inputs for the paged-attention kernels (TEST INFRASTRUCTURE, not product).

Random caches put the softmax mass nearly uniformly over hundreds of tokens, so one wrong token, scale or zero point moves the output by
about |v| / L: below any bar a kernel can meet.  These inputs put the mass where the test chooses:
  * background tokens: random codes with small K scales, so their logits are near 0;
  * a needle token per (sequence, kv head): its K row is aligned with the rotated queries that read it (`needle_key`), with a logit of
    about 14 natural units, so it carries all but ~L e^-14 of the softmax mass;
  * tagged V rows: V scales large enough that |v| is about 1 to 3 and every token's row is an independent draw, so reading the wrong
    token, scale or zero point moves the output by O(1).

`exact` is the float64 attention over given (dequantised) keys and values, and returns with it the per-element bar derived from the
kernels' arithmetic (see `exact` for the derivation).  `decode_splits` / `split_of` mirror the host's context-split plan of the decode op.
"""
from __future__ import annotations

import numpy as np

from .kv import TOKENS_PER_PAGE, PagePool, kv_dequant, kv_quant_codes, kv_quant_params, pack_nibbles, rope_neox

D = 128
NEEDLE_LOGIT = 14.0
K_BACKGROUND_SCALE = (2e-3, 4e-3)
# V of the background: (scale range, zero range) of even and odd slots.  Neighbouring slots never share a scale or a zero point within
# 25 % of the range, so a kernel that takes a neighbour's scale or zero moves the output by O(1); |v| is up to about 3.
V_TAGGED = {4: (((0.15, 0.2), (4.0, 6.0)), ((0.25, 0.3), (9.0, 11.0))), 8: (((0.008, 0.0105), (100.0, 120.0)), ((0.0125, 0.015), (135.0, 155.0)))}
CODE_MAX = {4: 15.0, 8: 255.0}


def background_pools(rng, n_pages: int, hkv: int, bits: int):
    """K / V pools of background tokens: random codes, K scales in K_BACKGROUND_SCALE, tagged V."""
    kp, vp = PagePool(n_pages, hkv, D, bits), PagePool(n_pages, hkv, D, bits)
    kp.randomize(rng, K_BACKGROUND_SCALE)
    vp.randomize(rng)
    for parity, (sr, zr) in enumerate(V_TAGGED[bits]):
        shape = vp.scales()[:, :, parity::2].shape
        vp.scales()[:, :, parity::2] = rng.uniform(*sr, size=shape).astype(np.float16)
        vp.zeros()[:, :, parity::2] = rng.uniform(*zr, size=shape).astype(np.float16)
    return kp, vp


def poison(pool: PagePool, block_row, start: int, n_blocks: int):
    """NaN scales in every slot of the sequence's pages at positions >= start: a kernel that reads one produces NaN."""
    for t in range(start, n_blocks * TOKENS_PER_PAGE):
        pool.scales()[block_row[t // TOKENS_PER_PAGE], :, t % TOKENS_PER_PAGE] = np.float16("nan")


def write_row(pool: PagePool, page: int, slot: int, hk: int, x):
    """Quantise one token of one kv head (fp16 [D]) into the pool, as the append kernels do."""
    x = np.asarray(x, np.float16)[None]
    s, z = kv_quant_params(x, pool.bits)
    u = kv_quant_codes(x, s, z, pool.bits)
    pool.codes()[page, hk, slot] = pack_nibbles(u)[0] if pool.bits == 4 else u[0]
    pool.scales()[page, hk, slot] = s[0]
    pool.zeros()[page, hk, slot] = z[0]


def quantised(x, bits: int):
    """fp16 [D] -> what the cache returns for it after quantisation (float64)."""
    x = np.asarray(x, np.float16)[None]
    s, z = kv_quant_params(x, bits)
    return kv_dequant(kv_quant_codes(x, s, z, bits), s, z, bits)[0].astype(np.float64)


def needle_key(queries, bits: int, logit: float = NEEDLE_LOGIT, quant: bool = True, scale: float = D ** -0.5):
    """queries float [n, D]: the rotated query rows that will read the key.  Returns the fp16 key k = a * sum_i q_i / |q_i| whose cached
    (quantised, if `quant`) form gives every query a logit of at least `logit` (natural units)."""
    q = np.asarray(queries, np.float64).reshape(-1, D)
    u = (q / np.linalg.norm(q, axis=1, keepdims=True)).sum(axis=0)
    m = scale * (q @ u).min()
    assert m > 0, "needle queries are not aligned enough to share one key"
    a = logit / m
    for _ in range(3):  # the quantisation shrinks some logits a little: rescale on the cached form
        k = (a * u).astype(np.float16)
        kd = quantised(k, bits) if quant else k.astype(np.float64)
        a *= logit / (scale * (q @ kd).min())
    return (a * u).astype(np.float16)


def unrotate(x, pos: int, base: float):
    """The pre-RoPE row whose rotation at `pos` is x (up to fp16 rounding)."""
    return rope_neox(np.asarray(x, np.float16), -pos, base)


# ----------------------------------------------------------------------------------------------------------------------------------------
# context splits, as the host plans them (attention.cu decode_attention(); plan_multi_token() applies the same rule with its own CTA count)
# ----------------------------------------------------------------------------------------------------------------------------------------
def _splits(ctas: int, slots: int, ctx: int) -> int:
    n = 1
    if 2 * ctas <= slots and ctx > 512:
        n = min((slots + ctas - 1) // ctas, (ctx + 255) // 256, 32)
    return n


def decode_splits(batch: int, hq: int, hkv: int, max_len: int, sms: int) -> int:
    """Context splits of single_query_attention: max_len is the timestep argument (the longest length, new token included)."""
    g = hq // hkv
    return _splits(hkv * ((g + 7) // 8) * batch, sms * 4, max_len)


def split_of(t: int, n_cached: int, nsplit: int) -> int:
    """The split that streams cache position t of a sequence with n_cached cached tokens (pages are dealt out in equal runs)."""
    n_pages = (n_cached + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE
    pps = (n_pages + nsplit - 1) // nsplit
    return (t // TOKENS_PER_PAGE) // pps


# ----------------------------------------------------------------------------------------------------------------------------------------
# float64 attention and its bar
# ----------------------------------------------------------------------------------------------------------------------------------------
def ulp16(a):
    a = np.abs(np.asarray(a, np.float64))
    return np.where(a >= 2.0 ** -14, 2.0 ** (np.floor(np.log2(np.maximum(a, 2.0 ** -14))) - 10), 2.0 ** -24)


def exact(q, keys, vals, allowed=None, *, v_op, acc_mag, n_acc: int, k_mma=None, rope_rel: float = 0.0, scale: float = D ** -0.5):
    """Float64 attention of query columns over a shared token list, with the per-element bar of the kernel that computes it.

    q [C, D]: rotated queries; keys / vals [n, D]: the cached tokens as the kernel reads them (dequantised) and the un-quantised own
    tokens; allowed [C, n] bool (None: all).  Per token:
      v_op    bound of |P' x operand| per unit p: the V scale times the largest code (paged kernels: s_v * 15 | 255; fp16 rows: max |v|)
      acc_mag what the fp32 PV accumulator holds per unit p: 2^11 s_v for the biased code operands (1024 + u, 1024 + 16 u < 2^11), max |v|
              for fp16 rows
      k_mma   for cached K rows read through biased-code MMAs, the K scale (else 0): the QK accumulator holds up to 2^11 s_k sum_d |q_d|
    Returns (out [C, D], bar [C, D]).

    Bar, per element:   |out - exact| <= 2 ulp16(|exact|) + 2^-11 sum_t p_t v_op_t + n_acc 2^-23 sum_t p_t acc_mag_t
                                        + 2.2 delta sum_t p_t |v_t - exact|
      * 2 ulp16: the final fp16 rounding (half an ulp) with room for the fp32 merges of warps and splits;
      * 2^-11: P' = p s_v (or P) is rounded to fp16 before the PV MMA, one relative rounding of every token's contribution;
      * n_acc 2^-23: each of the n_acc MMAs that accumulate into one fp32 output register rounds (or truncates) at most one ulp of its
        magnitude;
      * delta bounds the logit error (natural units): with logit errors e_t the normalised weights move by at most
        (exp(2 max|e|) - 1) p_t <= 2.2 delta p_t (delta < 0.05), and sum_t dp_t = 0, so the output moves by at most that times
        sum_t p_t |v_t - exact|.  delta = the QK terms (16 2^-23 2^11 + 20 2^-24 2^10) sum_d |q_d| s_k scale: 8 accumulating MMAs per
        16-token chunk, each rounding twice (its aligned product sum and the accumulator), and the fp32 sums of q behind the bias 1024 sum q
        (about 20 fp32 additions per sum)
        + rope_rel |logit| (the query rotated by another RoPE implementation, 1 fp16 ulp per element: 2^-10 relative) + 2^-20 (ex2.approx).
    The QK term is a model of the tensor cores' fp32 accumulation, not a proof: Hopper aligns the products to the largest exponent and
    truncates, and the model allows two ulps of the accumulator's magnitude per MMA, with the accumulator bounded by 2^11 sum_d |q_d|.
    A one-ulp model without the bias sums was exceeded by up to 2.2x on the chain verify at KV8 outlier magnitudes (K channels of 20 to
    50, |q| up to 10), where the cancellation of 1024 sum q against the code sum is largest relative to s_k; the outlier tests measure
    the kernels against this model.
    """
    q = np.asarray(q, np.float64)
    keys, vals = np.asarray(keys, np.float64), np.asarray(vals, np.float64)
    lg = (q @ keys.T) * scale
    if allowed is not None:
        lg = np.where(allowed, lg, -np.inf)
    p = np.exp(lg - lg.max(axis=1, keepdims=True))
    p /= p.sum(axis=1, keepdims=True)
    out = p @ vals
    finite = np.where(np.isfinite(lg), np.abs(lg), 0.0)
    qa = np.abs(q).sum(axis=1, keepdims=True)
    dl = rope_rel * finite + 2.0 ** -20
    if k_mma is not None:
        dl = dl + (16 * 2.0 ** -12 + 20 * 2.0 ** -14) * qa * np.asarray(k_mma, np.float64)[None] * scale
    delta = np.where(p > 0, dl, 0.0).max(axis=1, keepdims=True)
    spread = np.einsum("ct,ctd->cd", p, np.abs(vals[None] - out[:, None]))
    bar = (2 * ulp16(out) + 2.0 ** -11 * (p @ np.asarray(v_op, np.float64))[:, None]
           + n_acc * 2.0 ** -23 * (p @ np.asarray(acc_mag, np.float64))[:, None] + 2.2 * delta * spread)
    return out, bar


def cached_rows(kpool: PagePool, vpool: PagePool, block_row, n: int, hk: int):
    """Tokens 0..n-1 of kv head hk: (K float64 [n, D], V float64 [n, D], K scale [n], V scale [n]) as the cache returns them."""
    from .kv import unpack_nibbles
    t = np.arange(n)
    pages, slots = np.asarray(block_row)[t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE
    res = []
    for pool in (kpool, vpool):
        raw = pool.codes()[pages, hk, slots]
        codes = unpack_nibbles(raw) if pool.bits == 4 else raw
        s, z = pool.scales()[pages, hk, slots], pool.zeros()[pages, hk, slots]
        res += [kv_dequant(codes, s, z, pool.bits).astype(np.float64), s.astype(np.float64)]
    return res[0], res[2], res[1], res[3]


def paged_exact(q, kpool, vpool, block_row, n: int, hk: int, own_k, own_v, allowed=None, *, n_acc: int, rope_rel: float = 0.0, rows=None):
    """exact() for the paged kernels: columns q [C, D] over cache tokens 0..n-1 of kv head hk, then one un-quantised own token per column
    (own_k / own_v [C, D], None: no own token).  allowed [C, n] masks the cache tokens.  rows: cached_rows() of these arguments, if the
    caller already has them."""
    kd, vd, ks, vs = cached_rows(kpool, vpool, block_row, n, hk) if rows is None else rows
    U = CODE_MAX[vpool.bits]
    q = np.asarray(q, np.float64)
    C = q.shape[0]
    al = np.ones((C, n), bool) if allowed is None else np.asarray(allowed, bool)
    if own_k is None:
        return exact(q, kd, vd, al, v_op=vs * U, acc_mag=2.0 ** 11 * vs, n_acc=n_acc, k_mma=ks, rope_rel=rope_rel)
    # each column has its own "own" token: append all of them and let column c see only its own
    own_k, own_v = np.asarray(own_k, np.float64), np.asarray(own_v, np.float64)
    keys, vals = np.concatenate([kd, own_k]), np.concatenate([vd, own_v])
    al = np.concatenate([al, np.eye(C, dtype=bool)], axis=1)
    vmag = np.abs(own_v).max(axis=1)
    return exact(q, keys, vals, al, v_op=np.concatenate([vs * U, np.zeros(C)]), acc_mag=np.concatenate([2.0 ** 11 * vs, vmag]), n_acc=n_acc,
                 k_mma=np.concatenate([ks, np.zeros(C)]), rope_rel=rope_rel)


# ----------------------------------------------------------------------------------------------------------------------------------------
# decode: single_query_attention over needle caches
# ----------------------------------------------------------------------------------------------------------------------------------------
class DecodeCase:
    """A decode batch (lengths count the new token) whose (sequence, kv head) pairs hold a needle at the position `needles[(b, hk)]`
    (lens[b] - 1: the new token itself), and optionally a second needle `second[(b, hk)] = (t, gap)` whose logit is `gap` below the first.
    Pages are background (`background_pools`); every slot at or beyond the new token's holds NaN scales."""

    def __init__(self, seed, B, hq, hkv, lens, bits, needles, second=None, rope: float = 500000.0):
        rng = np.random.default_rng(seed)
        self.B, self.hq, self.hkv, self.lens, self.bits, self.rope = B, hq, hkv, list(lens), bits, rope
        self.G = hq // hkv
        self.n_blocks = (max(lens) + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE
        pages = B * self.n_blocks + 1
        self.kp, self.vp = background_pools(rng, pages, hkv, bits)
        self.bt = 1 + np.arange(B * self.n_blocks).reshape(B, self.n_blocks)
        for b, L in enumerate(lens):
            for p in (self.kp, self.vp):
                poison(p, self.bt[b], L - 1, self.n_blocks)
        base = rng.standard_normal((B, hkv, 1, D))  # the heads of a group share a direction, so one key can serve all of them
        self.q = (np.repeat(base, self.G, axis=2).reshape(B, hq, D) + 0.5 * rng.standard_normal((B, hq, D))).astype(np.float16)
        self.k = (0.02 * rng.standard_normal((B, hkv, D))).astype(np.float16)
        self.v = (1.5 * rng.standard_normal((B, hkv, D))).astype(np.float16)
        self.qr = np.stack([rope_neox(self.q[b], L - 1, rope) for b, L in enumerate(lens)])
        self.needles = dict(needles)
        marks = [(key, t, 0.0) for key, t in self.needles.items()]
        marks += [(key, t, gap) for key, (t, gap) in (second or {}).items()]
        for (b, hk), t, gap in marks:
            L = lens[b]
            qs = self.qr[b, hk * self.G:(hk + 1) * self.G]
            if t == L - 1:
                self.k[b, hk] = unrotate(needle_key(qs, bits, NEEDLE_LOGIT - gap, quant=False), L - 1, rope)
            else:
                key = needle_key(qs, bits, NEEDLE_LOGIT - gap)
                write_row(self.kp, self.bt[b, t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE, hk, key)

    def exact_head(self, b: int, hk: int, kpool=None, vpool=None, drop=None):
        """(out, bar) [G, D] of the query heads of kv head hk of sequence b; `drop`: cache positions the attention must not see."""
        L = self.lens[b]
        n = L - 1
        allowed = np.ones((self.G, n), bool)
        if drop is not None:
            allowed[:, list(drop)] = False
        kr = rope_neox(self.k[b, hk], n, self.rope)
        own_k = np.repeat(kr[None].astype(np.float64), self.G, 0)
        own_v = np.repeat(self.v[b, hk][None].astype(np.float64), self.G, 0)
        n_acc = (n + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE + 2  # 16-token chunks one warp accumulates: two per page it streams
        return paged_exact(self.qr[b, hk * self.G:(hk + 1) * self.G], kpool or self.kp, vpool or self.vp, self.bt[b], n, hk, own_k, own_v,
                           allowed, n_acc=n_acc, rope_rel=2.0 ** -10)

    def exact(self):
        out = np.zeros((self.B, self.hq, D))
        bar = np.zeros_like(out)
        for b in range(self.B):
            for hk in range(self.hkv):
                o, r = self.exact_head(b, hk)
                out[b, hk * self.G:(hk + 1) * self.G], bar[b, hk * self.G:(hk + 1) * self.G] = o, r
        return out, bar


def sweep(lens, hkv: int):
    """Launches of a needle sweep: in launch r, kv head hk of sequence b holds its needle at r * hkv + hk (while < lens[b]), so after
    ceil(max(lens) / hkv) launches every position 0 .. L-1 of every sequence, the new token included, has held a needle."""
    rounds = (max(lens) + hkv - 1) // hkv
    return [{(b, hk): r * hkv + hk for b, L in enumerate(lens) for hk in range(hkv) if r * hkv + hk < L} for r in range(rounds)]


# ----------------------------------------------------------------------------------------------------------------------------------------
# chain / tree verify (multi_token_decode_attention) and prefix prefill (prefix_prefill_attention) over needle caches
# ----------------------------------------------------------------------------------------------------------------------------------------
class ChunkCase:
    """n_b rows per sequence behind cached prefixes P_b.  kind "chain" / "tree": draft tokens of a verify (row i sits at cache position
    P_b + i; tree rows are rotated at P_b + depth); kind "prefix": a prompt chunk (every chunk key is used un-quantised).

    needles[(b, hk)] = t: a needle at cache position t < P_b (in the prefix) or, for t >= P_b, on row j = t - P_b, aligned with the rows
    `targets(b, j)` (chain: j and later rows, tree / prefix: every row).  The queries of a (sequence, kv head) share a direction
    (base + 0.5 noise), so one key can serve all of them.  The rows' pre-RoPE q / k / v are `qkv`; `append` quantises them into the
    pools as the append op does; `exact` takes the rows as rotated by the op (`q`, `k` [T, H, D]) and the pools it left."""

    def __init__(self, seed, kind, P, N, hq, hkv, bits, needles, masks=None, logit: float = NEEDLE_LOGIT, rope: float = 500000.0):
        from .tree import depth
        rng = np.random.default_rng(seed)
        self.kind, self.P, self.N, self.hq, self.hkv, self.bits, self.rope = kind, list(P), list(N), hq, hkv, bits, rope
        self.G = hq // hkv
        self.masks = masks
        B, T = len(P), sum(N)
        self.cu = np.concatenate([[0], np.cumsum(N)]).astype(np.int32)
        self.n_blocks = max(1, (max(P) + max(N) + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE)  # the ops check max(P) + max(N) against the table
        self.kp, self.vp = background_pools(rng, B * self.n_blocks + 1, hkv, bits)
        self.bt = 1 + np.arange(B * self.n_blocks).reshape(B, self.n_blocks)
        for b in range(B):
            for p in (self.kp, self.vp):
                poison(p, self.bt[b], P[b], self.n_blocks)
        base = rng.standard_normal((B, hkv, 1, D))
        q = (np.repeat(base, self.G, axis=2).reshape(B, hq, D)[np.repeat(np.arange(B), N)]
             + 0.5 * rng.standard_normal((T, hq, D))).astype(np.float16)
        k = (0.02 * rng.standard_normal((T, hkv, D))).astype(np.float16)
        v = (1.5 * rng.standard_normal((T, hkv, D))).astype(np.float16)
        self.pos = np.zeros(T, np.int64)  # RoPE position of every row
        for b in range(B):
            for i in range(N[b]):
                d = depth(masks[b][i], i) if kind == "tree" else i
                self.pos[self.cu[b] + i] = P[b] + d
        qr = np.stack([rope_neox(q[t], self.pos[t], rope) for t in range(T)]) if T else q
        self.needles = dict(needles)
        for (b, hk), t in self.needles.items():
            rows = self.cu[b] + (np.arange(N[b]) if t < P[b] else np.asarray(self.targets(b, t - P[b])))
            qs = qr[rows, hk * self.G:(hk + 1) * self.G].reshape(-1, D)
            if t < P[b]:
                write_row(self.kp, self.bt[b, t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE, hk, needle_key(qs, bits, logit))
            else:
                row = self.cu[b] + t - P[b]
                k[row, hk] = unrotate(needle_key(qs, bits, logit, quant=(kind != "prefix")), self.pos[row], rope)
        self.qkv = np.concatenate([q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)], axis=1)

    def targets(self, b, j):
        n = self.N[b]
        return list(range(j, n)) if self.kind == "chain" else list(range(n))

    def allowed(self, b, i):
        """Cache positions row i of sequence b attends to (its own key aside)."""
        from .tree import ancestors
        P = self.P[b]
        if self.kind == "prefix":
            return np.arange(P)
        if self.kind == "tree":
            return np.array(list(range(P)) + [P + j for j in ancestors(self.masks[b][i], i)], np.int64)
        return np.arange(P + i)

    def append(self):
        """Host model of the append op: -> (rotated qkv, K pool, V pool) after it."""
        from .prefix import prefill_rope_append_at
        from .tree import tree_rope_append
        kp, vp = PagePool(self.kp.data.shape[0], self.hkv, D, self.bits), PagePool(self.vp.data.shape[0], self.hkv, D, self.bits)
        kp.data[:], vp.data[:] = self.kp.data, self.vp.data
        qkv = self.qkv.copy()
        T = qkv.shape[0]
        pad = np.concatenate([np.full(n, b * max(self.N) - self.cu[b]) for b, n in enumerate(self.N)]).astype(np.int64)
        if self.kind == "tree":
            tm = np.concatenate([np.asarray(m, np.int64) for m in self.masks]).astype(np.int32)
            tree_rope_append(qkv, self.N, pad, self.P, tm, kp, vp, self.bt, self.hq, self.hkv, max(self.N), self.rope, 8192)
        else:
            prefill_rope_append_at(qkv, self.N, pad, self.P, kp, vp, self.bt, self.hq, self.hkv, max(self.N), self.rope, 8192)
        return qkv.reshape(T, -1), kp, vp

    def exact_head(self, b, hk, q, k, v, kpool, vpool, extra=None, drop=None):
        """(out, bar) [n_b * G, D] of kv head hk of sequence b (rows major, heads minor).  q / k / v: the rows as the op rotated them.
        extra[i] / drop[i]: cache positions row i additionally sees / does not see."""
        n, P, G = self.N[b], self.P[b], self.G
        s = self.cu[b]
        cached = P if self.kind == "prefix" else P + n - 1
        qs = np.asarray(q[s:s + n, hk * G:(hk + 1) * G], np.float64).reshape(n * G, D)
        allowed = np.zeros((n * G, cached), bool)
        for i in range(n):
            a = (set(self.allowed(b, i).tolist()) | set((extra or {}).get(i, ()))) - set((drop or {}).get(i, ()))
            allowed[i * G:(i + 1) * G, sorted(a)] = True
        if self.kind != "prefix":
            own_k = np.repeat(np.asarray(k[s:s + n, hk], np.float64), G, 0)
            own_v = np.repeat(np.asarray(v[s:s + n, hk], np.float64), G, 0)
            n_acc = (cached + TOKENS_PER_PAGE - 1) // TOKENS_PER_PAGE + 2
            return paged_exact(qs, kpool, vpool, self.bt[b], cached, hk, own_k, own_v, allowed, n_acc=n_acc)
        # prefix prefill: the dequantised prefix and the fp16 chunk (causal), both as fp16 wgmma operands
        from .prefix import dequant_prefix
        pk = dequant_prefix(kpool, self.bt[b], P)[:, hk].astype(np.float64)
        pv = dequant_prefix(vpool, self.bt[b], P)[:, hk].astype(np.float64)
        keys = np.concatenate([pk, np.asarray(k[s:s + n, hk], np.float64)])
        vals = np.concatenate([pv, np.asarray(v[s:s + n, hk], np.float64)])
        causal = np.repeat(np.tril(np.ones((n, n), bool)), G, 0)
        vmag = np.abs(vals).max(axis=1)
        n_blk = (P + 127) // 128 + (n + 127) // 128 + 2  # 128-key blocks accumulated into one output register
        return exact(qs, keys, vals, np.concatenate([allowed, causal], axis=1), v_op=vmag, acc_mag=vmag, n_acc=8 * n_blk, rope_rel=2.0 ** -18)

    def exact(self, q, k, v, kpool, vpool):
        out = np.zeros((sum(self.N), self.hq, D))
        bar = np.zeros_like(out)
        G = self.G
        for b in range(len(self.P)):
            s, n = self.cu[b], self.N[b]
            for hk in range(self.hkv):
                if n == 0:
                    continue
                o, r = self.exact_head(b, hk, q, k, v, kpool, vpool)
                out[s:s + n, hk * G:(hk + 1) * G], bar[s:s + n, hk * G:(hk + 1) * G] = o.reshape(n, G, D), r.reshape(n, G, D)
        return out, bar


# ----------------------------------------------------------------------------------------------------------------------------------------
# outlier magnitudes: LLM-like key statistics
# ----------------------------------------------------------------------------------------------------------------------------------------
OUTLIER_CHANNELS = (60, 61, 62, 63, 124, 125, 126, 127)  # the lowest RoPE frequencies: a rotation by any position of a 2k context leaves them


def outlier_rows(rng, n: int, mags):
    """n key rows: N(0, 0.7^2) plus the outlier channels at f_t * mags (f_t ~ U(0.5, 1) per token).  With mags in [20, 50] a row's KV4
    scale is about 1 to 4."""
    x = 0.7 * rng.standard_normal((n, D))
    f = rng.uniform(0.5, 1.0, size=(n, 1))
    x[:, list(OUTLIER_CHANNELS)] += f * mags[None]
    return x.astype(np.float16)


def outlier_queries(rng, shape):
    """Query rows N(0, 1) with the outlier channels at U(3, 10): |q| up to 10, logits spread over tens of natural units (a peaked
    softmax with a few tokens near the top)."""
    q = rng.standard_normal(shape)
    q[..., list(OUTLIER_CHANNELS)] = rng.uniform(3.0, 10.0, size=shape[:-1] + (len(OUTLIER_CHANNELS),))
    return q.astype(np.float16)


def write_rows(pool: PagePool, block_row, hk: int, X):
    """Quantise rows X fp16 [n, D] into cache positions 0 .. n-1 of kv head hk."""
    X = np.asarray(X, np.float16)
    t = np.arange(X.shape[0])
    pages, slots = np.asarray(block_row)[t // TOKENS_PER_PAGE], t % TOKENS_PER_PAGE
    s, z = kv_quant_params(X, pool.bits)
    u = kv_quant_codes(X, s, z, pool.bits)
    pool.codes()[pages, hk, slots] = pack_nibbles(u) if pool.bits == 4 else u
    pool.scales()[pages, hk, slots] = s
    pool.zeros()[pages, hk, slots] = z


def with_outliers(case, seed: int):
    """Replace the keys and queries of a DecodeCase / ChunkCase (built without needles) by outlier statistics: every cached key of every
    (sequence, kv head), the new / draft keys and all queries."""
    rng = np.random.default_rng(seed)
    hq, hkv, G = case.hq, case.hkv, case.G
    mags = rng.uniform(20.0, 50.0, size=(hkv, len(OUTLIER_CHANNELS)))
    if isinstance(case, DecodeCase):
        cached = [L - 1 for L in case.lens]
        case.q[:] = outlier_queries(rng, case.q.shape)
        for b in range(case.B):
            for hk in range(hkv):
                case.k[b, hk] = unrotate(outlier_rows(rng, 1, mags[hk])[0], case.lens[b] - 1, case.rope)
        case.qr = np.stack([rope_neox(case.q[b], L - 1, case.rope) for b, L in enumerate(case.lens)])
    else:
        cached = list(case.P)
        T = case.qkv.shape[0]
        q = case.qkv[:, : hq * D].reshape(T, hq, D)
        k = case.qkv[:, hq * D: (hq + hkv) * D].reshape(T, hkv, D)
        q[:] = outlier_queries(rng, q.shape)
        for t in range(T):
            for hk in range(hkv):
                k[t, hk] = unrotate(outlier_rows(rng, 1, mags[hk])[0], int(case.pos[t]), case.rope)
    for b, n in enumerate(cached):
        for hk in range(hkv):
            if n:
                write_rows(case.kp, case.bt[b], hk, outlier_rows(rng, n, mags[hk]))
    return case
