"""The head-tagged needle inputs of test_gpu_attention_gqa.py have the power to see a column -> (token, head) mapping mistake (float64
oracle, no GPU).

For every configuration the GPU tests use, each mistake below is applied to the oracle the way a kernel bug would compute it, and the exact
output must move by at least 10x the bar (oracle/needles.py `exact`) at the columns the mistake affects:
  * two heads of a group swapped;
  * a column given the causal limit, ancestor word or query of the first or the last token of its n8 tile or column part (the column
    parts of multi_token_decode_attention: 8 columns when a sequence's G n fit one n8 tile, else 16);
  * a shared-prefix member's query rotated at another member's position;
  * the second or third decode head group starting at query head hk * 8 instead of hk * G + 8 gpart;
  * query head h read through KV head h % Hkv instead of h / G.
Group sizes G = 3, 5, 6, 7 (Llama-3.2-3B, Qwen2.5-14B / 32B, Qwen2.5-1.5B, Qwen2.5-7B and Yi-34B) and the synthetic 12 and 20, whose decode
head groups are 8 + 4 and 8 + 8 + 4.
"""
import numpy as np
import pytest

from oracle import gqa_needles as gq

D = 128
BITS = [4, 8]

DECODE = [  # (B, Hq, Hkv, lens): lengths count the new token
    (2, 24, 8, [1500, 700]),        # G = 3, context splits
    (3, 40, 8, [300, 65, 130]),     # G = 5, no splits
    (2, 12, 2, [2000, 1000]),       # G = 6, splits
    (2, 28, 4, [600, 129]),         # G = 7, splits
    (4, 14, 2, [200, 64, 65, 2]),   # G = 7 (Qwen2.5-7B at TP = 2), no splits; one cached token
    (2, 24, 2, [1100, 300]),        # G = 12: head groups 8 + 4, splits
    (2, 40, 2, [700, 90]),          # G = 20: head groups 8 + 8 + 4, splits
    (2, 40, 2, [400, 257]),         # G = 20, no splits
]
CHAIN = [  # (P, N, Hq, Hkv)
    ([1000, 300, 70], [1, 2, 3], 28, 4),   # G = 7: a padding column (n = 1), a tile seam (n = 2), a part seam (n = 3); splits
    ([1200, 40], [16, 5], 28, 4),          # G = 7, n = 16: 7 parts; the short sequence leaves the later parts empty
    ([700, 129], [4, 2], 40, 8),           # G = 5
    ([1100, 64, 1], [11, 3, 1], 24, 8),    # G = 3, n = 11: the last part has one column
    ([600, 65], [1, 3], 12, 2),            # G = 6, n = 1 and 3
    ([1000, 200], [1, 6], 40, 2),          # G = 20: one token across two parts, and six tokens
]
TREE_HEADS = [(28, 4), (40, 8)]             # G = 7, 5 on the binary, random and medusa trees
TREE_P = [1000, 200, 130]  # room for a cache needle per column
SHARED_G = [3, 5, 7]
SHARED_HKV = 2
SHARED_GROUPS = [[4, 0], [1], [2, 5, 3], [6, 7, 8, 9, 10], list(range(11, 29))]  # 1, 2, 3, 5 and 18 members; rows 29, 30 in no group
SHARED_PAGES = [16, 1, 3, 2, 2]
# a member's length is 64 S + suffix: member j of a group has suffix 1 + 37 j (member 0: the own token only, past the shared pages), so
# the members' RoPE positions differ by multiples of 37
SHARED_SUFFIX = [0] * 29 + [5, 100]
for _g in SHARED_GROUPS:
    for _j, _r in enumerate(_g):
        SHARED_SUFFIX[_r] = 1 + 37 * _j
PROMPT_HEADS = [(28, 4), (40, 8), (24, 2)]
PROMPT_PREFIX = ([191, 64, 1], [66, 130, 64])   # (P, N) of prefix_prefill_attention
PROMPT_FLASH = ([0, 0], [130, 65])              # (P, N) of flash_attn_varlen_func (no prefix)


def tree_masks():
    from tests.test_gpu_tree_verify import tree
    return [tree("binary"), tree("random", 16, seed=4), tree("medusa")]


def chunk_plan(G, N):
    """Columns per column part of multi_token_decode_attention: 8 if G max(N) fits one n8 tile, else 16."""
    return 8 if G * max(N) <= 8 else 16


def _moved(a, b, bar):
    return float((np.abs(np.asarray(a) - np.asarray(b)) / bar).max())


def _rows(c, qkv):
    T = qkv.shape[0]
    q = qkv[:, : c.hq * D].reshape(T, c.hq, D)
    k = qkv[:, c.hq * D: (c.hq + c.hkv) * D].reshape(T, c.hkv, D)
    v = qkv[:, (c.hq + c.hkv) * D:].reshape(T, c.hkv, D)
    return q, k, v


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode_mapping_mistakes_move_the_oracle(bits, B, Hq, Hkv, lens):
    c = gq.decode_case(11 + bits, B, Hq, Hkv, lens, bits)
    G = c.G
    worst = {"swap": np.inf, "head group": np.inf, "kv head": np.inf}
    for b in range(B):
        base = {hk: gq.decode_head(c, b, hk) for hk in range(Hkv)}
        for hk in range(Hkv):
            o, bar = base[hk]
            tagged = [h for h in range(G) if (b, hk * G + h) in c.needle_at]
            # every head has its own needle unless the sequence caches fewer than G - 1 tokens (the length-2 row at 14 / 2: heads
            # 1 .. G-2 there have none and return the same output, so a swap among them is invisible; other rows cover G = 7)
            assert len(tagged) == G or lens[b] - 1 < G - 1, (b, hk, tagged)
            for h, h2 in zip(tagged, tagged[1:]):
                worst["swap"] = min(worst["swap"], _moved(o[h2], o[h], bar[h]), _moved(o[h], o[h2], bar[h2]))
            for gpart in range(1, (G + 7) // 8):
                gc = min(8, G - 8 * gpart)
                wrong = [min(hk * 8 + 8 * gpart + r, Hq - 1) for r in range(gc)]
                if hk * 8 == hk * G:  # kv head 0: the mistake is the right mapping
                    continue
                ow, _ = gq.decode_head(c, b, hk, q=c.qr[b, wrong])
                sl = slice(8 * gpart, 8 * gpart + gc)
                worst["head group"] = min(worst["head group"], _moved(ow, o[sl], bar[sl]))
        for h in range(Hq):
            if h % Hkv != h // G and (b, h) in c.needle_at:
                ow, _ = gq.decode_head(c, b, h % Hkv, q=c.qr[b, h][None])
                o, bar = base[h // G]
                worst["kv head"] = min(worst["kv head"], _moved(ow[0], o[h % G], bar[h % G]))
    for name, m in worst.items():
        assert m >= 10, (name, m)


# ---------------------------------------------------------------------------------------------------------------------------------
# chain / tree verify
# ---------------------------------------------------------------------------------------------------------------------------------
def _seam_mistakes(c, b, hk, q, k, v, kp, vp, C):
    """The moves (one per tile / part that holds more than one token) of each straddle mistake of kv head hk of sequence b.  In each n8 tile
    and column part, every column is given the causal limit / ancestor word (kind "limit") or the query (kind "q") of the tile's first or
    last token; a tile's move is the largest over the columns whose token changed."""
    n, G = c.N[b], c.G
    base, bar = gq.chunk_head(c, b, hk, q, k, v, kp, vp)
    al_rows = gq.chunk_allowed(c, b)
    s = int(c.cu[b])
    qcols = np.asarray(q[s:s + n, hk * G:(hk + 1) * G], np.float64).reshape(n * G, D)
    res = {}
    for width in sorted({8, C}):
        for c0 in range(0, n * G, width):
            cols = np.arange(c0, min(c0 + width, n * G))
            toks = cols // G
            if toks[0] == toks[-1]:
                continue
            for end, tok in (("first", toks[0]), ("last", toks[-1])):
                hit = cols[toks != tok]
                qc = qcols.copy()
                qc[hit] = qcols[tok * G + hit % G]
                o3, _ = gq.chunk_head(c, b, hk, q, k, v, kp, vp, qcols=qc, cols=hit)
                res.setdefault((f"q of the {end} token", width), []).append(_moved(o3, base[hit], bar[hit]))
                # tree siblings share their ancestor words: only the columns whose limit / word changes are affected
                hit = np.array([x for x in hit if (al_rows[x // G] != al_rows[tok]).any()], np.int64)
                if hit.size == 0:
                    continue
                al = np.repeat(al_rows, G, 0)
                al[hit] = al_rows[tok]
                o2, _ = gq.chunk_head(c, b, hk, q, k, v, kp, vp, allowed=al, cols=hit)
                res.setdefault((f"limit of the {end} token", width), []).append(_moved(o2, base[hit], bar[hit]))
    return res, base, bar


def _chunk_checks(c, C):
    qkv, kp, vp = c.append()
    q, k, v = _rows(c, qkv)
    G = c.G
    worst = {}
    for b, n in enumerate(c.N):
        for hk in range(c.hkv):
            if n == 0:
                continue
            res, o, bar = _seam_mistakes(c, b, hk, q, k, v, kp, vp, C)
            for key, moves in res.items():
                # an ancestor word differs from a cousin's in nodes whose keys need not be aligned with the columns of that tile: the tree
                # mistake has to show in some tile of the launch, the chain mistake (a limit one token off) in every tile
                m = max(moves) if c.kind == "tree" and key[0].startswith("limit") else min(moves)
                worst[key] = (max if c.kind == "tree" and key[0].startswith("limit") else min)(worst.get(key, m), m)
            for i in range(n):
                for h in range(G - 1):
                    a, a2 = i * G + h, i * G + h + 1
                    worst["swap"] = min(worst.get("swap", np.inf), _moved(o[a2], o[a], bar[a]), _moved(o[a], o[a2], bar[a2]))
            # the draft key of row r let in for the last column of row r - 1 (a mask one position late)
            for r, (i, h) in c.probe_forbidden[(b, hk)]:
                if r == n - 1:  # the last row's slot is beyond every column's cache range: no limit can reach it
                    continue
                x = i * G + h
                al = np.repeat(gq.chunk_allowed(c, b), G, 0)
                al[x, c.P[b] + r] = True
                o2, _ = gq.chunk_head(c, b, hk, q, k, v, kp, vp, allowed=al, cols=[x])
                worst["forbidden draft key let in"] = min(worst.get("forbidden draft key let in", np.inf), _moved(o2[0], o[x], bar[x]))
    return worst


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("P,N,Hq,Hkv", CHAIN)
def test_chain_mapping_mistakes_move_the_oracle(bits, P, N, Hq, Hkv):
    c = gq.chunk_case(21 + bits, "chain", P, N, Hq, Hkv, bits)
    worst = _chunk_checks(c, chunk_plan(c.G, N))
    for name, m in worst.items():
        assert m >= 10, (name, m)


@pytest.mark.parametrize("bits", [4])  # KV4: the larger K scales and bars; the chain cases cover KV8 on the same kernel
@pytest.mark.parametrize("Hq,Hkv", TREE_HEADS)
def test_tree_mapping_mistakes_move_the_oracle(bits, Hq, Hkv):
    masks = tree_masks()
    c = gq.chunk_case(31 + bits, "tree", TREE_P, [len(m) for m in masks], Hq, Hkv, bits, masks=masks)
    worst = _chunk_checks(c, chunk_plan(c.G, c.N))
    for name, m in worst.items():
        assert m >= 10, (name, m)


# ---------------------------------------------------------------------------------------------------------------------------------
# shared-prefix decode
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("G", SHARED_G)
def test_shared_prefix_mapping_mistakes_move_the_oracle(bits, G):
    c = gq.SharedCase(41 + bits + G, G * SHARED_HKV, SHARED_HKV, bits, SHARED_GROUPS, SHARED_PAGES, SHARED_SUFFIX)
    worst = {"swap": np.inf, "member position": np.inf}
    from oracle.kv import rope_neox
    for g in SHARED_GROUPS:
        for hk in range(SHARED_HKV):
            base = {r: c.head(r, hk) for r in g}
            for r in g:
                o, bar = base[r]
                for h in range(G - 1):
                    worst["swap"] = min(worst["swap"], _moved(o[h + 1], o[h], bar[h]), _moved(o[h], o[h + 1], bar[h + 1]))
            if len(g) > 1:  # every member rotated at the next member's position: the largest move over the group's columns
                moved = 0.0
                for j, r in enumerate(g):
                    o, bar = base[r]
                    qw = rope_neox(c.q[r, hk * G:(hk + 1) * G], c.lens[g[(j + 1) % len(g)]] - 1, c.rope)
                    moved = max(moved, _moved(c.head(r, hk, q=qw)[0], o, bar))
                worst["member position"] = min(worst["member position"], moved)
    for name, m in worst.items():
        assert m >= 10, (name, m)


# ---------------------------------------------------------------------------------------------------------------------------------
# prompt kernels
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hq,Hkv", PROMPT_HEADS)
@pytest.mark.parametrize("P,N,bits", [PROMPT_PREFIX + (4,), PROMPT_PREFIX + (8,), PROMPT_FLASH + (8,)])  # no prefix: no cache read
def test_prompt_mapping_mistakes_move_the_oracle(bits, Hq, Hkv, P, N):
    c = gq.prompt_case(51 + bits, P, N, Hq, Hkv, bits)
    qkv, kp, vp = c.append()
    q, k, v = _rows(c, qkv)
    G = c.G
    worst = {"swap": np.inf, "kv head": np.inf}
    for b, n in enumerate(N):
        for hk in range(Hkv):
            o, bar = gq.prompt_head(c, b, hk, q, k, v, kp, vp)
            o, bar = o.reshape(n, G, D), bar.reshape(n, G, D)
            late = max([c.chunk_needle.get((b, hk * G + h), 0) for h in range(G)])  # rows that see every head's needle
            for h in range(G - 1):
                worst["swap"] = min(worst["swap"], _moved(o[late:, h + 1], o[late:, h], bar[late:, h]))
            if Hkv > 1:
                s = int(c.cu[b])
                for h in range(G):
                    hq_ = hk * G + h
                    if hq_ % Hkv == hk:
                        continue
                    qc = np.asarray(q[s:s + n, hq_], np.float64)
                    ow, _ = gq.prompt_head(c, b, hk, q, k, v, kp, vp, kv_head=hq_ % Hkv, qcols=qc)
                    worst["kv head"] = min(worst["kv head"], _moved(ow[late:], o[late:, h], bar[late:, h]))
    for name, m in worst.items():
        assert m >= 10, (name, m)
