"""Oracle: verification of tree-structured drafts (TEST INFRASTRUCTURE, not product).

Restates the four extension ops of speculative decoding with token trees on top of `oracle.kv`, `oracle.prefix` and `oracle.multi_token`:
  * qs_apply_bias_rope_update_kv_cache_tree   `tree_rope_append`: node i of sequence b is rotated at position P_b + depth(i) and quantised
                                             into slot P_b + i (`kv.rope_neox`, `kv.pool_write_token`)
  * qs_tree_decode_attention                 `tree_decode_attention`: float64 attention of node i over the dequantised prefix
                                             (`prefix.dequant_prefix`), the slots of its ancestors and its own un-quantised key / value
  * qs_tree_accept_greedy                    `tree_accept_greedy`: the greedy walk from the root
  * qs_kv_cache_compact                      `kv_compact`: slot P_b + path[k] -> slot P_b + k

Tree mask: one int32 word per node; bit j of node i's word says that node j is an ancestor of node i; bits >= i are ignored.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .kv import TOKENS_PER_PAGE, PagePool, pool_write_token, rope_neox
from .prefix import dequant_prefix


def ancestors(word: int, i: int):
    """Ancestor node indices of node i, ascending (its root path without itself)."""
    w = int(word) & ((1 << i) - 1)
    return [j for j in range(i) if (w >> j) & 1]


def depth(word: int, i: int) -> int:
    return len(ancestors(word, i))


def chain_mask(n: int):
    return np.array([(1 << i) - 1 for i in range(n)], np.int32)


def root_path(mask_row, i: int):
    """The nodes a greedy acceptance of node i would accept, in order: its ancestors and itself."""
    return ancestors(mask_row[i], i) + [i]


def tree_rope_append(qkv, seq_lens, padding_offset, start_pos, tree_mask, kpool: PagePool, vpool: PagePool, block_tables, num_heads: int,
                     num_kv_heads: int, max_seq_len: int, rope_base: float, max_positions: int):
    """qkv fp16 [T, (Hq+2Hkv)*D] modified IN PLACE; tree_mask int32 [T] (one word per row).  As prefix.prefill_rope_append_at, except that
    node cpos is rotated at start_pos[b] + depth(cpos) while its page / slot and the cyclic window keep the slot position start_pos[b] + cpos."""
    qkv = np.asarray(qkv)
    T = qkv.shape[0]
    D = kpool.D
    Hq, Hkv = num_heads, num_kv_heads
    g = np.arange(T) + np.asarray(padding_offset, np.int64)
    b = g // max_seq_len
    cpos = g % max_seq_len
    start = np.asarray(start_pos, np.int64)
    slot_pos = cpos + start[b]
    rot_pos = np.array([start[b[t]] + depth(tree_mask[t], int(cpos[t])) for t in range(T)], np.int64)
    q = qkv[:, : Hq * D].reshape(T, Hq, D)
    k = qkv[:, Hq * D: (Hq + Hkv) * D].reshape(T, Hkv, D)
    v = qkv[:, (Hq + Hkv) * D:].reshape(T, Hkv, D)
    q[:] = rope_neox(q, rot_pos[:, None], rope_base)
    k[:] = rope_neox(k, rot_pos[:, None], rope_base)
    lens = np.asarray(seq_lens, np.int64) + start
    for t in range(T):
        if slot_pos[t] >= max(lens[b[t]] - max_positions, 0) and slot_pos[t] < lens[b[t]]:
            page = int(np.asarray(block_tables)[b[t], slot_pos[t] // TOKENS_PER_PAGE])
            pool_write_token(kpool, page, int(slot_pos[t] % TOKENS_PER_PAGE), k[t])
            pool_write_token(vpool, page, int(slot_pos[t] % TOKENS_PER_PAGE), v[t])
    return qkv


def tree_decode_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, cu_seqlens: Sequence[int], prefix_lens: Sequence[int], tree_mask,
                          kpool: PagePool, vpool: PagePool, block_tables, softmax_scale: Optional[float] = None) -> np.ndarray:
    """q [T, Hq, D], k / v [T, Hkv, D] fp16: the rotated node rows; tree_mask [T].  Node i of sequence b attends to the cache positions
    0 .. P_b - 1, to the slots P_b + j of its ancestors j (dequantised) and to its own key / value.  -> float64 [T, Hq, D]."""
    q, k, v = np.asarray(q), np.asarray(k), np.asarray(v)
    T, Hq, D = q.shape
    Hkv = k.shape[1]
    assert Hq % Hkv == 0 and k.shape == v.shape and k.shape[0] == T
    g = Hq // Hkv
    scale = float(softmax_scale) if softmax_scale is not None else D ** -0.5
    out = np.zeros((T, Hq, D), dtype=np.float64)
    for b in range(len(cu_seqlens) - 1):
        s, e = int(cu_seqlens[b]), int(cu_seqlens[b + 1])
        if e == s:
            continue
        P = int(prefix_lens[b])
        ck = dequant_prefix(kpool, np.asarray(block_tables)[b], P + e - s - 1).astype(np.float64)
        cv = dequant_prefix(vpool, np.asarray(block_tables)[b], P + e - s - 1).astype(np.float64)
        for i in range(e - s):
            t = s + i
            keep = list(range(P)) + [P + j for j in ancestors(tree_mask[t], i)]
            for h in range(Hq):
                hk = h // g
                qq = q[t, h].astype(np.float64)
                kk = np.concatenate([ck[keep, hk], k[t, hk][None].astype(np.float64)])
                vv = np.concatenate([cv[keep, hk], v[t, hk][None].astype(np.float64)])
                sc = kk @ qq * scale
                p = np.exp(sc - sc.max())
                out[t, h] = (p / p.sum()) @ vv
    return out


def tree_accept_greedy(draft, tree_mask, target):
    """draft / target int64 [B, n], tree_mask int32 [B, n] -> (accept_len int32 [B], path int32 [B, n] (-1 past accept_len), bonus int64 [B])."""
    draft, tree_mask, target = np.asarray(draft), np.asarray(tree_mask), np.asarray(target)
    B, n = draft.shape
    accept_len = np.zeros(B, np.int32)
    path = np.full((B, n), -1, np.int32)
    bonus = np.zeros(B, np.int64)
    for b in range(B):
        parent = [-1] + [max(ancestors(tree_mask[b, c], c), default=-1) for c in range(1, n)]
        cur, walk = 0, [0]
        while True:
            kids = [c for c in range(1, n) if parent[c] == cur and draft[b, c] == target[b, cur]]
            if not kids:
                break
            cur = kids[0]
            walk.append(cur)
        accept_len[b] = len(walk)
        path[b, : len(walk)] = walk
        bonus[b] = target[b, cur]
    return accept_len, path, bonus


def kv_compact(kpool: PagePool, vpool: PagePool, block_tables, start_pos, path, accept_len) -> None:
    """In place: slot start_pos[b] + path[b, k] -> slot start_pos[b] + k (codes, scale, zero) for k < accept_len[b]; one layer's pools."""
    bt = np.asarray(block_tables)
    for b in range(bt.shape[0]):
        P = int(start_pos[b])
        src = [P + int(path[b, k]) for k in range(int(accept_len[b]))]
        loc = lambda pos: (int(bt[b, pos // TOKENS_PER_PAGE]), pos % TOKENS_PER_PAGE)
        for pool in (kpool, vpool):
            saved = [(pool.codes()[loc(p)[0], :, loc(p)[1]].copy(), pool.scales()[loc(p)[0], :, loc(p)[1]].copy(),
                      pool.zeros()[loc(p)[0], :, loc(p)[1]].copy()) for p in src]
            for kk, (c, s, z) in enumerate(saved):
                pg, sl = loc(P + kk)
                pool.codes()[pg, :, sl], pool.scales()[pg, :, sl], pool.zeros()[pg, :, sl] = c, s, z
