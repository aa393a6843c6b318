"""Oracle: prompt chunks over a cached prefix (TEST INFRASTRUCTURE, not product).

Restates the two extension ops that have no reference counterpart, on top of the reference restatements in `oracle.kv`:
  * qs_apply_bias_rope_update_kv_cache_at   `prefill_rope_append_at`: `kv.prefill_rope_append` with every position and length shifted by the
                                            sequence's cached length start_pos[b]
  * qs_prefix_prefill_attention            `prefix_causal_attention`: float64 causal attention of a chunk over the dequantised prefix
                                            (`dequant_prefix`, the reference's kv_dequant arithmetic) and the fp16 chunk itself
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .kv import TOKENS_PER_PAGE, PagePool, kv_dequant, pool_read_tokens, pool_write_token, rope_neox


def prefill_rope_append_at(qkv, seq_lens, padding_offset, start_pos, kpool: PagePool, vpool: PagePool, block_tables, num_heads: int,
                           num_kv_heads: int, max_seq_len: int, rope_base: float, max_positions: int):
    """qkv fp16 [T, (Hq+2Hkv)*D] modified IN PLACE (q and k rotated; v untouched); pages appended.

    seq_lens are CHUNK lengths of sequences whose first start_pos[b] tokens are cached.  token -> (batch, chunk position) as in
    kv.prefill_rope_append; the position is start_pos[b] + chunk position for the rotation and the page / slot, and the window uses the total
    length start_pos[b] + seq_lens[b].  With start_pos = 0 this is kv.prefill_rope_append.
    """
    qkv = np.asarray(qkv)
    T = qkv.shape[0]
    D = kpool.D
    Hq, Hkv = num_heads, num_kv_heads
    g = np.arange(T) + np.asarray(padding_offset, np.int64)
    b = g // max_seq_len
    cpos = g % max_seq_len
    start = np.asarray(start_pos, np.int64)
    pos = cpos + start[b]
    q = qkv[:, : Hq * D].reshape(T, Hq, D)
    k = qkv[:, Hq * D: (Hq + Hkv) * D].reshape(T, Hkv, D)
    v = qkv[:, (Hq + Hkv) * D:].reshape(T, Hkv, D)
    q[:] = rope_neox(q, pos[:, None], rope_base)
    k[:] = rope_neox(k, pos[:, None], rope_base)
    lens = np.asarray(seq_lens, np.int64) + start
    for t in range(T):
        if pos[t] >= max(lens[b[t]] - max_positions, 0) and pos[t] < lens[b[t]]:
            page = int(np.asarray(block_tables)[b[t], pos[t] // TOKENS_PER_PAGE])
            pool_write_token(kpool, page, int(pos[t] % TOKENS_PER_PAGE), k[t])
            pool_write_token(vpool, page, int(pos[t] % TOKENS_PER_PAGE), v[t])
    return qkv


def dequant_prefix(pool: PagePool, block_row, n_tokens: int):
    """The first n_tokens cached tokens of one sequence, dequantised as the reference does (kv.kv_dequant): fp16 [n, Hkv, D]."""
    if n_tokens == 0:
        return np.zeros((0, pool.Hkv, pool.D), np.float16)
    c, s, z = pool_read_tokens(pool, block_row, n_tokens)
    return np.ascontiguousarray(kv_dequant(c, s, z, pool.bits).transpose(1, 0, 2))


def prefix_causal_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, cu_seqlens: Sequence[int], prefix_k: Sequence[np.ndarray],
                            prefix_v: Sequence[np.ndarray], softmax_scale: Optional[float] = None) -> np.ndarray:
    """q [T, Hq, D], k / v [T, Hkv, D]: the chunk rows; prefix_k[b] / prefix_v[b] [P_b, Hkv, D]: the cached prefix of sequence b
    (dequant_prefix).  Query i of sequence b attends to all P_b prefix keys and to chunk keys 0..i.  -> float64 [T, Hq, D]."""
    T, Hq, D = q.shape
    Hkv = k.shape[1]
    assert Hq % Hkv == 0 and k.shape == v.shape and k.shape[0] == T
    g = Hq // Hkv
    scale = float(softmax_scale) if softmax_scale is not None else D ** -0.5
    out = np.zeros((T, Hq, D), dtype=np.float64)
    for b in range(len(cu_seqlens) - 1):
        s, e = int(cu_seqlens[b]), int(cu_seqlens[b + 1])
        L = e - s
        if L == 0:
            continue
        pk, pv = np.asarray(prefix_k[b]), np.asarray(prefix_v[b])
        P = pk.shape[0]
        assert pv.shape[0] == P
        mask = np.zeros((L, P + L), dtype=bool)
        mask[:, P:] = np.triu(np.ones((L, L), dtype=bool), 1)
        for h in range(Hq):
            qq = q[s:e, h].astype(np.float64)
            kk = np.concatenate([pk[:, h // g], k[s:e, h // g]]).astype(np.float64)
            vv = np.concatenate([pv[:, h // g], v[s:e, h // g]]).astype(np.float64)
            sc = qq @ kk.T * scale
            sc[mask] = -np.inf
            sc -= sc.max(axis=1, keepdims=True)
            pr = np.exp(sc)
            out[s:e, h] = (pr / pr.sum(axis=1, keepdims=True)) @ vv
    return out
