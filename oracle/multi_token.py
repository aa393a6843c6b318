"""Oracle: multi-token decode attention for speculative-decoding verification (TEST INFRASTRUCTURE, not product).

Restates qs_multi_token_decode_attention, an extension op without a reference counterpart, on top of `oracle.kv` and `oracle.prefix`:
query token i of sequence b (position P_b + i, rotated and appended by `prefix.prefill_rope_append_at`) is the decode step at that position
(`kv.decode_attention`): it attends to the cache positions 0 .. P_b + i - 1 dequantised from the pages (`prefix.dequant_prefix`, the
reference's kv_dequant arithmetic; the earlier draft tokens of the step are read back quantised) and to its own key and value as the
un-quantised fp16 rows.  Float64 after the dequantisation.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .kv import PagePool
from .prefix import dequant_prefix


def multi_token_decode_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, cu_seqlens: Sequence[int], prefix_lens: Sequence[int],
                                 kpool: PagePool, vpool: PagePool, block_tables, softmax_scale: Optional[float] = None) -> np.ndarray:
    """q [T, Hq, D], k / v [T, Hkv, D] fp16: the rotated draft rows; cu_seqlens [B + 1] draft offsets; prefix_lens [B]; the pools hold the
    prefix and the appended draft tokens.  -> float64 [T, Hq, D]."""
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
        ck = dequant_prefix(kpool, np.asarray(block_tables)[b], P + e - s - 1).astype(np.float64)  # [P + n - 1, Hkv, D]
        cv = dequant_prefix(vpool, np.asarray(block_tables)[b], P + e - s - 1).astype(np.float64)
        for i in range(e - s):
            t = s + i
            n_cached = P + i
            for h in range(Hq):
                hk = h // g
                qq = q[t, h].astype(np.float64)
                kk = np.concatenate([ck[:n_cached, hk], k[t, hk][None].astype(np.float64)])
                vv = np.concatenate([cv[:n_cached, hk], v[t, hk][None].astype(np.float64)])
                sc = kk @ qq * scale
                p = np.exp(sc - sc.max())
                out[t, h] = (p / p.sum()) @ vv
    return out
