"""CPU: the oracle of prompt chunks over a cached prefix (oracle/prefix.py) against the oracles it builds on (oracle/kv.py,
oracle/prefill_attention.py)."""
import numpy as np

from oracle import kv
from oracle import prefill_attention as o
from oracle import prefix as op

ROPE = 500000.0


def test_empty_prefix_is_causal_varlen_attention(rng):
    lens, hq, hkv = [7, 1, 0, 33], 4, 2
    T = sum(lens)
    q, k, v = (rng.standard_normal((T, h, 128)).astype(np.float16) for h in (hq, hkv, hkv))
    cu = np.concatenate([[0], np.cumsum(lens)])
    empty = [np.zeros((0, hkv, 128), np.float16)] * len(lens)
    got = op.prefix_causal_attention(q, k, v, cu, empty, empty)
    assert np.allclose(got, o.causal_varlen_attention(q, k, v, cu), rtol=0, atol=1e-12)


def _chunked_vs_oneshot(rng, bits, lens, split):
    Hq, Hkv, D = 4, 2, 128
    B = len(lens)
    max_blocks = (max(lens) + 63) // 64
    bt = np.arange(B * max_blocks).reshape(B, max_blocks)
    qkv = rng.standard_normal((sum(lens), (Hq + 2 * Hkv) * D)).astype(np.float16)
    # one shot
    kp1, vp1 = kv.PagePool(B * max_blocks, Hkv, D, bits), kv.PagePool(B * max_blocks, Hkv, D, bits)
    cu = np.concatenate([[0], np.cumsum(lens)])
    one = kv.prefill_rope_append(qkv.copy(), lens, kv.compute_padding_offsets(cu, max(lens), sum(lens)), kp1, vp1, bt, Hq, Hkv, max(lens), ROPE, 8192)
    # two chunks: the first min(split, len) tokens, then the rest behind start_pos
    kp2, vp2 = kv.PagePool(B * max_blocks, Hkv, D, bits), kv.PagePool(B * max_blocks, Hkv, D, bits)
    a = [min(split, L) for L in lens]
    rest = [L - x for L, x in zip(lens, a)]
    rows_a = np.concatenate([np.arange(cu[b], cu[b] + a[b]) for b in range(B)])
    rows_b = np.concatenate([np.arange(cu[b] + a[b], cu[b + 1]) for b in range(B)])
    cua, cub = np.concatenate([[0], np.cumsum(a)]), np.concatenate([[0], np.cumsum(rest)])
    qa = op.prefill_rope_append_at(qkv[rows_a].copy(), a, kv.compute_padding_offsets(cua, max(max(a), 1), sum(a)), [0] * B, kp2, vp2, bt, Hq,
                                   Hkv, max(max(a), 1), ROPE, 8192)
    qb = op.prefill_rope_append_at(qkv[rows_b].copy(), rest, kv.compute_padding_offsets(cub, max(max(rest), 1), sum(rest)), a, kp2, vp2, bt, Hq,
                                   Hkv, max(max(rest), 1), ROPE, 8192)
    two = np.empty_like(one)
    two[rows_a], two[rows_b] = qa, qb
    return one, two, kp1, vp1, kp2, vp2


def test_start_pos_two_chunks_equal_one_shot(rng):
    for bits in (4, 8):
        for split in (1, 64, 65):
            one, two, kp1, vp1, kp2, vp2 = _chunked_vs_oneshot(rng, bits, [70, 130, 3], split)
            assert np.array_equal(one.view(np.uint16), two.view(np.uint16))
            assert np.array_equal(kp1.data, kp2.data) and np.array_equal(vp1.data, vp2.data)


def test_zero_start_pos_is_prefill_rope_append(rng):
    lens = [5, 70]
    Hq, Hkv, D = 4, 2, 128
    qkv = rng.standard_normal((sum(lens), (Hq + 2 * Hkv) * D)).astype(np.float16)
    cu = np.concatenate([[0], np.cumsum(lens)])
    pad = kv.compute_padding_offsets(cu, 70, sum(lens))
    bt = np.arange(4).reshape(2, 2)
    pools = [kv.PagePool(4, Hkv, D, 4) for _ in range(4)]
    a = kv.prefill_rope_append(qkv.copy(), lens, pad, pools[0], pools[1], bt, Hq, Hkv, 70, ROPE, 8192)
    b = op.prefill_rope_append_at(qkv.copy(), lens, pad, [0, 0], pools[2], pools[3], bt, Hq, Hkv, 70, ROPE, 8192)
    assert np.array_equal(a.view(np.uint16), b.view(np.uint16)) and np.array_equal(pools[0].data, pools[2].data)


def test_one_token_chunk_matches_decode_oracle(rng):
    """A 1-token chunk over a cached prefix is a decode step: append it at start_pos = P, then attend over the dequantised prefix and the
    un-quantised token; the float64 decode oracle (faithful=False) computes the same thing."""
    for bits in (4, 8):
        Hq, Hkv, D = 8, 2, 128
        P = [0, 1, 63, 64, 130]
        B = len(P)
        max_blocks = (max(P) + 1 + 63) // 64
        kp, vp = kv.PagePool(B * max_blocks + 1, Hkv, D, bits, rng), kv.PagePool(B * max_blocks + 1, Hkv, D, bits, rng)
        bt = 1 + np.arange(B * max_blocks).reshape(B, max_blocks)
        q, k, v = (rng.standard_normal((B, h, D)).astype(np.float16) for h in (Hq, Hkv, Hkv))
        kp2, vp2 = kv.PagePool(kp.data.shape[0], Hkv, D, bits), kv.PagePool(vp.data.shape[0], Hkv, D, bits)
        kp2.data[:], vp2.data[:] = kp.data, vp.data
        want = kv.decode_attention(q, k, v, kp, vp, bt, [p + 1 for p in P], ROPE, faithful=False).astype(np.float64)
        qkv = np.concatenate([q.reshape(B, -1), k.reshape(B, -1), v.reshape(B, -1)], axis=1)
        cu = np.arange(B + 1)
        qkv = op.prefill_rope_append_at(qkv, [1] * B, kv.compute_padding_offsets(cu, 1, B), P, kp2, vp2, bt, Hq, Hkv, 1, ROPE, 8192)
        pk = [op.dequant_prefix(kp2, bt[b], P[b]) for b in range(B)]
        pv = [op.dequant_prefix(vp2, bt[b], P[b]) for b in range(B)]
        qr, kr, vr = qkv[:, : Hq * D].reshape(B, Hq, D), qkv[:, Hq * D: (Hq + Hkv) * D].reshape(B, Hkv, D), qkv[:, (Hq + Hkv) * D:].reshape(B, Hkv, D)
        got = op.prefix_causal_attention(qr, kr, vr, cu, pk, pv)
        assert np.array_equal(kp.data, kp2.data) and np.array_equal(vp.data, vp2.data)  # the same token was appended at the same slot
        assert np.abs(got - want).max() <= 3e-3 * max(1.0, np.abs(want).max())
