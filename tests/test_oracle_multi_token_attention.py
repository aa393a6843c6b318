"""CPU: the oracle of multi-token decode attention (oracle/multi_token.py) against the decode oracle it restates (oracle/kv.py): verifying n
draft tokens in one step gives, token for token, what n sequential decode steps give."""
import numpy as np
import pytest

from oracle import kv
from oracle import multi_token as om
from oracle import prefix as op

ROPE = 500000.0
D = 128
# ragged (prefix, draft) pairs: every draft length of the plan (0, 1, 2, 5, 16) and every prefix length (0, 1, 63, 64, 65, 1000)
PREFIX = [0, 1, 63, 64, 65, 1000, 62]
DRAFT = [5, 16, 0, 2, 1, 5, 16]


def _ulp(x):
    a = np.abs(x)
    return np.where(a >= 2.0 ** -14, 2.0 ** (np.floor(np.log2(np.maximum(a, 2.0 ** -14))) - 10), 2.0 ** -24)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("hq,hkv", [(8, 2), (2, 2)])
def test_equals_sequential_decode_oracle(rng, bits, hq, hkv):
    B = len(PREFIX)
    nb = (max(p + n for p, n in zip(PREFIX, DRAFT)) + 63) // 64
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    kp, vp = kv.PagePool(B * nb + 1, hkv, D, bits, rng), kv.PagePool(B * nb + 1, hkv, D, bits, rng)
    kp2, vp2 = kv.PagePool(B * nb + 1, hkv, D, bits), kv.PagePool(B * nb + 1, hkv, D, bits)
    kp2.data[:], vp2.data[:] = kp.data, vp.data
    T = sum(DRAFT)
    cu = np.concatenate([[0], np.cumsum(DRAFT)])
    qkv = rng.standard_normal((T, (hq + 2 * hkv) * D)).astype(np.float16)

    # n sequential decode steps per sequence (the decode oracle rotates and appends the token itself)
    want = np.zeros((T, hq, D), np.float64)
    for b in range(B):
        for i in range(DRAFT[b]):
            t = cu[b] + i
            q = qkv[t, : hq * D].reshape(1, hq, D)
            k = qkv[t, hq * D: (hq + hkv) * D].reshape(1, hkv, D)
            v = qkv[t, (hq + hkv) * D:].reshape(1, hkv, D)
            want[t] = kv.decode_attention(q, k, v, kp, vp, bt[b: b + 1], [PREFIX[b] + i + 1], ROPE, faithful=False)[0]

    # one verify step: append every draft token at its offset, then the multi-token oracle
    mx = max(DRAFT)
    rot = op.prefill_rope_append_at(qkv.copy(), DRAFT, kv.compute_padding_offsets(cu, mx, T), PREFIX, kp2, vp2, bt, hq, hkv, mx, ROPE, 8192)
    q, k, v = rot[:, : hq * D].reshape(T, hq, D), rot[:, hq * D: (hq + hkv) * D].reshape(T, hkv, D), rot[:, (hq + hkv) * D:].reshape(T, hkv, D)
    got = om.multi_token_decode_attention(q, k, v, cu, PREFIX, kp2, vp2, bt)

    assert np.array_equal(kp.data, kp2.data) and np.array_equal(vp.data, vp2.data)  # the same tokens went to the same slots
    assert np.isfinite(got).all()
    # the decode oracle rounds its float64 result to fp16 once: within one fp16 ulp of the float64 verify
    assert (np.abs(got - want) <= _ulp(got)).all(), np.abs(got - want).max()


def test_one_token_is_the_prefix_oracle(rng):
    """With one draft token per sequence the op is a 1-token prompt chunk over the cached prefix (oracle/prefix.py)."""
    hq, hkv, bits = 4, 1, 4
    P = [0, 1, 64, 200]
    B = len(P)
    nb = (max(P) + 1 + 63) // 64
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    kp, vp = kv.PagePool(B * nb + 1, hkv, D, bits, rng), kv.PagePool(B * nb + 1, hkv, D, bits, rng)
    cu = np.arange(B + 1)
    qkv = rng.standard_normal((B, (hq + 2 * hkv) * D)).astype(np.float16)
    rot = op.prefill_rope_append_at(qkv, [1] * B, kv.compute_padding_offsets(cu, 1, B), P, kp, vp, bt, hq, hkv, 1, ROPE, 8192)
    q, k, v = rot[:, : hq * D].reshape(B, hq, D), rot[:, hq * D: (hq + hkv) * D].reshape(B, hkv, D), rot[:, (hq + hkv) * D:].reshape(B, hkv, D)
    got = om.multi_token_decode_attention(q, k, v, cu, P, kp, vp, bt)
    pk = [op.dequant_prefix(kp, bt[b], P[b]) for b in range(B)]
    pv = [op.dequant_prefix(vp, bt[b], P[b]) for b in range(B)]
    assert np.allclose(got, op.prefix_causal_attention(q, k, v, cu, pk, pv), rtol=0, atol=1e-12)
