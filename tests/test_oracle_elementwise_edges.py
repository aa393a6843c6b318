"""CPU: the elementwise oracle (oracle/ops.py) on hand-worked edge rows -- the inputs where a quantiser's amax, its division and
its row sum go wrong: a zero row, NaN and inf elements, a one-hot negative maximum, and the fp16 rounding of the per-tensor norm."""
import numpy as np

from oracle import ops

INF, NAN = np.float16(np.inf), np.float16(np.nan)


def _row(*v):
    return np.array([v], dtype=np.float16)


def test_zero_row_gives_zero_scale_and_zero_codes():
    q, s, m = ops.quant_per_token(np.zeros((1, 16), np.float16))
    # amax = 0: scale = half(0/127) = 0, and 0 * (127/0) = NaN, which cvt.rni.sat turns into 0
    assert s[0] == 0 and not np.signbit(s[0]) and m[0] == 0
    assert np.array_equal(q, np.zeros((1, 16), np.int8))


def test_nan_element_is_ignored_by_amax():
    q, s, m = ops.quant_per_token(_row(1.0, NAN, -2.0, 0.5, 0, 0, 0, 0))
    assert s[0] == np.float16(np.float32(2.0) / np.float32(127.0))
    assert list(q[0]) == [64, 0, -127, 32, 0, 0, 0, 0]  # 1 * 127/2 = 63.5 rounds to even 64; NaN quantises to 0
    assert np.isnan(m[0])  # ... but the row sum is an IEEE sum: NaN


def test_nonfinite_row_sums_follow_ieee():
    _, s, m = ops.quant_per_token(_row(INF, 1.0, 2.0, 0, 0, 0, 0, 0))
    assert m[0] == np.inf and s[0] == np.inf
    _, _, m = ops.quant_per_token(_row(INF, INF, 1.0, 0, 0, 0, 0, 0))
    assert m[0] == np.inf
    _, _, m = ops.quant_per_token(_row(-INF, -INF, 1.0, 0, 0, 0, 0, 0))
    assert m[0] == -np.inf
    _, _, m = ops.quant_per_token(_row(INF, -INF, 1.0, 0, 0, 0, 0, 0))
    assert np.isnan(m[0])


def test_inf_row_quantises_every_code_to_zero():
    q, s, _ = ops.quant_per_token(_row(INF, 1.0, -65504.0, 3.0, 0, 0, 0, 0))
    # tmp = 127/inf = 0: finite * 0 = 0 and inf * 0 = NaN -> 0
    assert s[0] == np.inf and np.array_equal(q, np.zeros((1, 8), np.int8))


def test_finite_sum_overflowing_fp16_is_inf():
    _, _, m = ops.quant_per_token(_row(65504.0, 65504.0, 0, 0, 0, 0, 0, 0))
    assert m[0] == np.inf


def test_one_hot_negative_maximum_is_minus_127_never_minus_128():
    x = np.zeros((1, 64), np.float16)
    x[0, 5] = -2000.0
    x[0, 9] = 3.0
    q, s, m = ops.quant_per_token(x)
    assert q[0, 5] == -127 and q[0, 9] == 0 and int(q.min()) == -127  # 3 * 127/2000 = 0.19
    assert s[0] == np.float16(np.float32(2000.0) / np.float32(127.0)) and m[0] == np.float16(-1997.0)
    x[0, 5] = -65504.0
    q, _, _ = ops.quant_per_token(x)
    assert q[0, 5] == -127 and int(q.min()) == -127


def test_subnormal_row():
    x = (np.array([[1, -3, 7, 0, 2, -1, 5, 4]]) * 2.0 ** -24).astype(np.float16)
    q, s, m = ops.quant_per_token(x)
    assert list(q[0]) == [18, -54, 127, 0, 36, -18, 91, 73]  # k * 127/7 rounded
    assert s[0] == np.float16(7 * 2.0 ** -24 / 127) and m[0] == np.float16(15 * 2.0 ** -24)


def test_quant_given_amax():
    x = _row(1.0, -2.0, 0.25, 0, 0, 0, 0, 0)
    # with the row's own amax it is quant_per_token
    for a, b in zip(ops.quant_given_amax(x, np.array([2.0], np.float32)), ops.quant_per_token(x)):
        assert np.array_equal(a, b)
    # with a larger amax from another shard: codes and scale follow that amax, the sum stays this row's own
    q, s, m = ops.quant_given_amax(x, np.array([4.0], np.float32))
    assert list(q[0]) == [32, -64, 8, 0, 0, 0, 0, 0] and s[0] == np.float16(np.float32(4.0) / np.float32(127.0)) and m[0] == np.float16(-0.75)
    q, _, m = ops.quant_given_amax(x, np.array([4.0], np.float32), fuse_sum=False)
    assert m is None and q[0, 1] == -64


def test_per_tensor_norm_quantises_half_y():
    # x = (4, -4, ...): mean 0, var = 16, y = +-1.5 * rsqrt(1 + eps/16) = +-1.4999995 in fp32, and half(y) = +-1.5.
    # With scale 1: half(y) * 1 = 1.5 rounds to even 2, while the fp32 y would give 1.
    x = np.array([[4.0, -4.0] * 4], np.float16)
    q, y = ops.layernorm_general_quant_per_tensor(x, np.full(8, 1.5, np.float16), 1e-5, np.float16(1.0))
    assert np.all(np.abs(y) < 1.5) and np.all(np.abs(y.astype(np.float16)) == 1.5)
    assert list(q[0]) == [2, -2] * 4


def test_per_tensor_norm_matches_per_token_statistics():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((4, 256)) * 2 + 0.5).astype(np.float16)
    gamma = (1 + 0.1 * rng.standard_normal(256)).astype(np.float16)
    _, _, _, y_tok = ops.layernorm_general_quant(x, gamma, 1e-5, False)
    q, y = ops.layernorm_general_quant_per_tensor(x, gamma, 1e-5, np.float16(20.0))
    assert np.array_equal(y, y_tok)
    assert np.array_equal(q, ops.cvt_rni_sat_s8(y.astype(np.float16).astype(np.float32) * np.float32(20.0)))


def test_norm_constant_row_is_clamped_amax():
    x = np.full((1, 64), 0.75, np.float16)
    q, s, m, y = ops.layernorm_general_quant(x, np.ones(64, np.float16), 1e-5)
    assert not np.any(y) and not np.any(q) and m[0] == 0
    assert s[0] == np.float16(np.float32(np.float16(1e-6)) / np.float32(127.0))


def test_dequant_silu_and_mul_quant_per_token():
    acc = np.array([[0, 0, 0, 0, 0, 0, 0, 0],          # zero row
                    [1000, -1000, 0, 5, 2000, 2000, 7, 3]], np.int32)
    q, so, t = ops.dequant_silu_and_mul_quant_per_token(acc, 1e-3, 2e-3)
    assert so.dtype == np.float32 and t.dtype == np.float32 and so[0] == 0 and not np.any(q[0]) and not np.any(t[0])
    x = np.float32(1000) * np.float32(1e-3)
    silu1 = np.float32(x / (np.float32(1) + np.exp(-x, dtype=np.float32)))
    assert t[1, 0] == np.float32(silu1 * np.float32(np.float32(2000) * np.float32(2e-3)))
    amax = np.abs(t[1]).max()
    assert so[1] == np.float32(amax / np.float32(127)) and abs(int(q[1, np.argmax(np.abs(t[1]))])) == 127
    assert np.array_equal(q[1], ops.cvt_rni_sat_s8((np.float32(127) / amax) * t[1]))
