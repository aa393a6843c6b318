"""Edge-case inputs of the W4A8 / W8A8 GEMM epilogue, their oracle outputs, and a torch restatement of the oracle that runs on the device.

Every builder returns a Case whose oracle output (oracle/w4a8.py) is asserted to contain the edge the case is named for, so a case cannot
quietly stop exercising it:
  * acc_ties        |acc| in [2^24, 2^25) and odd: every such value is a tie of the int -> fp32 conversion (round to nearest even), and the
                    scales are powers of two chosen so that half the columns turn a round-toward-zero conversion into a different fp16;
                    rows of +-127, of -128, and (W8A8) -128 x -128 at K = 14336;
  * fp16_range      outputs rounding to 65504 and overflowing to +-inf, fp16 subnormals, and negative underflow to -0;
  * signed_zero     per-channel t - u cancelling to +0, a -0 product minus +0, and zero rows with ascale = asum = 0 (idle rows);
  * nonfinite       an inf activation scale (what a row with an inf amax quantises to) with acc = 0 (NaN) and acc != 0 (+-inf), and the
                    per-channel inf - inf;
  * level2          per-group level-2 scales 16 / 17 (the edge of 15 s2 <= 255) with zeros 0 / 15, and s2 >= 18, where the 32-bit multiply
                    of four nibble bytes carries into the next byte.

The activation rows of most cases reach a chosen accumulator per column: `_target_codes` sets the column's nibbles so that the row
[127] * (K - 9) + [1] * 9 gives exactly that value.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np

from oracle import w4a8

F16 = np.float16
SMALL = 9  # trailing positions where the target row holds +-1: they carry target % 127 (<= 126 <= 9 * 15)
MODES = ("chn", "grp", "w8")


class Weights(NamedTuple):
    mode: str
    args: tuple                 # the op's arguments after in_feats: chn (qweight, s1, s1z), grp (qweight, s2_zeros, s2_scales, s1), w8 (w, sw)
    w8: np.ndarray              # int8 [N, K]: the weights the kernel multiplies (unpacked nibbles, level-2 dequantised, or the INT8 weight)
    ws: np.ndarray              # fp16 [N]
    wsz: Optional[np.ndarray]   # fp16 [N], per-channel only


class Case(NamedTuple):
    name: str
    wt: Weights
    aq: np.ndarray              # int8 [M, K]
    sa: np.ndarray              # fp16 [M]
    asum: np.ndarray            # fp16 [M] (read by the per-channel epilogue only)
    out: np.ndarray             # fp16 [M, N], the oracle's
    acc: np.ndarray             # int32 [M, N], the oracle's


def weights(mode: str, q: np.ndarray, ws, wsz=None, s2=None, z=None, w=None) -> Weights:
    """Pack uint4 codes q [N, K] (or take the INT8 weight w) as the op takes them.  grp: level-2 scales s2 / zeros z [N, K/128]
    (default 1 / 0, so the weight is q itself)."""
    ws = np.asarray(ws, F16)
    if mode == "chn":
        qw = w4a8.pack_w4(q)
        wsz = np.asarray(wsz, F16)
        return Weights(mode, (qw, ws, wsz), q.astype(np.int8), ws, wsz)
    if mode == "grp":
        N, K = q.shape
        s2 = np.ones((N, K // 128), np.int64) if s2 is None else s2
        z = np.zeros((N, K // 128), np.int64) if z is None else z
        qw, s1, s2s, s2z = w4a8.pack_per_group(q, ws, s2, z)
        return Weights(mode, (qw, s2z, s2s, s1), w4a8.dequant_level2(q, s2s, s2z), ws, None)
    w = np.asarray(q if w is None else w).astype(np.int8)
    return Weights(mode, (w, ws), w, ws, None)


def oracle(wt: Weights, aq, sa, asum):
    """oracle/w4a8.py on these inputs -> (out fp16 [M, N], acc int32 [M, N]); non-finite results are expected, not warned about."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        if wt.mode == "chn":
            qw, s1, s1z = wt.args
            return w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        if wt.mode == "grp":
            qw, s2z, s2s, s1 = wt.args
            return w4a8.gemm_w4a8_per_group(aq, qw, s2z, s2s, s1, sa, return_acc=True)
        w, sw = wt.args
        return w4a8.gemm_w8a8(aq, w, sw, sa, return_acc=True)


def _case(name, wt, aq, sa, asum) -> Case:
    aq = np.asarray(aq, np.int8)
    sa, asum = np.asarray(sa, F16), np.asarray(asum, F16)
    out, acc = oracle(wt, aq, sa, asum)
    return Case(name, wt, aq, sa, asum, out, acc)


def target_row(K: int, sign: int = 1) -> np.ndarray:
    return sign * np.r_[np.full(K - SMALL, 127), np.ones(SMALL)].astype(np.int8)


def _target_codes(targets, K: int) -> np.ndarray:
    """uint4 codes [len(targets), K] with target_row(K) . q[n] == targets[n]: 15s then the remainder, front-loaded in both parts."""
    q = np.zeros((len(targets), K), np.uint8)
    for n, t in enumerate(targets):
        big, small = divmod(int(t), 127)
        for lo, hi, v in ((0, K - SMALL, big), (K - SMALL, K, small)):
            f, r = divmod(v, 15)
            assert f < hi - lo or (f == hi - lo and r == 0), f"target {t} out of reach at K={K}"
            q[n, lo:lo + f] = 15
            if r:
                q[n, lo + f] = r
    assert np.array_equal(q.astype(np.int64) @ target_row(K).astype(np.int64), np.asarray(targets, np.int64))
    return q


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint16)


# ------------------------------------------------------------------------------------------------------------------------------------
# the builders
# ------------------------------------------------------------------------------------------------------------------------------------


def acc_ties(mode: str) -> Case:
    K, N = 14336, 256
    rng = np.random.default_rng(24)
    # columns [0, 128): acc = 8192 (2j + 1) - 1 with 2j + 1 = 3 (mod 4): the fp32 tie rounds up (to nearest even) onto an fp16 midpoint
    # whose upper neighbour is even, so the output is one fp16 step higher than with a truncating conversion.  [128, 256): odd acc.
    sens = [2**24 + 32768 * i + 24575 for i in range(128)]
    odd = [2**24 + 1 + 2 * int(v) for v in rng.integers(0, 5_000_000, N - 128)]
    q = _target_codes(sens + odd, K)
    ws = np.full(N, 2.0**-6)
    w = None
    if mode == "w8":  # two all -128 columns: -128 x -128 over the whole K, |acc| = 128 * 128 * 14327 + 1152 ~ 2.35e8
        w = q.astype(np.int8)
        w[-2:] = -128
    wt = weights(mode, q, ws, wsz=np.zeros(N), w=w)
    mixed = rng.integers(-128, 128, K)
    minus128 = np.r_[np.full(K - SMALL, -128), -np.ones(SMALL)]
    aq = np.stack([target_row(K), target_row(K, -1), minus128, mixed])
    c = _case(f"acc_ties-{mode}", wt, aq, np.full(4, 2.0**-6), np.ones(4))
    a = c.acc.astype(np.int64)
    assert ((np.abs(a) >= 2**24) & (np.abs(a) < 2**25) & (a % 2 == 1)).sum() >= 3 * 128, "odd accumulators in [2^24, 2^25)"
    assert (aq == -128).any() and (np.abs(aq) == 127).any()
    assert not np.array_equal(_bits(restated_out(c, rz=True)), _bits(c.out)), "a truncating int -> fp32 conversion must change the output"
    if mode == "w8":
        assert np.abs(a).max() > 2.3e8
    return c


def fp16_range(mode: str) -> Case:
    K, N = 384, 256  # K % 256 == 128: the last pipeline stage is half zero-filled
    # columns [0, 128): ws = 1, acc 65440 .. 65567 at scale 1: below 65504, rounding to 65504, and from 65520 on +inf
    # columns [128, 256): ws = 2^-12, acc 0 .. 127 -> fp16 subnormals at ascale 0.75 * 2^-12, underflow to -0 at ascale 2^-14
    q = _target_codes(list(range(65440, 65568)) + list(range(128)), K)
    ws = np.r_[np.ones(128), np.full(128, 2.0**-12)]
    wt = weights(mode, q, ws, wsz=np.zeros(N))
    aq = np.stack([target_row(K), target_row(K, -1), target_row(K), target_row(K, -1), target_row(K, -1)])
    sa = [1.0, 1.0, 0.75 * 2.0**-12, 0.75 * 2.0**-12, 2.0**-14]
    c = _case(f"fp16_range-{mode}", wt, aq, sa, np.ones(5))
    b = _bits(c.out)
    assert (b == 0x7BFF).any() and (b == 0xFBFF).any(), "65504 and -65504"
    assert (b == 0x7C00).any() and (b == 0xFC00).any(), "+inf and -inf"
    sub = ((b & 0x7C00) == 0) & ((b & 0x3FF) != 0)
    assert (sub & (b < 0x8000)).any() and (sub & (b >= 0x8000)).any(), "positive and negative subnormals"
    assert (b == 0x8000).any(), "-0 by underflow"
    return c


def signed_zero(mode: str) -> Case:
    K, N = 256, 128
    # columns [0, 64): ws = 1, per-channel s1z = acc of the target row, so t - u cancels exactly to +0; columns [64, 128): ws = -1 with
    # s1z >= 0, so a zero row (codes, ascale and asum all 0, as idle rows are) gives t = -0 and t - u = -0 - +0 = -0
    t = list(range(1000, 1064)) * 2
    q = _target_codes(t, K)
    wt = weights(mode, q, np.r_[np.ones(64), -np.ones(64)], wsz=np.asarray(t, np.float64))
    aq = np.stack([target_row(K), np.zeros(K), np.zeros(K), target_row(K, -1)])
    c = _case(f"signed_zero-{mode}", wt, aq, [1.0, 0.0, 0.0, 1.0], [1.0, 0.0, 0.0, -1.0])
    b = _bits(c.out)
    assert (b[1:3] & 0x7FFF == 0).all(), "zero rows give zeros"
    assert (b[1:3, :64] == 0).all() and (b[1:3, 64:] == 0x8000).all(), "+0 and -0"
    if mode == "chn":
        assert (b[0, :64] == 0).all() and (c.acc[0, :64] != 0).all(), "t - u cancels to +0"
        assert (b[3, :64] == 0).all(), "-t - -u cancels to +0"
    return c


def nonfinite(mode: str) -> Case:
    K, N = 256, 128
    rng = np.random.default_rng(7)
    q = rng.integers(0, 16, (N, K), dtype=np.uint8)
    q[:, 0] = 15  # no column sums to 0 against a non-negative row
    s1 = rng.uniform(0.005, 0.02, N).astype(F16)
    wt = weights(mode, q, s1, wsz=(rng.integers(1, 16, N) * s1.astype(np.float32)).astype(F16))
    pos = rng.integers(1, 128, K)
    # a row with an inf amax quantises to inf scale and sum; its codes are 0 (inf * 0 is NaN, cvt NaN -> 0) or, with a finite
    # element beside it, whatever the producer wrote: the kernel must give NaN for acc = 0 and +-inf (chn: inf - inf = NaN) otherwise
    aq = np.stack([np.zeros(K), pos, pos, -pos, rng.integers(-128, 128, K)])
    inf = np.inf
    c = _case(f"nonfinite-{mode}", wt, aq, [inf, inf, inf, inf, 0.01], [inf, 0.0, inf, inf, 3.0])
    o = c.out.astype(np.float32)
    assert np.isnan(o[0]).all(), "acc = 0 times an inf scale"
    assert np.isposinf(o[1]).all() and np.isneginf(o[3]).all(), "+inf and -inf"
    if mode == "chn":
        assert np.isnan(o[2]).all() and (c.acc[2] != 0).all(), "inf - inf"
    assert np.isfinite(o[4]).all()
    return c


def level2() -> Case:
    K, N = 384, 128
    rng = np.random.default_rng(17)
    q = rng.integers(0, 16, (N, K), dtype=np.uint8)
    q[:, ::7] = 15  # every 4-k word of a group holds a 15 now and then: 15 s2 > 255 carries for s2 >= 18
    s2 = rng.choice([16, 17, 18, 19, 31, 64, 128, 255], size=(N, K // 128))
    s2[:16] = 16
    s2[16:32] = 17
    z = rng.choice([0, 15], size=(N, K // 128))
    wt = weights("grp", q, rng.uniform(0.0005, 0.002, N), s2=s2, z=z)
    aq = rng.integers(-128, 128, (8, K))
    c = _case("level2-grp", wt, aq, rng.uniform(0.005, 0.02, 8), np.zeros(8))
    # the byte-wise product (no carries) differs from the 32-bit multiply the kernel does: the case depends on the carries
    qw, s2z, s2s, _ = wt.args
    s2c = w4a8.unshuffle_n32(s2s.view(np.uint8).astype(np.int64)).T.repeat(128, axis=1)
    z2c = w4a8.unshuffle_n32(s2z.view(np.uint8).astype(np.int64)).T.repeat(128, axis=1)
    bytewise = ((q.astype(np.int64) * s2c + z2c) & 0xFF).astype(np.uint8).view(np.int8)
    assert not np.array_equal(bytewise, wt.w8), "carries across nibble bytes"
    assert np.array_equal(bytewise[:32], wt.w8[:32]), "s2 <= 17 never carries"
    for s in (16, 17):
        for zz in (0, 15):
            assert ((s2 == s) & (z == zz)).any(), (s, zz)
    return c


CASE_NAMES = [f"{e}-{m}" for e in ("acc_ties", "fp16_range", "signed_zero", "nonfinite") for m in MODES] + ["level2-grp"]


def build(name: str) -> Case:
    """The case called `name` (one of CASE_NAMES)."""
    edge, mode = name.rsplit("-", 1)
    return level2() if edge == "level2" else globals()[edge](mode)


# ------------------------------------------------------------------------------------------------------------------------------------
# torch restatement of the oracle (any device): exact INT accumulators in float64, the oracle's fp32 epilogue op by op
# ------------------------------------------------------------------------------------------------------------------------------------


def restated(mode, aq, w8, ws, wsz, sa, asum, rz: bool = False):
    """torch tensors aq int8 [M, K], w8 int8 [N, K], fp16 scales -> (out fp16 [M, N], acc float64 [M, N]).  The float64 matmul of integers
    is exact (|acc| < 2^53); the int -> fp32 conversion rounds to nearest even (rz=True: toward zero, to show a case depends on it); every
    fp32 operation is its own rounded torch op, in the order of oracle/w4a8.py."""
    import torch

    acc = aq.double() @ w8.double().T
    ps = acc.float()
    if rz:
        ps = torch.where(ps.double().abs() > acc.abs(), torch.nextafter(ps, torch.zeros_like(ps)), ps)
    ws, sa = ws.float()[None, :], sa.float()[:, None]
    if mode == "chn":
        t = ps * ws
        t = t * sa
        u = wsz.float()[None, :] * asum.float()[:, None]
        return (t - u).half(), acc
    return (ps * (ws * sa)).half(), acc


def restated_out(c: Case, rz: bool = False) -> np.ndarray:
    import torch

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    wsz = t(c.wt.wsz) if c.wt.wsz is not None else None
    return restated(c.wt.mode, t(c.aq), t(c.wt.w8), t(c.wt.ws), wsz, t(c.sa), t(c.asum), rz)[0].numpy()


def same_bits(out, ref) -> bool:
    """fp16 arrays equal bit for bit, except that a NaN only has to be a NaN (cvt.rn.f16.f32 and numpy give different NaN payloads)."""
    out, ref = np.asarray(out, F16), np.asarray(ref, F16)
    nan = np.isnan(ref)
    return bool(np.array_equal(np.isnan(out), nan) and np.array_equal(_bits(out)[~nan], _bits(ref)[~nan]))
