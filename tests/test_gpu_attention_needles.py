"""GPU: the paged-attention kernels on needle caches (oracle/needles.py), where one wrong token, scale, zero point, split or mask bit
moves the output by O(1) instead of by |v| / L.

Kernels: single_query_attention (decode, and the fused-quant form bit-equal to quantising its output), multi_token_decode_attention with
a causal chain (C = 8 and C = 16 columns per CTA) and with a tree mask, and prefix_prefill_attention.  Sweeps give every (sequence, kv head)
its own needle and repeat the launch until every cached position, the new token and the draft / chunk rows included, has held one.  Slots
the kernel must not read hold NaN scales.

Bar, per element (derivation in oracle/needles.py `exact`):
    |out - exact| <= 2 ulp16(|exact|) + 2^-11 sum_t p_t v_op_t + n_acc 2^-23 sum_t p_t acc_mag_t + 2.2 delta sum_t p_t |v_t - exact|
the fp16 output rounding, the fp16 rounding of P (times the V operand) before the PV MMA, the fp32 accumulation of the biased V operands,
and the logit error delta (QK MMA accumulation on biased K codes, RoPE of the decode query by numpy, ex2.approx) through the softmax
weights.  On needle inputs it is about 4e-3 to 1e-2, against O(1) for a wrong read (test_oracle_attention_needles.py).
"""
import numpy as np
import pytest
import torch

from oracle import needles as nd
from oracle.kv import PagePool
from tests.util import GpuPool, kv_pointer_table, np_of, to_dev

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128


def _ratio(got, want, bar, what):
    got = np.asarray(got, np.float64)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    r = np.abs(got - want) / bar
    assert r.max() <= 1.0, f"{what}: err / bar = {r.max():.3f} at {np.unravel_index(r.argmax(), r.shape)}"
    return float(r.max())


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _decode_check(c, out, what):
    """_ratio for a decode launch; a failure names the token whose V the worst output row is closest to."""
    want, bar = c.exact()
    r = np.abs(np.asarray(out, np.float64) - want) / bar
    if np.isfinite(out).all() and r.max() > 1.0:
        b, h, _ = np.unravel_index(r.argmax(), r.shape)
        hk = h // c.G
        _, vd, _, _ = nd.cached_rows(c.kp, c.vp, c.bt[b], c.lens[b] - 1, hk)
        rows = np.concatenate([vd, c.v[b, hk][None].astype(np.float64)])
        near = int(np.abs(rows - np.asarray(out[b, h], np.float64)).max(axis=1).argmin())
        what += f" (sequence {b}, head {h}: output closest to token {near}'s V; needle at {c.needles.get((b, hk))})"
    return _ratio(out, want, bar, what)


def _report(name, worst):
    print(f"\nNEEDLE-RATIO {name} {worst:.4f}")


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------------------
DECODE = [  # (B, Hq, Hkv, lens)
    (2, 64, 64, [2048, 1985]),  # G = 1; L mod 64 = 0 / 1, mod 32 = 0 / 1; context splits
    (2, 32, 8, [1087, 96]),     # G = 4; L mod 64 = 63, mod 32 = 31 / 0; context splits at small batch
    (2, 64, 4, [575, 33]),      # G = 16 (two head groups per kv head); L mod 64 = 63 / 33, mod 32 = 31 / 1
]


def _decode(dev, c, fused=False):
    import qserve_backend.fused_attention as fa
    from qserve_b200 import backend as ext
    gk, gv = GpuPool(c.kp, dev), GpuPool(c.vp, dev)
    table = kv_pointer_table(gk, gv, c.bt, dev)
    qd, kd, vd = to_dev(c.q, dev), to_dev(c.k, dev), to_dev(c.v, dev)
    lens = torch.tensor(c.lens, dtype=torch.int32, device=dev)
    args = (8192, 64, c.hkv * D * c.bits // 8, max(c.lens), D, ROPE)
    if fused:
        oq = torch.empty((c.B, c.hq * D), dtype=torch.int8, device=dev)
        sc = torch.empty(c.B, dtype=torch.half, device=dev)
        sm = torch.empty(c.B, dtype=torch.half, device=dev)
        ext.single_query_attention_quant(qd, kd, vd, table, lens, *args, c.bits == 4, True, oq, sc, sm)
        return oq, sc, sm
    return fa.single_query_attention(qd, kd, vd, table, lens, None, *args, True, c.bits == 4, True)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode_needle_sweep(dev, bits, B, Hq, Hkv, lens):
    assert nd.decode_splits(B, Hq, Hkv, max(lens), _sms(dev)) > 1  # every configuration is chosen to plan context splits on an H100
    worst = 0.0
    for r, needles in enumerate(nd.sweep(lens, Hkv)):
        c = nd.DecodeCase(1000 * bits + r, B, Hq, Hkv, lens, bits, needles)
        worst = max(worst, _decode_check(c, np_of(_decode(dev, c)), f"launch {r}"))
    _report(f"decode kv{bits} {B}x{Hq}/{Hkv} {lens}", worst)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode_two_needles(dev, bits, B, Hq, Hkv, lens):
    """Two needles ln 3 apart on each side of a split boundary, of a page boundary and of a 32-token slice boundary, and an old needle
    with the new token: a wrong running-max rescale or merge weight changes the 3:1 mix by O(|v|)."""
    nsplit = nd.decode_splits(B, Hq, Hkv, max(lens), _sms(dev))
    worst = 0.0
    for r in range(4):
        first, second = {}, {}
        for b, L in enumerate(lens):
            pps = -(-((L - 1 + 63) // 64) // nsplit)
            edge = [pps * 64 if nsplit > 1 else 64, 64, 32, 0][r]
            if r < 3 and edge >= L - 1:
                continue
            for hk in range(Hkv):
                t1, t2 = (edge - 1 - hk % 3, edge + hk % 3) if r < 3 else (hk % (L - 1) if L > 1 else 0, L - 1)
                if t1 < 0 or t2 >= L or t1 == t2:
                    continue
                if r < 3:
                    assert nsplit == 1 or r > 0 or nd.split_of(t1, L - 1, nsplit) != nd.split_of(t2, L - 1, nsplit)
                first[(b, hk)], second[(b, hk)] = t1, (t2, float(np.log(3)))
        c = nd.DecodeCase(500 + r, B, Hq, Hkv, lens, bits, first, second)
        worst = max(worst, _decode_check(c, np_of(_decode(dev, c)), f"edge kind {r}"))
    _report(f"decode-two kv{bits} {lens}", worst)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode_quant_is_quantised_decode_on_needles(dev, bits, B, Hq, Hkv, lens):
    """The fused-quant form equals invoke_quant_fuse_sum of the unfused output, bit for bit: on the sweep launch that puts the needles on
    the new tokens and on one in the middle of the cache."""
    import qserve_backend.fused_kernels as fk
    sweeps = nd.sweep(lens, Hkv)
    for r in (len(sweeps) // 2, (min(lens) - 1) // Hkv):
        c = nd.DecodeCase(77 + r, B, Hq, Hkv, lens, bits, {**sweeps[r], **{(b, hk): L - 1 for b, L in enumerate(lens) for hk in range(0, Hkv, 2)}})
        out = _decode(dev, c).reshape(B, -1).contiguous()
        q1 = torch.empty((B, Hq * D), dtype=torch.int8, device=dev)
        s1, m1 = torch.empty(B, dtype=torch.half, device=dev), torch.empty(B, dtype=torch.half, device=dev)
        fk.invoke_quant_fuse_sum(q1, out, m1, s1)
        q2, s2, m2 = _decode(dev, c, fused=True)
        torch.cuda.synchronize()
        assert torch.equal(q1, q2) and torch.equal(s1, s2) and torch.equal(m1, m2)


# ---------------------------------------------------------------------------------------------------------------------------------
# chain / tree verify and prefix prefill
# ---------------------------------------------------------------------------------------------------------------------------------
def _run_chunk(dev, c):
    """Upload the pools, append the rows with the op, run the attention op; -> (out, exact, bar)."""
    from qserve_b200 import backend
    gk, gv = GpuPool(c.kp, dev), GpuPool(c.vp, dev)
    table = kv_pointer_table(gk, gv, c.bt, dev)
    spt = c.hkv * D * c.bits // 8
    T = c.qkv.shape[0]
    qkv = to_dev(c.qkv, dev)
    cu = to_dev(c.cu, dev)
    prefix = torch.tensor(c.P, dtype=torch.int32, device=dev)
    lens = torch.tensor(c.N, dtype=torch.int32, device=dev)
    max_n = max(c.N)
    pad = backend.compute_padding_offsets(cu, max_n, T)
    kw = {}
    if c.kind == "tree":
        kw["tree_mask"] = to_dev(np.concatenate([np.asarray(m, np.int64) for m in c.masks]).astype(np.int32), dev)
    backend.apply_bias_rope_update_kv_cache_at(qkv, lens, pad, prefix, table, c.hq, c.hkv, max_n, 64, spt, D, ROPE, 8192, True, c.bits == 4, True,
                                               **kw)
    q, k, v = qkv.split([c.hq * D, c.hkv * D, c.hkv * D], dim=-1)
    q, k, v = q.reshape(T, c.hq, D), k.reshape(T, c.hkv, D), v.reshape(T, c.hkv, D)
    if c.kind == "prefix":
        out = backend.prefix_prefill_attention(q, k, v, cu, max_n, prefix, max(c.P), table, 64, spt, c.bits == 4)
    else:
        out = backend.multi_token_decode_attention(q, k, v, cu, max_n, prefix, max(c.P), table, 64, spt, c.bits == 4, **kw)
    torch.cuda.synchronize()
    kp = PagePool(c.kp.data.shape[0], c.hkv, D, c.bits); kp.data[:] = gk.download()
    vp = PagePool(c.vp.data.shape[0], c.hkv, D, c.bits); vp.data[:] = gv.download()
    want, bar = c.exact(np_of(q), np_of(k), np_of(v), kp, vp)
    return np_of(out), want, bar


def _chunk_sweep(dev, kind, P, N, hq, hkv, bits, masks=None, logit=nd.NEEDLE_LOGIT, seed=0):
    """Needles over every cache position 0 .. P_b + n_b - 1 (prefix and rows) of every sequence, one per (sequence, kv head) per launch."""
    ends = [p + n for p, n in zip(P, N)]
    worst = 0.0
    for r, needles in enumerate(nd.sweep(ends, hkv)):
        c = nd.ChunkCase(seed + r, kind, P, N, hq, hkv, bits, needles, masks=masks, logit=logit)
        out, want, bar = _run_chunk(dev, c)
        worst = max(worst, _ratio(out, want, bar, f"{kind} launch {r}"))
    return worst


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("P,N,hq,hkv", [
    ([700, 1, 64], [2, 1, 2], 32, 8),       # G x n <= 8: one n8 tile (C = 8); context splits
    ([1000, 63], [16, 16], 32, 8),          # C = 16, four column parts, splits
    ([127, 5], [1, 16], 8, 8),              # G = 1, draft length 1 and 16
])
def test_chain_verify_needle_sweep(dev, bits, P, N, hq, hkv):
    worst = _chunk_sweep(dev, "chain", P, N, hq, hkv, bits, seed=100 * bits)
    _report(f"chain kv{bits} P={P} N={N} {hq}/{hkv}", worst)


@pytest.mark.parametrize("bits", [4, 8])
def test_tree_verify_needle_sweep(dev, bits):
    """Every node and prefix position holds a needle with a logit of +16 for EVERY node of the tree: it dominates its descendants, and a
    sibling or cousin must not see it at all (the oracle masks it)."""
    from tests.test_gpu_tree_verify import tree
    masks = [tree("binary"), tree("random", 16, seed=4), tree("medusa")]
    worst = _chunk_sweep(dev, "tree", [300, 64, 1], [len(m) for m in masks], 8, 2, bits, masks=masks, logit=16.0, seed=200 * bits)
    _report(f"tree kv{bits}", worst)


@pytest.mark.parametrize("bits", [4, 8])
def test_prefix_prefill_needle_sweep(dev, bits):
    """Needles over the whole prefix (128-key block edges, the last prefix slot) and the chunk rows (64-row query blocks, the prefix /
    chunk seam of the mask)."""
    worst = _chunk_sweep(dev, "prefix", [191, 128, 1], [66, 64, 130], 16, 8, bits, seed=300 * bits)
    _report(f"prefix kv{bits}", worst)


# ---------------------------------------------------------------------------------------------------------------------------------
# outlier magnitudes: K channels of 20 to 50, KV4 K scales of about 1 to 4, |q| up to 10, a peaked softmax
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE[:2])
def test_decode_outlier_keys(dev, bits, B, Hq, Hkv, lens):
    """The biased-code QK MMAs at LLM key magnitudes: the k_mma term of the bar (oracle/needles.py `exact`) carries the accumulation error
    of 1024 + u (1024 + 16 u) times q through the softmax weights."""
    worst = 0.0
    for r in range(3):
        c = nd.with_outliers(nd.DecodeCase(40 + r, B, Hq, Hkv, lens, bits, {}), 60 + r)
        worst = max(worst, _decode_check(c, np_of(_decode(dev, c)), f"outliers {r}"))
    _report(f"decode-outliers kv{bits} {lens}", worst)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("P,N,hq,hkv", [([700, 1, 64], [2, 1, 2], 32, 8), ([1000, 63], [16, 16], 32, 8)])
def test_chain_verify_outlier_keys(dev, bits, P, N, hq, hkv):
    worst = 0.0
    for r in range(2):
        c = nd.with_outliers(nd.ChunkCase(80 + r, "chain", P, N, hq, hkv, bits, {}), 90 + r)
        out, want, bar = _run_chunk(dev, c)
        worst = max(worst, _ratio(out, want, bar, f"outliers {r}"))
    _report(f"chain-outliers kv{bits} P={P} N={N}", worst)
