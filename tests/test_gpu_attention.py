"""GPU parity: KV4 / KV8 paged decode attention, prefill RoPE+append and padding offsets vs the CPU oracle.

Stated tolerances (floating point, SURVEY.md 8c: the reference itself is order dependent here)
  * attention output: max |out - exact| <= 3e-3 * max(1, max|out|), where `exact` is the float64 attention over the
    same quantised cache (oracle faithful=False); the reference-faithful oracle (fp16 partial dots, fp16 logits,
    fp16 tree reduction of the output) is itself only within 1e-2 of `exact` (measured: 7e-3 with KV8), and our kernel
    may not be further from `exact` than 1.5x the faithful oracle plus 1e-3.
  * V pages (no RoPE, pure IEEE arithmetic): codes, scales and zeros bit-exact.
  * K pages: RoPE uses sincosf/powf whose last fp32 bit differs from numpy's; scales / zeros within 1 fp16 ulp and
    codes within 1 LSB, with at most 3% of the codes of a token differing.
"""
import os

import numpy as np
import pytest
import torch

from oracle import kv
from tests.util import GpuPool, bits16, kv_pointer_table, np_of, to_dev, ulp16_diff

pytestmark = pytest.mark.gpu
ROPE = 500000.0  # Llama-3 rope_theta


def _mk(rng, B, Hq, Hkv, lens, bits, pages=None):
    D = 128
    max_blocks = (max(lens) + 63) // 64
    pages = pages or (B * max_blocks + 1)
    kp, vp = kv.PagePool(pages, Hkv, D, bits, rng), kv.PagePool(pages, Hkv, D, bits, rng)
    bt = (1 + np.arange(B * max_blocks).reshape(B, max_blocks)) % pages
    for b in range(B):  # pad short rows with page 0 like model_runner.py:494-500
        bt[b, (lens[b] + 63) // 64:] = 0
    q = rng.standard_normal((B, Hq, D)).astype(np.float16)
    k = rng.standard_normal((B, Hkv, D)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, D)).astype(np.float16)
    return kp, vp, bt, q, k, v


def _run_gpu(dev, kp, vp, bt, q, k, v, lens, bits, rope=ROPE):
    import qserve_backend.fused_attention as fa
    B, Hq, D = q.shape
    Hkv = k.shape[1]
    gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
    table = kv_pointer_table(gk, gv, bt, dev)
    # strided views of a packed qkv buffer, as in llama_w4a8_unpad.py:245-252
    qkv = torch.from_numpy(np.concatenate([q.reshape(B, -1), k.reshape(B, -1), v.reshape(B, -1)], axis=1)).to(dev)
    qd, kd, vd = qkv.split([Hq * D, Hkv * D, Hkv * D], dim=-1)
    qd, kd, vd = qd.reshape(B, Hq, D), kd.reshape(B, Hkv, D), vd.reshape(B, Hkv, D)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    out = fa.single_query_attention(qd, kd, vd, table, lens_d, None, 8192, 64, Hkv * D * bits // 8, int(max(lens)), D, rope, True,
                                    bits == 4, True)
    torch.cuda.synchronize()
    return np_of(out), gk.download(), gv.download()


def _check_pages(kp_o, vp_o, k_gpu, v_gpu, bt, lens):
    kg = kv.PagePool(kp_o.data.shape[0], kp_o.Hkv, kp_o.D, kp_o.bits); kg.data[:] = k_gpu
    vg = kv.PagePool(vp_o.data.shape[0], vp_o.Hkv, vp_o.D, vp_o.bits); vg.data[:] = v_gpu
    # everything except the appended slots is untouched
    mk = np.ones_like(kp_o.data, dtype=bool)
    for b, L in enumerate(lens):
        page, slot = bt[b, (L - 1) // 64], (L - 1) % 64
        # V: bit exact
        assert np.array_equal(vg.codes()[page, :, slot], vp_o.codes()[page, :, slot])
        assert np.array_equal(bits16(vg.scales()[page, :, slot]), bits16(vp_o.scales()[page, :, slot]))
        assert np.array_equal(bits16(vg.zeros()[page, :, slot]), bits16(vp_o.zeros()[page, :, slot]))
        # K: within tolerance
        assert ulp16_diff(kg.scales()[page, :, slot], kp_o.scales()[page, :, slot]).max() <= 1
        assert ulp16_diff(kg.zeros()[page, :, slot], kp_o.zeros()[page, :, slot]).max() <= 1
        cg, co = kg.codes()[page, :, slot], kp_o.codes()[page, :, slot]
        if kp_o.bits == 4:
            cg, co = kv.unpack_nibbles(cg), kv.unpack_nibbles(co)
        d = np.abs(cg.astype(np.int32) - co.astype(np.int32))
        assert d.max() <= 1 and (d > 0).mean() <= 0.03
    # no other byte of either pool changed (compare against the oracle's post-state outside the appended slots)
    for g, o in ((kg, kp_o), (vg, vp_o)):
        same = g.data == o.data
        assert same.mean() > 0.999


CASES = [  # (B, Hq, Hkv, lens)
    (3, 8, 2, [1, 65, 200]),
    (4, 32, 8, [17, 16, 64, 129]),
    (2, 4, 4, [300, 31]),          # MHA (G = 1)
    (2, 16, 1, [90, 257]),         # G = 16 -> two head groups per kv head
    (2, 32, 8, [1025, 700]),       # context splits (flash-decoding merge)
    (1, 64, 64, [2048]),           # Qwen-72B-like MHA, long context
]


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens", CASES)
def test_decode_attention(dev, bits, B, Hq, Hkv, lens):
    rng = np.random.default_rng(B * 100 + Hq + sum(lens) + bits)
    kp, vp, bt, q, k, v = _mk(rng, B, Hq, Hkv, lens, bits)
    kp2, vp2 = kv.PagePool(kp.data.shape[0], Hkv, 128, bits), kv.PagePool(vp.data.shape[0], Hkv, 128, bits)
    kp2.data[:], vp2.data[:] = kp.data, vp.data
    out_g, k_gpu, v_gpu = _run_gpu(dev, kp, vp, bt, q, k, v, lens, bits)
    exact = kv.decode_attention(q, k, v, kp, vp, bt, lens, ROPE, faithful=False).astype(np.float32)
    _check_pages(kp, vp, k_gpu, v_gpu, bt, lens)
    scale = max(1.0, float(np.abs(exact).max()))
    err_g = np.abs(out_g.astype(np.float32) - exact).max()
    assert np.isfinite(out_g.astype(np.float32)).all()
    assert err_g <= 3e-3 * scale, (err_g, scale)
    if sum(lens) <= 1500:  # the faithful oracle is a python loop: only on the small cases
        faithful = kv.decode_attention(q, k, v, kp2, vp2, bt, lens, ROPE, faithful=True).astype(np.float32)
        err_f = np.abs(faithful - exact).max()
        assert err_f <= 1e-2 * scale
        assert err_g <= 1.5 * err_f + 1e-3 * scale, (err_g, err_f)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_attn_bits.npz")
GOLDEN_CASES = [  # (B, Hq, Hkv, lens): G = 4 with a length-1 sequence, G = 1, G = 16 (two head groups), and context splits at small batch
    (3, 8, 2, [1, 65, 200]),
    (2, 4, 4, [300, 31]),
    (2, 16, 1, [90, 257]),
    (2, 32, 8, [1025, 700]),
    (1, 16, 1, [1500]),
    (1, 64, 64, [2048]),
]


def decode_attn_outputs(dev, case, bits):
    """The outputs of single_query_attention (fp16 out) and single_query_attention_quant (int8 codes, scale, sum) for GOLDEN_CASES[case],
    each on a fresh copy of the cache built from a fixed seed, as int16 / int8 tensors on the host."""
    import qserve_backend.fused_attention as fa
    from qserve_b200 import backend as ext
    B, Hq, Hkv, lens = GOLDEN_CASES[case]
    D = 128
    kp, vp, bt, q, k, v = _mk(np.random.default_rng(9000 + 10 * case + bits), B, Hq, Hkv, lens, bits)
    res = {}
    for fused in (False, True):
        gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
        table = kv_pointer_table(gk, gv, bt, dev)
        qd, kd, vd = to_dev(q, dev), to_dev(k, dev), to_dev(v, dev)
        lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
        args = (8192, 64, Hkv * D * bits // 8, int(max(lens)), D, ROPE)
        if fused:
            oq = torch.empty((B, Hq * D), dtype=torch.int8, device=dev)
            sc = torch.empty(B, dtype=torch.half, device=dev)
            sm = torch.empty(B, dtype=torch.half, device=dev)
            ext.single_query_attention_quant(qd, kd, vd, table, lens_d, *args, bits == 4, True, oq, sc, sm)
            res.update(codes=oq, scale=sc.view(torch.int16), sum=sm.view(torch.int16))
        else:
            res["out"] = fa.single_query_attention(qd, kd, vd, table, lens_d, None, *args, True, bits == 4, True).view(torch.int16)
    torch.cuda.synchronize()
    return {key: t.cpu() for key, t in res.items()}


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("case", range(len(GOLDEN_CASES)))
def test_decode_attention_output_bits_are_pinned(dev, case, bits):
    """The output bits of both decode-attention ops equal the stored fixture (tests/golden/make_golden_decode_attn.py, written on an H100
    with 132 SMs: the context-split count, and so the summation order, depends on the SM count)."""
    want = np.load(GOLDEN)
    got = decode_attn_outputs(dev, case, bits)
    for key, t in got.items():
        assert torch.equal(t, torch.from_numpy(want[f"kv{bits}_{case}_{key}"])), key


def test_decode_attention_config2_properties(dev):
    """BASELINE config 2 size (B=64, Hq=32, Hkv=8, ctx=1024 -> len 1025): size-independent properties.
    (1) out is a convex combination of dequantised V rows: within [min V, max V] per dim;
    (2) idempotent append: running twice with the same inputs leaves the pages byte-identical and returns the same bits;
    (3) a sequence whose query is all zeros returns the plain mean of the V rows (uniform softmax) for a sampled head."""
    import qserve_backend.fused_attention as fa
    rng = np.random.default_rng(42)
    B, Hq, Hkv, D, L = 64, 32, 8, 128, 1025
    lens = [L] * B
    kp, vp, bt, q, k, v = _mk(rng, B, Hq, Hkv, lens, 4)
    q[5] = 0
    gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
    table = kv_pointer_table(gk, gv, bt, dev)
    qd, kd, vd = to_dev(q, dev), to_dev(k, dev), to_dev(v, dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    args = (qd, kd, vd, table, lens_d, None, 8192, 64, Hkv * D // 2, L, D, ROPE, True, True, True)
    o1 = fa.single_query_attention(*args)
    snap_k, snap_v = gk.t.clone(), gv.t.clone()
    o2 = fa.single_query_attention(*args)
    torch.cuda.synchronize()
    assert torch.equal(o1, o2) and torch.equal(snap_k, gk.t) and torch.equal(snap_v, gv.t)
    kg = kv.PagePool(kp.data.shape[0], Hkv, D, 4); kg.data[:] = gk.download()
    vg = kv.PagePool(vp.data.shape[0], Hkv, D, 4); vg.data[:] = gv.download()
    o = np_of(o1).astype(np.float32)
    for b, h in ((0, 0), (5, 13), (63, 31)):
        vc, vs, vz = kv.pool_read_tokens(vg, bt[b], L)
        vdq = kv.kv_dequant(vc, vs, vz, 4)[h // 4].astype(np.float32)  # [L, D]
        assert (o[b, h] <= vdq.max(axis=0) + 1e-2).all() and (o[b, h] >= vdq.min(axis=0) - 1e-2).all()
        if b == 5:
            vdq[L - 1] = v[b, h // 4].astype(np.float32)  # the current token is used un-quantised (Template.hpp:2147)
            assert np.abs(o[b, h] - vdq.mean(axis=0)).max() <= 3e-3 * max(1.0, np.abs(vdq.mean(axis=0)).max())


@pytest.mark.parametrize("bits", [4, 8])
def test_prefill_rope_append_and_padding_offsets(dev, bits):
    import qserve_backend.fused_attention as fa
    rng = np.random.default_rng(7 + bits)
    Hq, Hkv, D = 8, 2, 128
    lens = np.array([5, 70, 1, 130], np.int32)
    B, T, maxlen = len(lens), int(lens.sum()), int(lens.max())
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pad_o = kv.compute_padding_offsets(cu, maxlen, T)
    pad = fa.compute_padding_offsets(to_dev(cu, dev), maxlen, T)
    assert np.array_equal(np_of(pad), pad_o)
    qkv = rng.standard_normal((T, (Hq + 2 * Hkv) * D)).astype(np.float16)
    max_blocks = (maxlen + 63) // 64
    bt = np.arange(B * max_blocks).reshape(B, max_blocks)
    kp, vp = kv.PagePool(B * max_blocks, Hkv, D, bits), kv.PagePool(B * max_blocks, Hkv, D, bits)
    gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
    table = kv_pointer_table(gk, gv, bt, dev)
    qkv_d = to_dev(qkv, dev)
    fa.apply_bias_rope_update_kv_cache(qkv_d, to_dev(lens, dev), pad, table, Hq, Hkv, maxlen, 64, Hkv * D * bits // 8, D, ROPE, 8192,
                                       True, bits == 4, True)
    torch.cuda.synchronize()
    qkv_o = kv.prefill_rope_append(qkv.copy(), lens, pad_o, kp, vp, bt, Hq, Hkv, maxlen, ROPE, 8192)
    got = np_of(qkv_d)
    assert np.array_equal(got[:, (Hq + Hkv) * D:], qkv[:, (Hq + Hkv) * D:])  # v untouched
    d = ulp16_diff(got[:, : (Hq + Hkv) * D], qkv_o[:, : (Hq + Hkv) * D])
    big = np.abs(qkv_o[:, : (Hq + Hkv) * D].astype(np.float32)) > 2e-2  # ulp distance is meaningless next to zero
    assert d[big].max() <= 2 and (d[big] > 0).mean() < 0.02
    assert np.abs(got[:, : (Hq + Hkv) * D].astype(np.float32) - qkv_o[:, : (Hq + Hkv) * D].astype(np.float32)).max() <= 2e-3
    kg = kv.PagePool(B * max_blocks, Hkv, D, bits); kg.data[:] = gk.download()
    vg = kv.PagePool(B * max_blocks, Hkv, D, bits); vg.data[:] = gv.download()
    assert np.array_equal(vg.data, vp.data), "V pages must be bit-exact"
    assert ulp16_diff(kg.scales(), kp.scales()).max() <= 1 and ulp16_diff(kg.zeros(), kp.zeros()).max() <= 1
    cg, co = kg.codes(), kp.codes()
    if bits == 4:
        cg, co = kv.unpack_nibbles(cg), kv.unpack_nibbles(co)
    dd = np.abs(cg.astype(np.int32) - co.astype(np.int32))
    assert dd.max() <= 1 and (dd > 0).mean() < 0.01


def test_attention_argument_errors(dev):
    import qserve_backend.fused_attention as fa
    B, Hq, Hkv, D = 2, 4, 2, 128
    q = torch.zeros((B, Hq, D), dtype=torch.half, device=dev)
    k = torch.zeros((B, Hkv, D), dtype=torch.half, device=dev)
    table = torch.zeros((B, 2, 1), dtype=torch.int64, device=dev)
    lens = torch.ones(B, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError):  # length tensor must be int32 (fused_attention.cpp:189)
        fa.single_query_attention(q, k, k, table, lens.long(), None, 8192, 64, Hkv * D // 2, 1, D, 1e4, True, True, True)
    with pytest.raises(RuntimeError):  # fp32 is not dispatched by the reference either
        fa.single_query_attention(q.float(), k.float(), k.float(), table, lens, None, 8192, 64, Hkv * D // 2, 1, D, 1e4, True, True, True)
    with pytest.raises(RuntimeError):  # size_per_token inconsistent with the cache type
        fa.single_query_attention(q, k, k, table, lens, None, 8192, 64, Hkv * D, 1, D, 1e4, True, True, True)
    with pytest.raises(RuntimeError):  # kv cache without zero points is never produced by the engine (arg_utils.py:422)
        fa.single_query_attention(q, k, k, table, lens, None, 8192, 64, Hkv * D // 2, 1, D, 1e4, True, True, False)

    from qserve_b200 import backend as ext
    out_q = torch.zeros((B, Hq * D), dtype=torch.int8, device=dev)
    scale = torch.zeros(B, dtype=torch.half, device=dev)
    quant = dict(q=q, k=k, v=k, kv_pointers=table, length_per_sample=lens, memory_max_seqlen=8192, tokens_per_block=64, size_per_token=Hkv * D // 2,
                 timestep=1, rotary_embedding_dim=D, rotary_base=1e4, int4_kv_cache=True, kv_cache_with_zeros=True, out_q=out_q, out_scale=scale,
                 out_sum=scale)

    def bad_quant(**kw):
        with pytest.raises(RuntimeError):
            ext.single_query_attention_quant(**{**quant, **kw})

    bad_quant(q=q.cpu())                                      # CPU tensors
    bad_quant(k=k.cpu(), v=k.cpu())
    bad_quant(kv_pointers=table.cpu())
    bad_quant(length_per_sample=lens.cpu())
    bad_quant(out_q=out_q.cpu())
    bad_quant(out_scale=scale.cpu())
    bad_quant(k=k.float(), v=k.float())                       # dtypes
    bad_quant(kv_pointers=table.int())
    bad_quant(length_per_sample=lens.long())
    bad_quant(out_scale=scale.float())
    bad_quant(out_sum=scale.float())
    bad_quant(length_per_sample=lens[:1].clone())             # one entry per sequence
    bad_quant(out_sum=scale[:1].clone())
    bad_quant(length_per_sample=torch.ones((B, 2), dtype=torch.int32, device=dev)[:, 0])  # not contiguous
    if torch.cuda.device_count() > 1:                         # every tensor on q's device
        bad_quant(kv_pointers=table.to("cuda:1"))
        bad_quant(length_per_sample=lens.to("cuda:1"))
        bad_quant(out_scale=scale.to("cuda:1"))


def test_multi_wave_launches_are_stable(dev):
    """Regression (round 2): more CTAs than resident slots (4 per SM).  A late CTA of a multi-wave launch does not sit in
    griddepcontrol.wait, so its warps reach their first bulk copy immediately; in round 1 thread 0 initialised every warp's
    ring barriers without a block barrier, and a warp that armed its ring first lost its transaction count and hung (one
    warp in ~1e8 slices: seen only at Qwen1.5-72B size, 4096 CTAs per launch).  Many back-to-back launches must all finish
    and reproduce the first result bit for bit."""
    import qserve_backend.fused_attention as fa
    from qserve_b200.decode import DecodeRunner

    B = 192  # x 8 kv heads = 1536 CTAs, 592 resident slots
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=200, device=dev, layers=1, fused=False, seed=11)
    g = torch.Generator(device=dev).manual_seed(3)
    run.qkv_buf.copy_(torch.randn(run.qkv_buf.shape, device=dev, generator=g).half())
    D = 128
    q, k, v = run.qkv_buf.split([run.q_size, run.kv_size, run.kv_size], dim=-1)
    q, k, v = q.reshape(B, run.Hq, D), k.reshape(B, run.Hkv, D), v.reshape(B, run.Hkv, D)
    args = (q, k, v, run.block_tables[0], run.context_lens, None, 8192, 64, run.size_per_token, run.max_seq_len, D, run.cfg.rope_theta, True, True, True)
    first = fa.single_query_attention(*args).clone()
    for _ in range(400):
        out = fa.single_query_attention(*args)
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    assert torch.isfinite(first.float()).all()
