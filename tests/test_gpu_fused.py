"""GPU: the fused extensions are bit-identical to the reference op sequences they replace."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,H", [(64, 4096), (5, 8192), (3, 512)])
@pytest.mark.parametrize("with_sum", [True, False])
def test_add_rms_norm_general_equals_add_then_norm(dev, M, H, with_sum):
    from qserve_b200 import backend as ext
    import qserve_backend.layernorm_ops as ln
    g = torch.Generator(device="cpu").manual_seed(M + H)
    x = (torch.randn((M, H), generator=g) * 3).half().to(dev)
    delta = torch.randn((M, H), generator=g).half().to(dev)
    gamma = (1 + 0.1 * torch.randn(H, generator=g)).half().to(dev)
    q1 = torch.empty((M, H), dtype=torch.int8, device=dev); s1 = torch.empty(M, dtype=torch.half, device=dev); m1 = torch.zeros(M, dtype=torch.half, device=dev)
    q2 = torch.empty_like(q1); s2 = torch.empty_like(s1); m2 = torch.zeros_like(m1)
    hidden = x + delta
    if with_sum:
        ln.rms_norm_general_fuse_sum(q1, hidden, gamma, m1, s1, 1e-5, True)
    else:
        ln.rms_norm_general(q1, hidden, gamma, s1, 1e-5, True)
    h2 = torch.empty_like(x)
    ext.add_rms_norm_general(q2, h2, x, delta, gamma, m2 if with_sum else None, s2, 1e-5)
    torch.cuda.synchronize()
    assert torch.equal(h2, hidden) and torch.equal(q1, q2) and torch.equal(s1, s2) and torch.equal(m1, m2)


@pytest.mark.parametrize("M,d", [(64, 14336), (7, 1024), (2, 24576)])
@pytest.mark.parametrize("with_sum", [True, False])
def test_silu_and_mul_quant_equals_silu_then_quant(dev, M, d, with_sum):
    from qserve_b200 import backend as ext
    import qserve_backend.activation_ops as act
    import qserve_backend.fused_kernels as fk
    g = torch.Generator(device="cpu").manual_seed(M + d)
    x = (torch.randn((M, 2 * d), generator=g) * 2).half().to(dev)
    a = torch.empty((M, d), dtype=torch.half, device=dev)
    act.silu_and_mul(a, x)
    q1 = torch.empty((M, d), dtype=torch.int8, device=dev); s1 = torch.empty(M, dtype=torch.half, device=dev); m1 = torch.zeros(M, dtype=torch.half, device=dev)
    q2 = torch.empty_like(q1); s2 = torch.empty_like(s1); m2 = torch.zeros_like(m1)
    if with_sum:
        fk.invoke_quant_fuse_sum(q1, a, m1, s1)
    else:
        fk.invoke_quant(q1, a, s1)
    ext.silu_and_mul_quant(q2, x, m2 if with_sum else None, s2)
    torch.cuda.synchronize()
    assert torch.equal(q1, q2) and torch.equal(s1, s2) and torch.equal(m1, m2)


@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv4-g128", "w8a8kv8"])
def test_fused_runner_matches_reference_sequence(dev, precision):
    from qserve_b200.decode import DecodeRunner
    outs = []
    for fused in (False, True):
        run = DecodeRunner("tiny", precision, batch=6, ctx=100, device=dev, seed=5, fused=fused)
        run.tokens_in.copy_(torch.arange(6, device=dev) * 11)
        with torch.no_grad():
            outs.append(run.forward(run.tokens_in).clone())
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


INF, NAN = float("inf"), float("nan")
QUANT_CASES = [  # (B, Hq, Hkv, lens, with_sum, non-finite entries (sequence, kv head, dim, value) of the new token's V)
    (4, 32, 8, [17, 16, 64, 129], True, ()),  # Llama-3 head geometry, no context split -> bit identical to the two-op sequence
    (3, 8, 2, [1, 65, 200], False, ()),
    (2, 16, 1, [90, 257], True, ()),          # two head groups per kv head
    (2, 32, 8, [1025, 700], True, ()),        # context splits: two-level last-CTA merge
    (1, 64, 64, [2048], True, ()),            # 64 CTAs per token
    # an overflowed qkv GEMM: the output rows hold inf / NaN, and the row sum must say so as invoke_quant_fuse_sum does
    (4, 32, 8, [17, 16, 64, 129], True, ((0, 1, 5, INF), (2, 3, 7, NAN))),
    (2, 32, 8, [1025, 700], True, ((0, 2, 9, INF), (1, 0, 3, INF), (1, 5, 100, -INF))),
]


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("B,Hq,Hkv,lens,with_sum,bad_v", [
    pytest.param(*c, id=f"{c[0]}-{c[1]}-{c[2]}-lens{i}-{c[4]}" + ("-nonfinite" if c[5] else "")) for i, c in enumerate(QUANT_CASES)])
def test_attention_quant_equals_attention_then_quant(dev, bits, B, Hq, Hkv, lens, with_sum, bad_v):
    """single_query_attention_quant == invoke_quant[_fuse_sum](single_query_attention(...)); KV pages updated identically."""
    from oracle import kv
    from qserve_b200 import backend as ext
    import qserve_backend.fused_attention as fa
    import qserve_backend.fused_kernels as fk
    from tests.test_gpu_attention import _mk, ROPE
    from tests.util import GpuPool, kv_pointer_table
    rng = np.random.default_rng(B + Hq + sum(lens) + bits)
    kp, vp, bt, q, k, v = _mk(rng, B, Hq, Hkv, lens, bits)
    for b, h, d, x in bad_v:
        v[b, h, d] = x
    D = 128
    res = []
    for fused in (False, True):
        gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
        table = kv_pointer_table(gk, gv, bt, dev)
        qkv = torch.from_numpy(np.concatenate([q.reshape(B, -1), k.reshape(B, -1), v.reshape(B, -1)], axis=1)).to(dev)
        qd, kd, vd = qkv.split([Hq * D, Hkv * D, Hkv * D], dim=-1)
        qd, kd, vd = qd.reshape(B, Hq, D), kd.reshape(B, Hkv, D), vd.reshape(B, Hkv, D)
        lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
        oq = torch.empty((B, Hq * D), dtype=torch.int8, device=dev)
        sc = torch.empty(B, dtype=torch.half, device=dev)
        sm = torch.zeros(B, dtype=torch.half, device=dev)
        args = (8192, 64, Hkv * D * bits // 8, int(max(lens)), D, ROPE)
        if fused:
            ext.single_query_attention_quant(qd, kd, vd, table, lens_d, *args, bits == 4, True, oq, sc, sm if with_sum else None)
        else:
            out = fa.single_query_attention(qd, kd, vd, table, lens_d, None, *args, True, bits == 4, True).reshape(B, -1)
            if with_sum:
                fk.invoke_quant_fuse_sum(oq, out, sm, sc)
            else:
                fk.invoke_quant(oq, out, sc)
        torch.cuda.synchronize()
        res.append((oq.cpu(), sc.cpu(), sm.cpu(), gk.download(), gv.download()))
    (q1, s1, m1, k1, v1), (q2, s2, m2, k2, v2) = res
    assert np.array_equal(k1, k2) and np.array_equal(v1, v2)
    assert torch.equal(q1, q2) and torch.equal(s1.view(torch.int16), s2.view(torch.int16)) and torch.equal(m1.view(torch.int16), m2.view(torch.int16))


@pytest.mark.parametrize("rows,vocab", [(64, 128256), (3, 32000), (1, 1024), (5, 152064)])
def test_argmax_rows_matches_torch(dev, rows, vocab):
    """argmax_rows == torch.argmax(dim=-1), including ties (first index wins) and NaN (counts as the maximum)."""
    from qserve_b200 import backend as ext
    g = torch.Generator(device="cpu").manual_seed(rows + vocab)
    x = torch.randn((rows, vocab), generator=g).half()
    x[0, 7] = x[0].max() ; x[0, vocab - 5] = x[0, 7]          # a tie: the first index must win
    if rows > 1:
        x[1, 123] = float("nan")
    xd = x.to(dev)
    got = ext.argmax_rows(xd)
    torch.cuda.synchronize()
    want = torch.argmax(xd, dim=-1)
    assert torch.equal(got, want)
    assert int(got[0]) <= 7
