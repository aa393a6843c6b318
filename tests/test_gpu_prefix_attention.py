"""GPU: prompt chunks over a cached prefix -- qs_apply_bias_rope_update_kv_cache_at (RoPE + KV append at an offset) and
qs_prefix_prefill_attention (wgmma attention over the dequantised INT4 / INT8 prefix and the fp16 chunk).

Stated tolerance: the prompt-attention bar of test_gpu_prefill_attention.py, per element
    |out - exact| <= 2 fp16 ulps of |exact| + 1.5e-3 * max|v|
where `exact` is the float64 oracle over the dequantised prefix (kv_dequant, which the kernel reproduces element for element) and the chunk,
and v ranges over both.  Unwritten page slots are filled with NaN scales, so any read of a slot beyond the prefix shows up as NaN.
"""
import numpy as np
import pytest
import torch

from oracle import kv
from oracle import prefix as oprefix
from tests.util import GpuPool, kv_pointer_table, np_of, to_dev

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128


def _tol(exact, vmax):
    a = np.abs(exact)
    ulp = np.where(a >= 2.0 ** -14, 2.0 ** (np.floor(np.log2(np.maximum(a, 2.0 ** -14))) - 10), 2.0 ** -24)
    return 2 * ulp + 1.5e-3 * vmax


def _pools(rng, B, n_blocks, hkv, bits, prefix):
    """Random pages (SURVEY.md 8d config 2 statistics) with every slot at or beyond each sequence's prefix poisoned with NaN scales."""
    pages = B * n_blocks + 1
    kp, vp = kv.PagePool(pages, hkv, D, bits, rng), kv.PagePool(pages, hkv, D, bits, rng)
    bt = 1 + np.arange(B * n_blocks).reshape(B, n_blocks)
    for b in range(B):
        for t in range(prefix[b], n_blocks * 64):
            for p in (kp, vp):
                p.scales()[bt[b, t // 64], :, t % 64] = np.float16("nan")
    return kp, vp, bt


class Case:
    """A batch of chunks (lengths C) behind cached prefixes (lengths P): pages on the device, chunk appended with append_at."""

    def __init__(self, dev, P, C, hq, hkv, bits, seed, n_blocks=None):
        from qserve_b200 import backend
        rng = np.random.default_rng(seed)
        self.P, self.C, self.hq, self.hkv, self.bits = list(P), list(C), hq, hkv, bits
        B = len(P)
        self.n_blocks = n_blocks or max(1, (max(P) + max(C) + 63) // 64)
        self.kp, self.vp, self.bt = _pools(rng, B, self.n_blocks, hkv, bits, P)
        self.gk, self.gv = GpuPool(self.kp, dev), GpuPool(self.vp, dev)
        self.table = kv_pointer_table(self.gk, self.gv, self.bt, dev)
        self.spt = hkv * D * bits // 8
        T = sum(C)
        self.cu = np.concatenate([[0], np.cumsum(C)]).astype(np.int32)
        self.cu_d = to_dev(self.cu, dev)
        self.prefix_d = torch.tensor(P, dtype=torch.int32, device=dev)
        self.lens_d = torch.tensor(C, dtype=torch.int32, device=dev)
        self.max_c = max(max(C), 1)
        self.pad = backend.compute_padding_offsets(self.cu_d, self.max_c, T)
        self.qkv = torch.from_numpy(rng.standard_normal((T, (hq + 2 * hkv) * D)).astype(np.float16)).to(dev)
        self.append()
        q, k, v = self.qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        self.q, self.k, self.v = q.reshape(T, hq, D), k.reshape(T, hkv, D), v.reshape(T, hkv, D)

    def append(self):
        from qserve_b200 import backend
        backend.apply_bias_rope_update_kv_cache_at(self.qkv, self.lens_d, self.pad, self.prefix_d, self.table, self.hq, self.hkv, self.max_c, 64,
                                                   self.spt, D, ROPE, 8192, True, self.bits == 4, True)

    def attend(self, **kw):
        from qserve_b200 import backend
        return backend.prefix_prefill_attention(self.q, self.k, self.v, self.cu_d, max(self.C), self.prefix_d, max(self.P), self.table, 64, self.spt,
                                                self.bits == 4, **kw)

    def prefixes(self):
        kg = kv.PagePool(self.kp.data.shape[0], self.hkv, D, self.bits); kg.data[:] = self.gk.download()
        vg = kv.PagePool(self.vp.data.shape[0], self.hkv, D, self.bits); vg.data[:] = self.gv.download()
        pk = [oprefix.dequant_prefix(kg, self.bt[b], p) for b, p in enumerate(self.P)]
        pv = [oprefix.dequant_prefix(vg, self.bt[b], p) for b, p in enumerate(self.P)]
        return pk, pv

    def exact(self, softmax_scale=None):
        pk, pv = self.prefixes()
        q, k, v = np_of(self.q), np_of(self.k), np_of(self.v)
        vmax = max([float(np.abs(v).max()) if v.size else 0.0] + [float(np.abs(x).max()) for x in pv if x.size])
        return oprefix.prefix_causal_attention(q, k, v, self.cu, pk, pv, softmax_scale), vmax


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. RoPE + append at an offset: two chunks leave exactly the bytes of one call
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("split", [1, 63, 64, 65, 200])
def test_append_at_two_chunks_is_byte_identical(dev, bits, split):
    from qserve_b200 import backend
    rng = np.random.default_rng(split * 10 + bits)
    hq, hkv = 8, 2
    lens = [300, 70, 1, 201, 64]
    B, T = len(lens), sum(lens)
    nb = (max(lens) + 63) // 64
    spt = hkv * D * bits // 8
    qkv = rng.standard_normal((T, (hq + 2 * hkv) * D)).astype(np.float16)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    pool = lambda: GpuPool(kv.PagePool(B * nb + 1, hkv, D, bits, np.random.default_rng(0)), dev)  # noqa: E731
    k1, v1, k2, v2 = pool(), pool(), pool(), pool()
    one = to_dev(qkv, dev)
    backend.apply_bias_rope_update_kv_cache(one, to_dev(np.array(lens, np.int32), dev), backend.compute_padding_offsets(to_dev(cu, dev), max(lens), T),
                                            kv_pointer_table(k1, v1, bt, dev), hq, hkv, max(lens), 64, spt, D, ROPE, 8192, True, bits == 4, True)
    a = [min(split, L) for L in lens]
    rest = [L - x for L, x in zip(lens, a)]
    rows_a = np.concatenate([np.arange(cu[b], cu[b] + a[b]) for b in range(B)])
    rows_b = np.concatenate([np.arange(cu[b] + a[b], cu[b + 1]) for b in range(B)])
    table2 = kv_pointer_table(k2, v2, bt, dev)
    two = torch.empty_like(one)
    for rows, ln, start in ((rows_a, a, [0] * B), (rows_b, rest, a)):
        if len(rows) == 0:
            continue
        part = to_dev(qkv[rows], dev)
        cuc = np.concatenate([[0], np.cumsum(ln)]).astype(np.int32)
        mx = max(max(ln), 1)
        backend.apply_bias_rope_update_kv_cache_at(part, to_dev(np.array(ln, np.int32), dev), backend.compute_padding_offsets(to_dev(cuc, dev), mx, len(rows)),
                                                   to_dev(np.array(start, np.int32), dev), table2, hq, hkv, mx, 64, spt, D, ROPE, 8192, True, bits == 4, True)
        two[torch.from_numpy(rows).to(dev)] = part
    torch.cuda.synchronize()
    assert torch.equal(one.view(torch.int16), two.view(torch.int16))
    assert torch.equal(k1.t, k2.t) and torch.equal(v1.t, v2.t)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. parity with the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------------------
PREFIX = [0, 1, 63, 64, 65, 127, 128, 1000]
CHUNK = [17, 1, 128, 129, 300, 0, 17, 129]  # every chunk length of the plan, and one empty chunk


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("hq,hkv", [(1, 1), (4, 1), (8, 2), (32, 8)])
def test_matches_oracle(dev, bits, hq, hkv):
    c = Case(dev, PREFIX, CHUNK, hq, hkv, bits, seed=hq * 10 + hkv + bits)
    out = c.attend()
    torch.cuda.synchronize()
    assert out.shape == c.q.shape and out.dtype == torch.half
    exact, vmax = c.exact()
    got = np_of(out).astype(np.float64)
    assert np.isfinite(got).all()
    err = np.abs(got - exact)
    assert (err <= _tol(exact, vmax)).all(), f"max err {err.max():.3e}"


def test_reversed_lengths_and_scale(dev):
    """The same lengths paired the other way round (long chunks behind short prefixes and vice versa) and a non-default softmax scale."""
    c = Case(dev, PREFIX[::-1], CHUNK, 8, 2, 4, seed=77)
    out = c.attend(softmax_scale=0.05)
    exact, vmax = c.exact(softmax_scale=0.05)
    assert (np.abs(np_of(out).astype(np.float64) - exact) <= _tol(exact, vmax)).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. empty prefix: the prompt attention of the whole chunk
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
def test_empty_prefix_matches_prompt_attention(dev, bits):
    from qserve_b200 import backend
    C = [128, 1, 130, 333, 64]
    c = Case(dev, [0] * len(C), C, 8, 2, bits, seed=5 + bits)
    out = c.attend()
    ref = backend.flash_attn_varlen_func(c.q, c.k, c.v, c.cu_d, c.cu_d, max(C), max(C), dropout_p=0.0, causal=True)
    exact, vmax = c.exact()
    err = np.abs(np_of(out).astype(np.float64) - exact)
    assert (err <= _tol(exact, vmax)).all()
    assert err.max() <= 1.25 * np.abs(np_of(ref).astype(np.float64) - exact).max() + 1e-3


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. a 1-token chunk is a decode step: the decode kernel and the new path on copies of one cache
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
def test_one_token_chunk_agrees_with_decode(dev, bits):
    from qserve_b200 import backend
    rng = np.random.default_rng(40 + bits)
    hq, hkv = 32, 8
    P = [1, 63, 64, 65, 1000]
    B = len(P)
    nb = (max(P) + 1 + 63) // 64
    kp, vp = kv.PagePool(B * nb + 1, hkv, D, bits, rng), kv.PagePool(B * nb + 1, hkv, D, bits, rng)
    bt = 1 + np.arange(B * nb).reshape(B, nb)
    q, k, v = (rng.standard_normal((B, h, D)).astype(np.float16) for h in (hq, hkv, hkv))
    spt = hkv * D * bits // 8
    g1k, g1v, g2k, g2v = GpuPool(kp, dev), GpuPool(vp, dev), GpuPool(kp, dev), GpuPool(vp, dev)
    qkv = torch.from_numpy(np.concatenate([q.reshape(B, -1), k.reshape(B, -1), v.reshape(B, -1)], axis=1)).to(dev)
    # decode kernel
    qkv1 = qkv.clone()
    q1, k1, v1 = qkv1.split([hq * D, hkv * D, hkv * D], dim=-1)
    lens = torch.tensor([p + 1 for p in P], dtype=torch.int32, device=dev)
    dec = backend.single_query_attention(q1.reshape(B, hq, D), k1.reshape(B, hkv, D), v1.reshape(B, hkv, D), kv_pointer_table(g1k, g1v, bt, dev), lens, None,
                                         8192, 64, spt, max(P) + 1, D, ROPE, True, bits == 4, True)
    # append at the offset + prefix attention
    qkv2 = qkv.clone()
    table2 = kv_pointer_table(g2k, g2v, bt, dev)
    cu = torch.arange(B + 1, dtype=torch.int32, device=dev)
    prefix = torch.tensor(P, dtype=torch.int32, device=dev)
    backend.apply_bias_rope_update_kv_cache_at(qkv2, torch.ones(B, dtype=torch.int32, device=dev), backend.compute_padding_offsets(cu, 1, B), prefix,
                                               table2, hq, hkv, 1, 64, spt, D, ROPE, 8192, True, bits == 4, True)
    q2, k2, v2 = qkv2.split([hq * D, hkv * D, hkv * D], dim=-1)
    new = backend.prefix_prefill_attention(q2.reshape(B, hq, D), k2.reshape(B, hkv, D), v2.reshape(B, hkv, D), cu, 1, prefix, max(P), table2, 64, spt,
                                           bits == 4)
    torch.cuda.synchronize()
    exact = kv.decode_attention(q, k, v, kp, vp, bt, [p + 1 for p in P], ROPE, faithful=False).astype(np.float64)
    scale = max(1.0, float(np.abs(exact).max()))
    for got in (dec, new):
        g = np_of(got).astype(np.float64)
        assert np.isfinite(g).all()
        assert np.abs(g - exact).max() <= 3e-3 * scale


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. full size: Llama-3-8B heads, 8 x (1024 prefix + 512 chunk), KV4, against a float32 torch reference on the device
# ---------------------------------------------------------------------------------------------------------------------------------
def test_llama3_8b_full_size(dev):
    B, P, C = 8, 1024, 512
    c = Case(dev, [P] * B, [C] * B, 32, 8, 4, seed=3)
    out = c.attend()
    pk, pv = c.prefixes()
    mask = torch.cat([torch.zeros(C, P, dtype=torch.bool, device=dev), torch.triu(torch.ones(C, C, dtype=torch.bool, device=dev), 1)], dim=1)
    worst = 0.0
    for b in range(B):
        s = slice(int(c.cu[b]), int(c.cu[b + 1]))
        kk = torch.cat([torch.from_numpy(pk[b]).to(dev), c.k[s]]).float().repeat_interleave(4, dim=1).transpose(0, 1)
        vv = torch.cat([torch.from_numpy(pv[b]).to(dev), c.v[s]]).float().repeat_interleave(4, dim=1).transpose(0, 1)
        qq = c.q[s].float().transpose(0, 1)
        sc = (qq @ kk.transpose(1, 2)) * D ** -0.5
        ref = (torch.softmax(sc.masked_fill(mask, float("-inf")), dim=-1) @ vv).transpose(0, 1)
        worst = max(worst, float((out[s].float() - ref).abs().max()))
    assert worst <= 3e-3, worst


# ---------------------------------------------------------------------------------------------------------------------------------
# 6. determinism and CUDA-graph capture
# ---------------------------------------------------------------------------------------------------------------------------------
def test_deterministic_and_graph_capturable(dev):
    c = Case(dev, [65, 1000, 0, 300], [129, 64, 200, 1], 32, 8, 4, seed=11)
    pristine = c.qkv.clone()
    # the append rotates qkv in place: start every run from the un-rotated rows (re-appending the same tokens writes the same bytes)
    c.qkv.copy_(pristine)
    c.append()
    o1 = c.attend()
    o2 = c.attend()
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    pages_k, pages_v = c.gk.t.clone(), c.gv.t.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up on the capture stream
        c.qkv.copy_(pristine)
        c.append()
        c.attend()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.qkv.copy_(pristine)
        c.append()
        og = c.attend()
    c.qkv.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, o1)
    assert torch.equal(c.gk.t, pages_k) and torch.equal(c.gv.t, pages_v)


# ---------------------------------------------------------------------------------------------------------------------------------
# 7. argument errors
# ---------------------------------------------------------------------------------------------------------------------------------
def test_argument_errors(dev):
    from qserve_b200 import backend
    c = Case(dev, [70, 3], [20, 5], 4, 2, 4, seed=1)
    base = dict(q=c.q, k=c.k, v=c.v, cu_seqlens=c.cu_d, max_seqlen=20, prefix_lens=c.prefix_d, max_prefix_len=70, kv_pointers=c.table,
                tokens_per_block=64, size_per_token=c.spt, int4_kv_cache=True)
    backend.prefix_prefill_attention(**base)  # valid

    def bad(**kw):
        with pytest.raises(RuntimeError):
            backend.prefix_prefill_attention(**{**base, **kw})

    bad(q=c.q.cpu(), k=c.k.cpu(), v=c.v.cpu())                                   # CPU tensors
    bad(prefix_lens=c.prefix_d.cpu())
    bad(q=c.q.float(), k=c.k.float(), v=c.v.float())                            # dtype
    bad(prefix_lens=c.prefix_d.long())
    bad(q=c.q[..., :64], k=c.k[..., :64], v=c.v[..., :64])                      # head_dim != 128
    bad(tokens_per_block=32)                                                     # page size
    bad(size_per_token=c.spt * 2)                                                # KV8 size with the KV4 flag
    bad(max_prefix_len=c.n_blocks * 64)                                          # page table too short
    bad(kv_pointers=c.table[:, :, :1].contiguous())
    bad(k=c.k[:-1], v=c.v[:-1])                                                  # q / k / v cover different tokens
    with pytest.raises(RuntimeError):                                            # append_at: start_pos on the host / of the wrong dtype
        backend.apply_bias_rope_update_kv_cache_at(c.qkv, c.lens_d, c.pad, c.prefix_d.cpu(), c.table, 4, 2, 20, 64, c.spt, D, ROPE, 8192, True, True, True)
    with pytest.raises(RuntimeError):
        backend.apply_bias_rope_update_kv_cache_at(c.qkv, c.lens_d, c.pad, c.prefix_d.long(), c.table, 4, 2, 20, 64, c.spt, D, ROPE, 8192, True, True, True)
