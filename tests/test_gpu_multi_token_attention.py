"""GPU: multi-token decode attention over the paged INT4 / INT8 KV cache (qs_multi_token_decode_attention, speculative-decoding verification).

Stated tolerance: the decode bar of test_gpu_attention.py, |out - exact| <= 3e-3 * max(1, max|exact|), where `exact` is the float64 oracle
(oracle/multi_token.py) over the pages the kernel read.  Page slots at or beyond P_b + n_b hold NaN scales, so any read of a slot the op must
not touch shows up as NaN.

"Equals sequential decoding" compares each token's error with the decode kernel's own error on that token: at most 1.5x it plus 2.5e-4.  The
absolute 2.5e-4 (half an fp16 ulp at |x| in [0.5, 1)) is a deliberate addition to a pure 1.5x ratio: both kernels round their result to fp16
once, so when the decode kernel happens to land within a fraction of an ulp of the float64 value, the ratio alone would fail on rounding.
"""
import numpy as np
import pytest
import torch

from oracle import kv
from oracle import multi_token as omt
from oracle import prefix as oprefix
from tests.util import GpuPool, kv_pointer_table, np_of

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128


def _bar(exact):
    return 3e-3 * max(1.0, float(np.abs(exact).max()) if exact.size else 1.0)


def _pools(rng, B, n_blocks, hkv, bits, filled):
    pages = B * n_blocks + 1
    kp, vp = kv.PagePool(pages, hkv, D, bits, rng), kv.PagePool(pages, hkv, D, bits, rng)
    bt = 1 + np.arange(B * n_blocks).reshape(B, n_blocks)
    for b in range(B):
        for t in range(filled[b], n_blocks * 64):
            for p in (kp, vp):
                p.scales()[bt[b, t // 64], :, t % 64] = np.float16("nan")
    return kp, vp, bt


class Case:
    """A batch of n_b draft tokens behind cached prefixes P_b: pages on the device, drafts appended with append_at."""

    def __init__(self, dev, P, N, hq, hkv, bits, seed, n_blocks=None):
        from qserve_b200 import backend
        rng = np.random.default_rng(seed)
        self.P, self.N, self.hq, self.hkv, self.bits = list(P), list(N), hq, hkv, bits
        B = len(P)
        self.n_blocks = n_blocks or max(1, (max(P) + max(N) + 63) // 64)
        self.kp, self.vp, self.bt = _pools(rng, B, self.n_blocks, hkv, bits, [p + n for p, n in zip(P, N)])
        self.gk, self.gv = GpuPool(self.kp, dev), GpuPool(self.vp, dev)
        self.table = kv_pointer_table(self.gk, self.gv, self.bt, dev)
        self.spt = hkv * D * bits // 8
        T = sum(N)
        self.cu = np.concatenate([[0], np.cumsum(N)]).astype(np.int32)
        self.cu_d = torch.from_numpy(self.cu).to(dev)
        self.prefix_d = torch.tensor(P, dtype=torch.int32, device=dev)
        self.lens_d = torch.tensor(N, dtype=torch.int32, device=dev)
        self.max_n = max(max(N), 1)
        self.pad = backend.compute_padding_offsets(self.cu_d, self.max_n, T)
        self.raw = rng.standard_normal((T, (hq + 2 * hkv) * D)).astype(np.float16)
        self.qkv = torch.from_numpy(self.raw).to(dev)
        self.append()
        q, k, v = self.qkv.split([hq * D, hkv * D, hkv * D], dim=-1)
        self.q, self.k, self.v = q.reshape(T, hq, D), k.reshape(T, hkv, D), v.reshape(T, hkv, D)

    def append(self):
        from qserve_b200 import backend
        backend.apply_bias_rope_update_kv_cache_at(self.qkv, self.lens_d, self.pad, self.prefix_d, self.table, self.hq, self.hkv, self.max_n, 64,
                                                   self.spt, D, ROPE, 8192, True, self.bits == 4, True)

    def attend(self, **kw):
        from qserve_b200 import backend
        return backend.multi_token_decode_attention(self.q, self.k, self.v, self.cu_d, self.max_n, self.prefix_d, max(self.P), self.table, 64,
                                                    self.spt, self.bits == 4, **kw)

    def host_pools(self):
        kg = kv.PagePool(self.kp.data.shape[0], self.hkv, D, self.bits); kg.data[:] = self.gk.download()
        vg = kv.PagePool(self.vp.data.shape[0], self.hkv, D, self.bits); vg.data[:] = self.gv.download()
        return kg, vg

    def exact(self, softmax_scale=None):
        kg, vg = self.host_pools()
        return omt.multi_token_decode_attention(np_of(self.q), np_of(self.k), np_of(self.v), self.cu, self.P, kg, vg, self.bt, softmax_scale)


def _check(out, exact):
    got = np_of(out).astype(np.float64)
    assert np.isfinite(got).all()
    err = np.abs(got - exact)
    assert err.max(initial=0.0) <= _bar(exact), f"max err {err.max():.3e}"
    return err


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. parity with the float64 oracle: ragged prefixes x draft lengths (0, 63 / 64 / 65 boundaries, 16 tokens), KV4 / KV8, GQA
# ---------------------------------------------------------------------------------------------------------------------------------
PREFIX = [0, 1, 63, 64, 65, 1000, 62, 5, 127]
DRAFT = [5, 16, 0, 2, 1, 3, 16, 1, 4]


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("hq,hkv", [(1, 1), (4, 1), (8, 2), (32, 8), (64, 64)])
def test_matches_oracle(dev, bits, hq, hkv):
    c = Case(dev, PREFIX, DRAFT, hq, hkv, bits, seed=hq * 10 + hkv + bits)
    out = c.attend()
    torch.cuda.synchronize()
    assert out.shape == c.q.shape and out.dtype == torch.half
    _check(out, c.exact())


def test_softmax_scale(dev):
    c = Case(dev, [70, 3, 200], [4, 7, 1], 8, 2, 4, seed=9)
    out = c.attend(softmax_scale=0.05)
    torch.cuda.synchronize()
    _check(out, c.exact(softmax_scale=0.05))


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. equals sequential decoding: n single_query_attention steps on one copy of the cache, append_at + the new op on another
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
def test_equals_sequential_decode(dev, bits):
    from qserve_b200 import backend
    hq, hkv = 32, 8
    P, N = [1, 63, 64, 1000, 130], [4, 2, 16, 3, 1]
    c = Case(dev, P, N, hq, hkv, bits, seed=50 + bits)
    dec_pools = (GpuPool(c.kp, dev), GpuPool(c.vp, dev))  # the pristine pages, before the append
    table1 = kv_pointer_table(dec_pools[0], dec_pools[1], c.bt, dev)
    dec = torch.empty_like(c.q)
    for i in range(max(N)):
        act = [b for b in range(len(P)) if i < N[b]]
        rows = torch.tensor([int(c.cu[b]) + i for b in act], device=dev)
        x = torch.from_numpy(c.raw).to(dev)[rows]
        q, k, v = (t.reshape(len(act), -1, D) for t in x.split([hq * D, hkv * D, hkv * D], dim=-1))
        lens = torch.tensor([P[b] + i + 1 for b in act], dtype=torch.int32, device=dev)
        dec[rows] = backend.single_query_attention(q, k, v, table1[torch.tensor(act, device=dev)].contiguous(), lens, None, 8192, 64, c.spt,
                                                   int(lens.max()), D, ROPE, True, bits == 4, True)
    new = c.attend()
    torch.cuda.synchronize()
    assert torch.equal(dec_pools[0].t, c.gk.t) and torch.equal(dec_pools[1].t, c.gv.t), "decode and append_at wrote different pages"
    exact = c.exact()
    err_new = _check(new, exact).reshape(len(exact), -1).max(axis=1)
    err_dec = _check(dec, exact).reshape(len(exact), -1).max(axis=1)
    # per token: no further from the truth than 1.5x the decode kernel (+ half an fp16 ulp at |x| < 1: both round their result once)
    assert (err_new <= 1.5 * err_dec + 2.5e-4).all(), (err_new, err_dec)


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. n = 1 is a decode step
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
def test_one_token_agrees_with_decode(dev, bits):
    from qserve_b200 import backend
    hq, hkv = 32, 8
    P = [0, 1, 63, 64, 65, 1000]
    c = Case(dev, P, [1] * len(P), hq, hkv, bits, seed=60 + bits)
    dec_pools = (GpuPool(c.kp, dev), GpuPool(c.vp, dev))
    B = len(P)
    q, k, v = (t.reshape(B, -1, D) for t in torch.from_numpy(c.raw).to(dev).split([hq * D, hkv * D, hkv * D], dim=-1))
    lens = torch.tensor([p + 1 for p in P], dtype=torch.int32, device=dev)
    dec = backend.single_query_attention(q, k, v, kv_pointer_table(dec_pools[0], dec_pools[1], c.bt, dev), lens, None, 8192, 64, c.spt, max(P) + 1, D,
                                         ROPE, True, bits == 4, True)
    new = c.attend()
    torch.cuda.synchronize()
    exact = c.exact()
    _check(new, exact)
    _check(dec, exact)
    assert float((new.float() - dec.float()).abs().max()) <= _bar(exact)


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. context splits and column parts
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,N,hq,hkv", [
    ([8000], [4], 32, 8),             # one sequence: many context splits
    ([7999], [16], 32, 8),            # 4 x 16 columns per KV head, many splits
    ([300, 200], [16, 9], 32, 8),     # several column parts, one split
    ([8000, 0, 64], [3, 16, 0], 8, 8),  # G = 1, splits, empty and ragged drafts
])
def test_splits_and_column_parts(dev, P, N, hq, hkv):
    c = Case(dev, P, N, hq, hkv, 4, seed=sum(P) + sum(N))
    out = c.attend()
    torch.cuda.synchronize()
    _check(out, c.exact())


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. determinism and CUDA-graph capture
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,N", [([3000], [5]), ([65, 1000, 0, 300], [4, 16, 2, 1])])
def test_deterministic_and_graph_capturable(dev, P, N):
    c = Case(dev, P, N, 32, 8, 4, seed=11)
    pristine = torch.from_numpy(c.raw).to(dev)
    o1 = c.attend()
    o2 = c.attend()
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    pages_k, pages_v = c.gk.t.clone(), c.gv.t.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
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
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, o1)
    assert torch.equal(c.gk.t, pages_k) and torch.equal(c.gv.t, pages_v)


# ---------------------------------------------------------------------------------------------------------------------------------
# 6. full size: Llama-3-8B heads, 64 x (1024 prefix + 4 drafts), KV4, against a float32 torch reference on the device
# ---------------------------------------------------------------------------------------------------------------------------------
def test_llama3_8b_full_size(dev):
    B, P, n, hq, hkv = 64, 1024, 4, 32, 8
    c = Case(dev, [P] * B, [n] * B, hq, hkv, 4, seed=3)
    out = c.attend()
    kg, vg = c.host_pools()
    G = hq // hkv
    limit = P + torch.arange(n, device=dev)
    mask = torch.arange(P + n - 1, device=dev)[None, :] >= limit[:, None]  # [n, P + n - 1]: cache position >= P + i
    worst = 0.0
    for b in range(B):
        s = slice(int(c.cu[b]), int(c.cu[b + 1]))
        kc = torch.from_numpy(oprefix.dequant_prefix(kg, c.bt[b], P + n - 1)).to(dev).float().repeat_interleave(G, dim=1)  # [P+n-1, Hq, D]
        vc = torch.from_numpy(oprefix.dequant_prefix(vg, c.bt[b], P + n - 1)).to(dev).float().repeat_interleave(G, dim=1)
        q = c.q[s].float()                                   # [n, Hq, D]
        ko, vo = c.k[s].float().repeat_interleave(G, dim=1), c.v[s].float().repeat_interleave(G, dim=1)
        sc = torch.einsum("ihd,thd->hit", q, kc).masked_fill(mask[None], float("-inf"))
        own = (q * ko).sum(-1).transpose(0, 1)[..., None]    # [Hq, n, 1]
        p = torch.softmax(torch.cat([sc, own], dim=-1) * D ** -0.5, dim=-1)
        ref = torch.einsum("hit,thd->ihd", p[..., :-1], vc) + p[..., -1].transpose(0, 1)[..., None] * vo
        worst = max(worst, float((out[s].float() - ref).abs().max()))
    assert worst <= 3e-3, worst


# ---------------------------------------------------------------------------------------------------------------------------------
# 7. argument errors
# ---------------------------------------------------------------------------------------------------------------------------------
def test_argument_errors(dev):
    from qserve_b200 import backend
    c = Case(dev, [70, 3], [5, 2], 4, 2, 4, seed=1)
    base = dict(q=c.q, k=c.k, v=c.v, cu_seqlens=c.cu_d, max_seqlen=5, prefix_lens=c.prefix_d, max_prefix_len=70, kv_pointers=c.table,
                tokens_per_block=64, size_per_token=c.spt, int4_kv_cache=True)
    backend.multi_token_decode_attention(**base)  # valid

    def bad(**kw):
        with pytest.raises(RuntimeError):
            backend.multi_token_decode_attention(**{**base, **kw})

    bad(max_seqlen=0)
    bad(max_seqlen=17)
    bad(q=c.q[..., :64], k=c.k[..., :64], v=c.v[..., :64])   # head_dim != 128
    bad(tokens_per_block=32)
    bad(size_per_token=c.spt * 2)                             # KV8 size with the KV4 flag
    bad(max_prefix_len=c.n_blocks * 64)                       # page table too short
    bad(kv_pointers=c.table[:, :, :1].contiguous())
    bad(q=c.q.cpu(), k=c.k.cpu(), v=c.v.cpu())                # CPU tensors
    bad(prefix_lens=c.prefix_d.cpu())
    bad(q=c.q.float(), k=c.k.float(), v=c.v.float())          # dtypes
    bad(prefix_lens=c.prefix_d.long())
    bad(cu_seqlens=c.cu_d.long())
    bad(k=c.k[:-1], v=c.v[:-1])
    if torch.cuda.device_count() > 1:                         # every tensor on q's device
        bad(k=c.k.to("cuda:1"), v=c.v.to("cuda:1"))
        bad(cu_seqlens=c.cu_d.to("cuda:1"))
        bad(kv_pointers=c.table.to("cuda:1"))


def test_workspace_reused_across_shapes(dev):
    """The library workspace is shared by every shape: the split partials of a long single-sequence verify must not leave non-zero words
    where the split counters of the next shape live."""
    a = Case(dev, [7999], [16], 32, 8, 4, seed=21)
    a.attend()
    b = Case(dev, [65, 1000, 0, 300], [4, 16, 2, 1], 32, 8, 4, seed=22)
    o1, o2 = b.attend(), b.attend()
    torch.cuda.synchronize()
    assert torch.equal(o1, o2)
    _check(o1, b.exact())


# ---------------------------------------------------------------------------------------------------------------------------------
# 8. the decode runner's verify step against n eager decode steps
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["w4a8kv4", "w4a8kv8"])
def test_runner_verify_equals_sequential_decode(dev, precision):
    from qserve_b200.decode import DecodeRunner
    B, ctx, n = 5, 130, 4
    seq = DecodeRunner("tiny", precision, batch=B, ctx=ctx, device=dev, seed=3, verify_len=n)
    ver = DecodeRunner("tiny", precision, batch=B, ctx=ctx, device=dev, seed=3, verify_len=n)
    tokens = (torch.arange(B * n, device=dev).view(B, n) * 37) % seq.cfg.vocab
    with torch.no_grad():
        want = []
        for i in range(n):  # decode steps at positions ctx .. ctx + n - 1
            seq.context_lens.fill_(ctx + 1 + i)
            seq.max_seq_len = ctx + 1 + i
            want.append(seq._forward_fused(tokens[:, i].contiguous(), return_logits=True).float())
        want = torch.stack(want, dim=1)
        got = ver.verify_forward(tokens, return_logits=True).float()
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert float((got - want).abs().max()) <= 1e-2 * float(want.abs().max())
    assert torch.equal(seq.kpools[0], ver.kpools[0]) and torch.equal(seq.vpools[0], ver.vpools[0])  # layer 0: the same bytes appended
    # the verify graph replays bitwise what the eager step computes
    with torch.no_grad():
        eager = ver.verify_forward(tokens).clone()
    ver.v_tokens_in.copy_(tokens)
    ver.capture_verify(n)
    ver.verify_step(n)
    torch.cuda.synchronize()
    assert torch.equal(ver.v_tokens_out, eager)
    assert torch.equal(ver.last_verify_logits.float(), got)
