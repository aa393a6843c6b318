"""GPU: the paged-attention, prompt-attention and append kernels at GQA group sizes that are not powers of two, on head-tagged needle inputs
(oracle/gqa_needles.py): every column (query head x row or member) of a KV head has its own orthogonal query and its own needle, so a
column -> (token, head) mistake at an n8-tile or column-part seam, a wrong first head of a decode head group or a wrong KV head of a query
head moves the output by many bars (test_oracle_gqa_needles.py).

G = 3 (Llama-3.2-3B, 24 / 8), 5 (Qwen2.5-14B / 32B, 40 / 8), 6 (Qwen2.5-1.5B, 12 / 2), 7 (Qwen2.5-7B 28 / 4, and at TP = 2 14 / 2) and the
synthetic 12 (24 / 2: decode head groups 8 + 4) and 20 (40 / 2: 8 + 8 + 4); KV4 and KV8.  Every attention comparison uses the bar of
oracle/needles.py `exact`, err / bar <= 1, and prints the worst ratio as a NEEDLE-RATIO line.
"""
import numpy as np
import pytest
import torch

from oracle import gqa_needles as gq
from oracle import kv
from oracle import needles as nd
from oracle import prefix as oprefix
from oracle import tree as otree
from oracle.kv import PagePool
from tests.test_gpu_attention import _check_pages
from tests.test_gpu_attention_needles import _ratio, _report, _run_chunk, _sms
from tests.test_oracle_gqa_needles import (BITS, CHAIN, DECODE, PROMPT_FLASH, PROMPT_HEADS, PROMPT_PREFIX, SHARED_GROUPS, SHARED_HKV,
                                           SHARED_PAGES, SHARED_SUFFIX, SHARED_G, TREE_HEADS, TREE_P, tree_masks)
from tests.util import GpuPool, kv_pointer_table, np_of, to_dev, ulp16_diff

pytestmark = pytest.mark.gpu
ROPE = 500000.0
D = 128


# ---------------------------------------------------------------------------------------------------------------------------------
# decode: single_query_attention and single_query_attention_quant
# ---------------------------------------------------------------------------------------------------------------------------------
def _decode_run(dev, c, fused=False):
    """-> (out or (codes, scale, sum), K pool bytes, V pool bytes) after the op."""
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
        out = (oq, sc, sm)
    else:
        out = fa.single_query_attention(qd, kd, vd, table, lens, None, *args, True, c.bits == 4, True)
    torch.cuda.synchronize()
    return out, gk.download(), gv.download()


def _appended(c):
    """The oracle's pools after the decode append: the rotated new key and the value quantised into slot L - 1."""
    kp, vp = PagePool(c.kp.data.shape[0], c.hkv, D, c.bits), PagePool(c.vp.data.shape[0], c.hkv, D, c.bits)
    kp.data[:], vp.data[:] = c.kp.data, c.vp.data
    for b, L in enumerate(c.lens):
        page, slot = c.bt[b, (L - 1) // 64], (L - 1) % 64
        for hk in range(c.hkv):
            nd.write_row(kp, page, slot, hk, kv.rope_neox(c.k[b, hk], L - 1, ROPE))
            nd.write_row(vp, page, slot, hk, c.v[b, hk])
    return kp, vp


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("B,Hq,Hkv,lens", DECODE)
def test_decode(dev, bits, B, Hq, Hkv, lens):
    c = gq.decode_case(11 + bits, B, Hq, Hkv, lens, bits, sms=_sms(dev))
    nsplit = nd.decode_splits(B, Hq, Hkv, max(lens), _sms(dev))
    assert (nsplit > 1) == (max(lens) > 512), "every configuration plans context splits exactly when its longest sequence exceeds 512"
    out, k_gpu, v_gpu = _decode_run(dev, c)
    want, bar = gq.decode_exact(c)
    worst = _ratio(np_of(out), want, bar, f"decode G={c.G} splits={nsplit}")
    _report(f"gqa-decode kv{bits} {Hq}/{Hkv} {lens} splits={nsplit}", worst)
    kp_o, vp_o = _appended(c)
    _check_pages(kp_o, vp_o, k_gpu, v_gpu, c.bt, lens)
    # the fused-quant form equals quantising the fp16 output, bit for bit (per-token counters over every head group of the row)
    import qserve_backend.fused_kernels as fk
    o16 = out.reshape(B, -1).contiguous()
    q1 = torch.empty((B, Hq * D), dtype=torch.int8, device=dev)
    s1, m1 = torch.empty(B, dtype=torch.half, device=dev), torch.empty(B, dtype=torch.half, device=dev)
    fk.invoke_quant_fuse_sum(q1, o16, m1, s1)
    (q2, s2, m2), _, _ = _decode_run(dev, c, fused=True)
    torch.cuda.synchronize()
    assert torch.equal(q1, q2) and torch.equal(s1.view(torch.int16), s2.view(torch.int16)) and torch.equal(m1.view(torch.int16), m2.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------------------
# multi_token_decode_attention: chain and tree verify
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("P,N,Hq,Hkv", CHAIN)
def test_chain_verify(dev, bits, P, N, Hq, Hkv):
    c = gq.chunk_case(21 + bits, "chain", P, N, Hq, Hkv, bits)
    out, want, bar = _run_chunk(dev, c)
    worst = _ratio(out, want, bar, f"chain G={c.G} N={N}")
    _report(f"gqa-chain kv{bits} {Hq}/{Hkv} P={P} N={N}", worst)


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("Hq,Hkv", TREE_HEADS)
def test_tree_verify(dev, bits, Hq, Hkv):
    masks = tree_masks()
    c = gq.chunk_case(31 + bits, "tree", TREE_P, [len(m) for m in masks], Hq, Hkv, bits, masks=masks)
    out, want, bar = _run_chunk(dev, c)
    worst = _ratio(out, want, bar, f"tree G={c.G}")
    _report(f"gqa-tree kv{bits} {Hq}/{Hkv}", worst)


# ---------------------------------------------------------------------------------------------------------------------------------
# shared_prefix_decode_attention
# ---------------------------------------------------------------------------------------------------------------------------------
def _shared_run(dev, c, table, **kw):
    from qserve_b200 import backend as ext
    gk, gv = GpuPool(c.kp, dev), GpuPool(c.vp, dev)
    t = kv_pointer_table(gk, gv, table, dev)
    layout = ext.shared_prefix_layout(c.groups, c.pages, c.B, device=dev)
    q, k, v = to_dev(c.q, dev), to_dev(c.k, dev), to_dev(c.v, dev)
    lens = torch.tensor(c.lens, dtype=torch.int32, device=dev)
    out = ext.shared_prefix_decode_attention(q, k, v, t, lens, layout, 64, c.hkv * D * c.bits // 8, max(c.lens), D, ROPE, c.bits == 4, True, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("G", SHARED_G)
def test_shared_prefix(dev, bits, G):
    """Groups of 1, 2, 3, 5 and 18 members (G = 7: 7 to 126 columns of (member, head)), members 37 positions apart, two rows in no
    group; the children's shared table entries point at a NaN page."""
    from qserve_b200 import backend as ext
    c = gq.SharedCase(41 + bits + G, G * SHARED_HKV, SHARED_HKV, bits, SHARED_GROUPS, SHARED_PAGES, SHARED_SUFFIX)
    out = _shared_run(dev, c, c.poisoned)
    want, bar = c.exact()
    worst = _ratio(np_of(out), want, bar, f"shared prefix G={G}")
    _report(f"gqa-shared-prefix kv{bits} G={G}", worst)
    o16 = out.reshape(c.B, -1).contiguous()
    q1 = torch.empty((c.B, c.hq * D), dtype=torch.int8, device=dev)
    s1, m1 = torch.empty(c.B, dtype=torch.half, device=dev), torch.empty(c.B, dtype=torch.half, device=dev)
    ext.invoke_quant_fuse_sum(q1, o16, m1, s1)
    q2, s2, m2 = torch.empty_like(q1), torch.empty_like(s1), torch.empty_like(m1)
    assert _shared_run(dev, c, c.poisoned, out_q=q2, out_scale=s2, out_sum=m2) is None
    assert torch.equal(q1, q2) and torch.equal(s1.view(torch.int16), s2.view(torch.int16)) and torch.equal(m1.view(torch.int16), m2.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------------------
# prompt kernels: prefix_prefill_attention and flash_attn_varlen_func
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("Hq,Hkv", PROMPT_HEADS)
def test_prefix_prefill(dev, bits, Hq, Hkv):
    P, N = PROMPT_PREFIX
    c = gq.prompt_case(51 + bits, P, N, Hq, Hkv, bits)
    out, want, bar = _run_chunk(dev, c)
    worst = _ratio(out, want, bar, f"prefix prefill {Hq}/{Hkv}")
    _report(f"gqa-prefix-prefill kv{bits} {Hq}/{Hkv}", worst)


@pytest.mark.parametrize("Hq,Hkv", PROMPT_HEADS)
def test_flash_attn_varlen(dev, Hq, Hkv):
    """The prompt kernel without a prefix: the rows as apply_bias_rope_update_kv_cache rotated them, over themselves (causal)."""
    from qserve_b200 import backend
    P, N = PROMPT_FLASH
    c = gq.prompt_case(61, P, N, Hq, Hkv, 8)
    T = sum(N)
    qkv = to_dev(c.qkv, dev)
    cu = to_dev(c.cu, dev)
    pad = backend.compute_padding_offsets(cu, max(N), T)
    backend.apply_bias_rope_update_kv_cache(qkv, torch.tensor(N, dtype=torch.int32, device=dev), pad, None, Hq, Hkv, max(N), 64, Hkv * D, D, ROPE,
                                            8192, True, False, True)
    q, k, v = qkv.split([Hq * D, Hkv * D, Hkv * D], dim=-1)
    q, k, v = q.reshape(T, Hq, D), k.reshape(T, Hkv, D), v.reshape(T, Hkv, D)
    out = backend.flash_attn_varlen_func(q, k, v, cu, cu, max(N), max(N), dropout_p=0.0, causal=True)
    torch.cuda.synchronize()
    want, bar = gq.prompt_exact(c, np_of(q), np_of(k), np_of(v), c.kp, c.vp)
    worst = _ratio(np_of(out), want, bar, f"flash {Hq}/{Hkv}")
    _report(f"gqa-flash {Hq}/{Hkv}", worst)


# ---------------------------------------------------------------------------------------------------------------------------------
# append kernels: apply_bias_rope_update_kv_cache, ..._at and the tree form
# ---------------------------------------------------------------------------------------------------------------------------------
def _check_append(qkv0, got, want, hq, hkv, kg, kp_o, vg, vp_o):
    """The tolerance of test_gpu_attention.py::test_prefill_rope_append_and_padding_offsets: v untouched, rotated q / k within 2 ulps (at
    most 2 % of them off) and 2e-3, V pages bit-exact, K scales / zeros within 1 ulp and codes within 1 LSB (at most 1 % off)."""
    n = (hq + hkv) * D
    assert np.array_equal(got[:, n:], qkv0[:, n:])
    d = ulp16_diff(got[:, :n], want[:, :n])
    big = np.abs(want[:, :n].astype(np.float32)) > 2e-2
    assert d[big].max() <= 2 and (d[big] > 0).mean() < 0.02
    assert np.abs(got[:, :n].astype(np.float32) - want[:, :n].astype(np.float32)).max() <= 2e-3
    assert np.array_equal(vg.data, vp_o.data), "V pages must be bit-exact"
    assert ulp16_diff(kg.scales(), kp_o.scales()).max() <= 1 and ulp16_diff(kg.zeros(), kp_o.zeros()).max() <= 1
    cg, co = kg.codes(), kp_o.codes()
    if kp_o.bits == 4:
        cg, co = kv.unpack_nibbles(cg), kv.unpack_nibbles(co)
    dd = np.abs(cg.astype(np.int32) - co.astype(np.int32))
    assert dd.max() <= 1 and (dd > 0).mean() < 0.01


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("G", [3, 5, 7, 12])
@pytest.mark.parametrize("form", ["plain", "at", "tree"])
def test_append(dev, bits, G, form):
    from qserve_b200 import backend
    rng = np.random.default_rng(71 + 10 * G + bits)
    hkv = 2
    hq = G * hkv
    if form == "tree":
        masks = tree_masks()
        lens = np.array([len(m) for m in masks], np.int32)
        start = np.array([65, 63, 1], np.int32)
    else:
        lens = np.array([5, 70, 1, 130], np.int32)
        start = np.array([0, 64, 200, 1], np.int32) if form == "at" else np.zeros(4, np.int32)
    B, T, maxlen = len(lens), int(lens.sum()), int(lens.max())
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pad = kv.compute_padding_offsets(cu, maxlen, T)
    nb = (int((start + lens).max()) + 63) // 64
    bt = np.arange(B * nb).reshape(B, nb)
    kp, vp = PagePool(B * nb, hkv, D, bits, rng), PagePool(B * nb, hkv, D, bits, rng)
    gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
    table = kv_pointer_table(gk, gv, bt, dev)
    qkv = rng.standard_normal((T, (hq + 2 * hkv) * D)).astype(np.float16)
    qkv_d = to_dev(qkv, dev)
    lens_d, pad_d = to_dev(lens, dev), backend.compute_padding_offsets(to_dev(cu, dev), maxlen, T)
    args = (hq, hkv, maxlen, 64, hkv * D * bits // 8, D, ROPE, 8192, True, bits == 4, True)
    if form == "plain":
        backend.apply_bias_rope_update_kv_cache(qkv_d, lens_d, pad_d, table, *args)
        want = kv.prefill_rope_append(qkv.copy(), lens, pad, kp, vp, bt, hq, hkv, maxlen, ROPE, 8192)
    elif form == "at":
        backend.apply_bias_rope_update_kv_cache_at(qkv_d, lens_d, pad_d, to_dev(start, dev), table, *args)
        want = oprefix.prefill_rope_append_at(qkv.copy(), lens, pad, start, kp, vp, bt, hq, hkv, maxlen, ROPE, 8192)
    else:
        tm = np.concatenate([np.asarray(m, np.int64) for m in masks]).astype(np.int32)
        backend.apply_bias_rope_update_kv_cache_at(qkv_d, lens_d, pad_d, to_dev(start, dev), table, *args, tree_mask=to_dev(tm, dev))
        want = otree.tree_rope_append(qkv.copy(), lens, pad, start, tm, kp, vp, bt, hq, hkv, maxlen, ROPE, 8192)
    torch.cuda.synchronize()
    kg = PagePool(B * nb, hkv, D, bits); kg.data[:] = gk.download()
    vg = PagePool(B * nb, hkv, D, bits); vg.data[:] = gv.download()
    _check_append(qkv, np_of(qkv_d), want, hq, hkv, kg, kp, vg, vp)
