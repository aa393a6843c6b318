"""GPU: pinned output bits of the kernels that stream the paged INT4 / INT8 KV cache (tests/golden/paged_attn_bits.npz).

Covers, KV4 and KV8 each:
  * multi_token_decode_attention (chain): one n8 tile (G n <= 8) and two, several column parts, with and without context splits, a sequence
    without draft tokens, a group size that is not a power of two (14 / 2), the default and an explicit softmax_scale;
  * tree_decode_attention: the same shapes with branching ancestor masks;
  * shared_prefix_decode_attention: one and two n8 tiles in the shared pass, shared-pass and row-pass context splits and none, rows in no
    group, fp16 output and the fused quantisation (codes, scale, sum);
  * single_query_attention(_quant): idle rows (length 0) among live ones, and G = 7 and G = 20 (head groups of 8 + 8 + 4), with splits;
  * the pages after every call that appends;
  * qs_multi_token_attention_workspace_bytes and qs_shared_prefix_attention_workspace_bytes over a small sweep (they follow the planned
    split count).
The inputs are rebuilt from fixed seeds with the builders of the attention suites; only the outputs are stored, tensors of more than 4096
elements and the page pools as SHA-256 digests.  Floats are compared as their bits.  The fixture was written on an H100 with 132 SMs: the
context-split count, and so the summation order, depends on the SM count."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_attention import ROPE, _mk
from tests.test_gpu_multi_token_attention import Case
from tests.test_gpu_shared_prefix_attention import LONG, MIXED, _build, _Dev
from tests.test_gpu_tree_verify import TreeCase, tree
from tests.util import GpuPool, kv_pointer_table, to_dev

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "paged_attn_bits.npz")
D = 128
_BIG = 4096  # tensors with more elements are stored as their digest

MULTI_TOKEN = {  # name: (prefix lengths, draft lengths, Hq, Hkv)
    "nt1": ([70, 3, 200], [2, 0, 1], 8, 2),                 # G n <= 8: one n8 tile; a sequence without draft tokens
    "nt1_splits": ([5000], [2], 8, 2),                      # one tile, context splits
    "nt2_parts": ([300, 200, 0, 64], [16, 9, 0, 5], 8, 2),  # four column parts of 16 columns, no splits
    "nt2_splits": ([8000], [4], 32, 8),                     # two tiles, context splits
    "g7": ([130, 1000, 64], [3, 1, 0], 14, 2),              # G = 7: columns of one token straddle the tiles; splits
}
SCALED = ("nt1", "g7")  # also run with an explicit softmax_scale
SHARED_PREFIX = {  # name: (G, groups, shared pages, batch)
    "nt1_splits": (2, *LONG),            # 6 columns: one tile; S = 64 gives splits in both passes; rows 2 and 6 in no group
    "nt2_splits": (4, *LONG),            # 12 columns: two tiles
    "nt2_mixed": (4, *MIXED),            # groups of up to 33 rows: several column parts; rows in no group
    "nosplit": (2, [[0, 2], [1, 3, 4]], [4, 2], 5),  # no split in either pass
}
DECODE = {  # name: (B, Hq, Hkv, lengths)
    "idle": (4, 8, 2, [0, 65, 0, 300]),  # length 0: an idle row
    "g7": (3, 14, 2, [1, 200, 700]),
    "g20": (3, 40, 2, [0, 90, 257]),     # head groups of 8 + 8 + 4
    "g20_splits": (1, 40, 2, [1500]),
}
WS_MULTI_TOKEN = [  # (batch, tokens, max_seqlen, max_prefix_len, Hq, Hkv)
    (1, 4, 4, 8000, 32, 8), (3, 3, 2, 200, 8, 2), (64, 256, 4, 1024, 32, 8), (4, 30, 16, 300, 8, 2), (3, 4, 3, 1000, 14, 2), (1, 2, 2, 5000, 8, 2),
]
WS_SHARED_PREFIX = [  # (batch, Hq, Hkv, timestep, groups, max_group, max_pages)
    (7, 4, 2, 4196, 2, 3, 64), (80, 8, 2, 1124, 8, 33, 16), (5, 4, 2, 356, 2, 3, 4), (64, 32, 8, 1100, 1, 64, 16), (64, 32, 8, 1100, 0, 0, 0),
]


def _digest(tensors) -> torch.Tensor:
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return torch.from_numpy(np.frombuffer(h.digest(), np.uint8).copy())


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.half else t


def _put(res, key, t):
    t = _bits(t.detach())
    res[key] = _digest([t]) if t.numel() > _BIG else t.cpu().clone()


def multi_token_outputs(dev, name, bits, tree_masks):
    P, N, hq, hkv = MULTI_TOKEN[name]
    seed = 7000 + 10 * list(MULTI_TOKEN).index(name) + bits
    if tree_masks:
        c = TreeCase(dev, P, [tree("random", n, seed=i + 1) if n else [] for i, n in enumerate(N)], hq, hkv, bits, seed=seed)
    else:
        c = Case(dev, P, N, hq, hkv, bits, seed=seed)
    res = {"pages": _digest([c.gk.t, c.gv.t])}
    _put(res, "out", c.attend())
    if name in SCALED:
        _put(res, "out_scaled", c.attend(softmax_scale=0.05))
    torch.cuda.synchronize()
    return res


def shared_prefix_outputs(dev, name, bits):
    G, groups, pages, batch = SHARED_PREFIX[name]
    d = _Dev(dev, _build(8000 + 10 * list(SHARED_PREFIX).index(name) + bits, G, bits, groups, pages, batch), groups, pages, bits)
    res = {}
    gk, gv = d.pools()
    _put(res, "out", d.shared(gk, gv, table="poisoned"))
    res["pages"] = _digest([gk.t, gv.t])
    gk, gv = d.pools()
    oq = torch.empty((batch, d.Hq * D), dtype=torch.int8, device=dev)
    sc = torch.empty(batch, dtype=torch.half, device=dev)
    sm = torch.empty(batch, dtype=torch.half, device=dev)
    d.shared(gk, gv, out_q=oq, out_scale=sc, out_sum=sm)
    _put(res, "codes", oq)
    _put(res, "scale", sc)
    _put(res, "sum", sm)
    res["pages_quant"] = _digest([gk.t, gv.t])
    torch.cuda.synchronize()
    return res


def decode_outputs(dev, name, bits):
    import qserve_backend.fused_attention as fa
    from qserve_b200 import backend as ext
    B, Hq, Hkv, lens = DECODE[name]
    kp, vp, bt, q, k, v = _mk(np.random.default_rng(9500 + 10 * list(DECODE).index(name) + bits), B, Hq, Hkv, lens, bits)
    args = (8192, 64, Hkv * D * bits // 8, int(max(lens)), D, ROPE)
    res = {}
    for fused in (False, True):
        gk, gv = GpuPool(kp, dev), GpuPool(vp, dev)
        table = kv_pointer_table(gk, gv, bt, dev)
        qd, kd, vd = to_dev(q, dev), to_dev(k, dev), to_dev(v, dev)
        lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
        if fused:
            oq = torch.empty((B, Hq * D), dtype=torch.int8, device=dev)
            sc = torch.empty(B, dtype=torch.half, device=dev)
            sm = torch.empty(B, dtype=torch.half, device=dev)
            ext.single_query_attention_quant(qd, kd, vd, table, lens_d, *args, bits == 4, True, oq, sc, sm)
            _put(res, "codes", oq)
            _put(res, "scale", sc)
            _put(res, "sum", sm)
            res["pages_quant"] = _digest([gk.t, gv.t])
        else:
            _put(res, "out", fa.single_query_attention(qd, kd, vd, table, lens_d, None, *args, True, bits == 4, True))
            res["pages"] = _digest([gk.t, gv.t])
    torch.cuda.synchronize()
    return res


def workspace_sizes():
    from qserve_b200.backend import lib
    mt = [lib.qs_multi_token_attention_workspace_bytes(*s, int4) for int4 in (1, 0) for s in WS_MULTI_TOKEN]
    sp = [lib.qs_shared_prefix_attention_workspace_bytes(*s, int4) for int4 in (1, 0) for s in WS_SHARED_PREFIX]
    return {"ws_multi_token": torch.tensor(mt, dtype=torch.int64), "ws_shared_prefix": torch.tensor(sp, dtype=torch.int64)}


KINDS = {
    "chain": (MULTI_TOKEN, lambda dev, name, bits: multi_token_outputs(dev, name, bits, False)),
    "tree": (MULTI_TOKEN, lambda dev, name, bits: multi_token_outputs(dev, name, bits, True)),
    "shared": (SHARED_PREFIX, shared_prefix_outputs),
    "decode": (DECODE, decode_outputs),
}
PARAMS = [(kind, name) for kind, (cases, _) in KINDS.items() for name in cases]


def all_outputs(dev):
    """Every pinned array, keyed as in the fixture."""
    res = {key: t for key, t in workspace_sizes().items()}
    for kind, name in PARAMS:
        for bits in (4, 8):
            for key, t in KINDS[kind][1](dev, name, bits).items():
                res[f"{kind}_{name}_kv{bits}_{key}"] = t
    return res


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("kind,name", PARAMS)
def test_output_bits_are_pinned(dev, kind, name, bits):
    want = np.load(GOLDEN)
    got = KINDS[kind][1](dev, name, bits)
    prefix = f"{kind}_{name}_kv{bits}_"
    assert sorted(got) == sorted(k[len(prefix):] for k in want.files if k.startswith(prefix))
    for key, t in got.items():
        assert torch.equal(t, torch.from_numpy(want[prefix + key])), key


def test_workspace_sizes_are_pinned(dev):
    want = np.load(GOLDEN)
    for key, t in workspace_sizes().items():
        assert torch.equal(t, torch.from_numpy(want[key])), key
