"""GPU parity: wgmma W4A8 / W8A8 GEMMs vs the CPU oracle.  INT32 accumulators bit-exact, FP16 outputs bit-exact
(the epilogue is IEEE fp32 in the reference's source order; tolerance 0 ulp) -- through the drop-in Python API.  The parity tests run
each problem on both instantiations of the kernel (_run_both): with the INT32 accumulator dump, and without it, as the decode runner
launches it."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ops, w4a8
from tests.util import bits16, np_of, to_dev, ulp16_diff

pytestmark = pytest.mark.gpu
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")


def _acts(rng, M, K):
    x = rng.standard_normal((M, K)).astype(np.float16)
    aq, sa, asum = ops.quant_per_token(x)
    return aq, sa, asum


def _run_both(dev, call, M, N):
    """call(out, acc) with acc an INT32 [M, N] tensor and again with acc=None -> (acc, fp16 out with the dump, fp16 out without), numpy.
    Both outputs are views [:M] of NaN-filled buffers whose rows past M must stay NaN."""
    outs = []
    for dump in (True, False):
        out = torch.full((M + 8, N), float("nan"), dtype=torch.half, device=dev)
        acc = torch.zeros((M, N), dtype=torch.int32, device=dev) if dump else None
        call(out[:M], acc)
        torch.cuda.synchronize()
        assert bool(torch.isnan(out[M:]).all()), dump
        outs.append(np_of(out[:M]))
        if dump:
            acc_g = np_of(acc)
    return acc_g, outs[0], outs[1]


def _report(name, acc_g, acc_o, out_g, out_o):
    os.makedirs(OUT, exist_ok=True)
    bad = np.argwhere(acc_g != acc_o)
    info = {"name": name, "acc_mismatch": int(bad.shape[0]), "acc_total": int(acc_o.size),
            "first_bad": bad[:10].tolist(), "acc_g": acc_g[tuple(bad[:10].T)].tolist() if len(bad) else [],
            "acc_o": acc_o[tuple(bad[:10].T)].tolist() if len(bad) else [],
            "bad_rows": sorted(set(bad[:, 0].tolist()))[:40], "bad_cols": sorted(set(bad[:, 1].tolist()))[:80],
            "out_max_ulp": int(ulp16_diff(out_g, out_o).max())}
    with open(os.path.join(OUT, "gemm_diag.jsonl"), "a") as f:
        f.write(json.dumps(info) + "\n")
    return info


SHAPES = [  # (M, N, K)
    (16, 128, 128), (1, 256, 256), (16, 4096, 4096), (33, 384, 512), (64, 256, 1024), (64, 4096, 4096),
    (100, 512, 640), (128, 256, 256), (200, 384, 384), (256, 256, 512), (300, 256, 256), (700, 384, 256),
    # prefill-sized M (128-token tiles): ragged last token block, K % 256 == 128, several tiles per SM
    (1000, 512, 1152), (513, 1024, 384), (2048, 768, 512),
    # wide layers at 128 < M < 512: ragged 128-token tiles (192 = 128 + 64, 448 = 3 x 128 + 64)
    (192, 19200, 512), (448, 9728, 640),
]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_w4a8_per_channel(dev, M, N, K):
    import qserve_backend.qgemm_w4a8_per_chn as op
    rng = np.random.default_rng(M * 7 + N + K)
    q, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
    aq, sa, asum = _acts(rng, M, K)
    out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
    args = [to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)]
    acc, out, out_n = _run_both(dev, lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc), M, N)
    info = _report(f"chn_{M}x{N}x{K}", acc, acc_o, out, out_o)
    assert info["acc_mismatch"] == 0, info
    assert np.array_equal(bits16(out), bits16(out_o)), info
    assert np.array_equal(bits16(out_n), bits16(out_o)), info


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_w4a8_per_group(dev, M, N, K):
    import qserve_backend.qgemm_w4a8_per_group as op
    rng = np.random.default_rng(M * 11 + N + K)
    q, qw, s1, s2s, s2z = w4a8.synth_per_group(rng, N, K)
    aq, sa, _ = _acts(rng, M, K)
    out_o, acc_o = w4a8.gemm_w4a8_per_group(aq, qw, s2z, s2s, s1, sa, return_acc=True)
    args = [to_dev(a, dev) for a in (aq, qw, s2z, s2s, s1, sa)]
    acc, out, out_n = _run_both(dev, lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc), M, N)
    info = _report(f"grp_{M}x{N}x{K}", acc, acc_o, out, out_o)
    assert info["acc_mismatch"] == 0, info
    assert np.array_equal(bits16(out), bits16(out_o)), info
    assert np.array_equal(bits16(out_n), bits16(out_o)), info


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_w8a8(dev, M, N, K):
    import qserve_backend.qgemm_w8a8 as op
    rng = np.random.default_rng(M * 13 + N + K)
    w = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
    sw = rng.uniform(0.001, 0.01, size=N).astype(np.float16)
    aq, sa, _ = _acts(rng, M, K)
    out_o, acc_o = w4a8.gemm_w8a8(aq, w, sw, sa, return_acc=True)
    args = [to_dev(a, dev) for a in (aq, w, sw, sa)]
    acc, out, out_n = _run_both(dev, lambda out, acc: op.w8a8_gemm_forward_cuda(*args, out, _acc_out=acc), M, N)
    info = _report(f"w8_{M}x{N}x{K}", acc, acc_o, out, out_o)
    assert info["acc_mismatch"] == 0, info
    assert np.array_equal(bits16(out), bits16(out_o)), info
    assert np.array_equal(bits16(out_n), bits16(out_o)), info


@pytest.mark.parametrize("split", [1, 2, 4, 8])
@pytest.mark.parametrize("mode", ["chn", "grp", "w8"])
def test_cluster_split_k_is_bit_identical(dev, split, mode):
    """INT32 partial tiles reduced through distributed shared memory: every split factor gives the same bits."""
    from qserve_b200._lib import lib
    import qserve_backend.qgemm_w4a8_per_chn as opc
    import qserve_backend.qgemm_w4a8_per_group as opg
    import qserve_backend.qgemm_w8a8 as op8
    M, N, K = 64, 512, 2048
    rng = np.random.default_rng(99)
    aq, sa, asum = _acts(rng, M, K)
    if mode == "chn":
        q, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        call = lambda out, acc: opc.gemm_forward_cuda(*[to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)], out, _acc_out=acc)
    elif mode == "grp":
        q, qw, s1, s2s, s2z = w4a8.synth_per_group(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_group(aq, qw, s2z, s2s, s1, sa, return_acc=True)
        call = lambda out, acc: opg.gemm_forward_cuda(*[to_dev(a, dev) for a in (aq, qw, s2z, s2s, s1, sa)], out, _acc_out=acc)
    else:
        w = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        sw = rng.uniform(0.001, 0.01, size=N).astype(np.float16)
        out_o, acc_o = w4a8.gemm_w8a8(aq, w, sw, sa, return_acc=True)
        call = lambda out, acc: op8.w8a8_gemm_forward_cuda(*[to_dev(a, dev) for a in (aq, w, sw, sa)], out, _acc_out=acc)
    lib.qs_gemm_force_split(split)
    try:
        for _ in range(2):
            out = torch.full((M, N), float("nan"), dtype=torch.half, device=dev)
            acc = torch.zeros((M, N), dtype=torch.int32, device=dev)
            call(out, acc)
            torch.cuda.synchronize()
            assert np.array_equal(np_of(acc), acc_o)
            assert np.array_equal(bits16(np_of(out)), bits16(out_o))
    finally:
        lib.qs_gemm_force_split(0)


def test_llama3_8b_layer_shapes_decode_b64(dev):
    """BASELINE config 2 GEMM shapes at M=64: bit-exact INT32 + FP16 against the oracle at full size."""
    import qserve_backend.qgemm_w4a8_per_chn as op
    rng = np.random.default_rng(5)
    for K, N in ((4096, 6144), (4096, 4096), (4096, 28672), (14336, 4096)):
        q, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
        aq, sa, asum = _acts(rng, 64, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        args = [to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)]
        acc, out, out_n = _run_both(dev, lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc), 64, N)
        assert np.array_equal(acc, acc_o), (K, N)
        assert np.array_equal(bits16(out), bits16(out_o)), (K, N)
        assert np.array_equal(bits16(out_n), bits16(out_o)), (K, N)


CONFIG_SHAPES = [  # BASELINE.json configs 3-5 (SURVEY.md 8d): (mode, M, N, K)
    ("grp", 64, 6144, 4096), ("grp", 64, 4096, 14336),                                  # 3: Llama-3-8B g128, decode batch 64
    ("w8", 128, 6144, 4096), ("w8", 128, 28672, 4096), ("w8", 128, 4096, 14336),        # 4: Mistral-7B W8A8, decode batch 128
    ("chn", 64, 6144, 8192), ("chn", 64, 8192, 2048), ("chn", 64, 12288, 8192), ("chn", 64, 8192, 6144),  # 5: Qwen1.5-72B, TP=4 shards
]


@pytest.mark.parametrize("mode,M,N,K", CONFIG_SHAPES)
def test_baseline_config_shapes_bit_exact(dev, mode, M, N, K):
    """The GEMM shapes of BASELINE configs 3, 4 and 5 (per-rank shards at TP=4): INT32 and FP16 bit-exact at full size."""
    rng = np.random.default_rng(N + K + M)
    aq, sa, asum = _acts(rng, M, K)
    if mode == "chn":
        import qserve_backend.qgemm_w4a8_per_chn as op
        q, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        args = [to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)]
        call = lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc)  # noqa: E731
    elif mode == "grp":
        import qserve_backend.qgemm_w4a8_per_group as op
        q, qw, s1, s2s, s2z = w4a8.synth_per_group(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_group(aq, qw, s2z, s2s, s1, sa, return_acc=True)
        args = [to_dev(a, dev) for a in (aq, qw, s2z, s2s, s1, sa)]
        call = lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc)  # noqa: E731
    else:
        import qserve_backend.qgemm_w8a8 as op
        w = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        sw = rng.uniform(0.001, 0.01, size=N).astype(np.float16)
        out_o, acc_o = w4a8.gemm_w8a8(aq, w, sw, sa, return_acc=True)
        args = [to_dev(a, dev) for a in (aq, w, sw, sa)]
        call = lambda out, acc: op.w8a8_gemm_forward_cuda(*args, out, _acc_out=acc)  # noqa: E731
    acc, out, out_n = _run_both(dev, call, M, N)
    assert np.array_equal(acc, acc_o)
    assert np.array_equal(bits16(out), bits16(out_o))
    assert np.array_equal(bits16(out_n), bits16(out_o))


@pytest.mark.parametrize("M,N,K", [(64, 28672, 4096), (16, 19072, 384), (33, 37888, 256), (1, 20480, 128), (64, 24576, 1152)])
def test_wide_layers_bit_exact(dev, M, N, K):
    """Layers with more 128-channel tiles than SMs (two CTAs per SM, several waves), including K % 256 == 128: bit-exact."""
    import qserve_backend.qgemm_w4a8_per_chn as op
    rng = np.random.default_rng(M + N + K)
    q, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
    aq, sa, asum = _acts(rng, M, K)
    out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
    args = [to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)]
    acc, out, out_n = _run_both(dev, lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc), M, N)
    assert np.array_equal(acc, acc_o)
    assert np.array_equal(bits16(out), bits16(out_o))
    assert np.array_equal(bits16(out_n), bits16(out_o))


def test_linearity_property_full_size(dev):
    """Size-independent property at prefill size (M=2048): acc(a1 + a2) == acc(a1) + acc(a2) for the INT32 accumulators."""
    import qserve_backend.qgemm_w4a8_per_chn as op
    M, N, K = 2048, 4096, 4096
    g = torch.Generator(device="cpu").manual_seed(3)
    a1 = torch.randint(-60, 60, (M, K), dtype=torch.int8, generator=g).to(dev)
    a2 = torch.randint(-60, 60, (M, K), dtype=torch.int8, generator=g).to(dev)
    qw = torch.randint(-128, 128, (N, K // 2), dtype=torch.int8, generator=g).to(dev)
    one_n = torch.ones(N, dtype=torch.half, device=dev)
    one_m = torch.ones(M, dtype=torch.half, device=dev)
    zero_n = torch.zeros(N, dtype=torch.half, device=dev)
    accs = []
    for a in (a1, a2, a1 + a2):
        out = torch.empty((M, N), dtype=torch.half, device=dev)
        acc = torch.zeros((M, N), dtype=torch.int32, device=dev)
        op.gemm_forward_cuda(a, qw, one_n, one_m, zero_n, one_m, out, _acc_out=acc)
        accs.append(acc)
    torch.cuda.synchronize()
    assert torch.equal(accs[0] + accs[1], accs[2])
    # spot-check 64 random rows against the oracle
    rows = np.random.default_rng(0).choice(M, 64, replace=False)
    acc_o = w4a8.int_matmul(np_of(a1)[rows], w4a8.unpack_w4(np_of(qw)))
    assert np.array_equal(np_of(accs[0])[rows], acc_o)


def test_invalid_shapes_raise(dev):
    import qserve_backend.qgemm_w4a8_per_chn as op
    h = lambda *s: torch.zeros(*s, dtype=torch.half, device=dev)
    i8 = lambda *s: torch.zeros(*s, dtype=torch.int8, device=dev)
    with pytest.raises(RuntimeError):  # N not a multiple of 128
        op.gemm_forward_cuda(i8(4, 128), i8(64, 64), h(64), h(4), h(64), h(4), h(4, 64))
    with pytest.raises(RuntimeError):  # K not a multiple of 128
        op.gemm_forward_cuda(i8(4, 64), i8(128, 32), h(128), h(4), h(128), h(4), h(4, 128))
    op.gemm_forward_cuda(i8(0, 128), i8(128, 64), h(128), h(0), h(128), h(0), h(0, 128))  # empty batch is a no-op
