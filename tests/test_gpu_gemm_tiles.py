"""GPU parity of every (tokens per tile, cluster split) plan of the decode GEMM: each forced tile of 32 / 64 / 128 tokens with each forced
split S in {1, 2, 4, 8}, at token counts on both sides of every tile boundary.  Split-K partials are INT32 and reduced in integer adds, so
every plan must give the oracle's INT32 accumulators and fp16 outputs bit for bit, and a partial token tile must write nothing past row M.
K = 384 is included: K % 256 == 128, so the last pipeline stage is half zero-filled.  One test replays a CUDA graph of split launches with
programmatic dependent launch on: the split-K receive buffer aliases the pipeline rings, so a partial that arrived late or early would show."""
import numpy as np
import pytest
import torch

from oracle import ops, w4a8
from tests.util import to_dev

pytestmark = pytest.mark.gpu

LLAMA3_8B = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]   # qkv, o, gate_up, down
QWEN72B_TP4 = [(6144, 8192), (8192, 2048), (12288, 8192), (8192, 6144)]  # per-rank shards at TP = 4
ODD_K = [(256, 384)]
TOKENS = (1, 31, 32, 33, 63, 64, 65, 128, 200)
PAD_ROWS = 8  # sentinel rows behind row M


def _problem(mode, N, K, dev):
    """Inputs of max(TOKENS) tokens on the device, a launcher for their first M rows, and the oracle's outputs as device tensors.  Every
    row depends only on its own token, so one oracle GEMM serves every M."""
    rng = np.random.default_rng(N * 7 + K)
    x = rng.standard_normal((max(TOKENS), K)).astype(np.float16)
    aq, sa, asum = ops.quant_per_token(x)
    if mode == "chn":
        import qserve_backend.qgemm_w4a8_per_chn as op
        _, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        d_aq, d_qw, d_s1, d_sa, d_s1z, d_asum = (to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum))
        call = lambda M, out, acc: op.gemm_forward_cuda(d_aq[:M], d_qw, d_s1, d_sa[:M], d_s1z, d_asum[:M], out, _acc_out=acc)  # noqa: E731
    elif mode == "grp":
        import qserve_backend.qgemm_w4a8_per_group as op
        _, qw, s1, s2s, s2z = w4a8.synth_per_group(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_group(aq, qw, s2z, s2s, s1, sa, return_acc=True)
        d_aq, d_qw, d_s2z, d_s2s, d_s1, d_sa = (to_dev(a, dev) for a in (aq, qw, s2z, s2s, s1, sa))
        call = lambda M, out, acc: op.gemm_forward_cuda(d_aq[:M], d_qw, d_s2z, d_s2s, d_s1, d_sa[:M], out, _acc_out=acc)  # noqa: E731
    else:
        import qserve_backend.qgemm_w8a8 as op
        w = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        sw = rng.uniform(0.001, 0.01, size=N).astype(np.float16)
        out_o, acc_o = w4a8.gemm_w8a8(aq, w, sw, sa, return_acc=True)
        d_aq, d_w, d_sw, d_sa = (to_dev(a, dev) for a in (aq, w, sw, sa))
        call = lambda M, out, acc: op.w8a8_gemm_forward_cuda(d_aq[:M], d_w, d_sw, d_sa[:M], out, _acc_out=acc)  # noqa: E731
    return call, to_dev(out_o, dev).view(torch.int16), to_dev(acc_o, dev)


@pytest.mark.parametrize("N,K", LLAMA3_8B + QWEN72B_TP4 + ODD_K)
@pytest.mark.parametrize("mode", ["chn", "grp", "w8"])
def test_every_tile_and_split_bit_exact(dev, mode, N, K):
    from qserve_b200._lib import lib
    call, out_o, acc_o = _problem(mode, N, K, dev)
    sentinel = torch.iinfo(torch.int32).min
    try:
        for M in TOKENS:
            for nt in (32, 64, 128):
                for split in (1, 2, 4, 8):
                    lib.qs_gemm_force_tile_tokens(nt)
                    lib.qs_gemm_force_split(split)
                    out = torch.full((M + PAD_ROWS, N), float("nan"), dtype=torch.half, device=dev)
                    acc = torch.full((M + PAD_ROWS, N), sentinel, dtype=torch.int32, device=dev)
                    call(M, out[:M], acc[:M])
                    torch.cuda.synchronize()
                    what = (M, nt, split)
                    assert torch.equal(acc[:M], acc_o[:M]), what
                    assert torch.equal(out[:M].view(torch.int16), out_o[:M]), what
                    assert bool(torch.isnan(out[M:]).all()) and bool((acc[M:] == sentinel).all()), what
    finally:
        lib.qs_gemm_force_split(0)
        lib.qs_gemm_force_tile_tokens(0)


@pytest.mark.parametrize("mode", ["chn", "grp", "w8"])
def test_split_plans_under_graph_replay_with_pdl(dev, mode):
    """Back-to-back split launches of every tile size in one CUDA graph, programmatic dependent launch on: 20 replays, every output
    equal to the oracle's every time."""
    from qserve_b200 import backend
    from qserve_b200._lib import lib
    N, K, M = 4096, 4096, 64
    call, out_o, acc_o = _problem(mode, N, K, dev)
    plans = [(nt, split) for nt in (32, 64, 128) for split in (2, 4, 8)] + [(0, 0)]
    outs = [torch.empty((M, N), dtype=torch.half, device=dev) for _ in plans]
    accs = [torch.empty((M, N), dtype=torch.int32, device=dev) for _ in plans]

    def chain():
        for (nt, split), out, acc in zip(plans, outs, accs):
            lib.qs_gemm_force_tile_tokens(nt)
            lib.qs_gemm_force_split(split)
            call(M, out, acc)

    was = backend.set_pdl(True)
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            chain()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            chain()
        for rep in range(20):
            for out, acc in zip(outs, accs):
                out.fill_(float("nan"))
                acc.zero_()
            g.replay()
            torch.cuda.synchronize()
            for plan, out, acc in zip(plans, outs, accs):
                assert torch.equal(acc, acc_o[:M]), (rep, plan)
                assert torch.equal(out.view(torch.int16), out_o[:M]), (rep, plan)
    finally:
        backend.set_pdl(was)
        lib.qs_gemm_force_split(0)
        lib.qs_gemm_force_tile_tokens(0)
