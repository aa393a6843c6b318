"""GPU parity of every split-K plan of the decode GEMM: the automatic plan (one wave, sized by the occupancy API) and each forced cluster
split S in {1, 2, 4, 8}, at the tile size the planner picks for M.  Split-K partials are INT32 and reduced in integer adds, so every plan
must give the oracle's INT32 accumulators and fp16 outputs bit for bit, on the instantiation that dumps the accumulators and on the one
the decode runner launches (no dump)."""
import numpy as np
import pytest
import torch

from oracle import ops, w4a8
from tests.util import bits16, np_of, to_dev

pytestmark = pytest.mark.gpu

LLAMA3_8B = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]   # qkv, o, gate_up, down
MISTRAL_7B = [(6144, 4096), (28672, 4096), (4096, 14336)]                # W8A8 decode batch 128
QWEN72B_TP4 = [(6144, 8192), (8192, 2048), (12288, 8192), (8192, 6144)]  # per-rank shards at TP = 4
SMALL_M = [(M, N, K) for M in (1, 16, 33) for N, K in ((4096, 4096), (4096, 14336))]

CASES = ([("chn", 64, N, K) for N, K in LLAMA3_8B + QWEN72B_TP4] + [("grp", 64, N, K) for N, K in LLAMA3_8B]
         + [("w8", 128, N, K) for N, K in MISTRAL_7B] + [(mode, M, N, K) for mode in ("chn", "grp", "w8") for M, N, K in SMALL_M])


def _problem(mode, M, N, K, dev):
    rng = np.random.default_rng(M * 31 + N + K)
    x = rng.standard_normal((M, K)).astype(np.float16)
    aq, sa, asum = ops.quant_per_token(x)
    if mode == "chn":
        import qserve_backend.qgemm_w4a8_per_chn as op
        _, qw, s1, s1z = w4a8.synth_per_channel(rng, N, K)
        out_o, acc_o = w4a8.gemm_w4a8_per_chn(aq, qw, s1, sa, s1z, asum, return_acc=True)
        args = [to_dev(a, dev) for a in (aq, qw, s1, sa, s1z, asum)]
        call = lambda out, acc: op.gemm_forward_cuda(*args, out, _acc_out=acc)  # noqa: E731
    elif mode == "grp":
        import qserve_backend.qgemm_w4a8_per_group as op
        _, qw, s1, s2s, s2z = w4a8.synth_per_group(rng, N, K)
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
    return call, out_o, acc_o


@pytest.mark.parametrize("mode,M,N,K", CASES)
def test_every_split_plan_bit_exact(dev, mode, M, N, K):
    from qserve_b200._lib import lib
    call, out_o, acc_o = _problem(mode, M, N, K, dev)
    try:
        for split in (0, 1, 2, 4, 8):  # 0: the automatic plan
            lib.qs_gemm_force_split(split)
            for dump in (True, False):
                out = torch.full((M, N), float("nan"), dtype=torch.half, device=dev)
                acc = torch.zeros((M, N), dtype=torch.int32, device=dev) if dump else None
                call(out, acc)
                torch.cuda.synchronize()
                if dump:
                    assert np.array_equal(np_of(acc), acc_o), split
                assert np.array_equal(bits16(np_of(out)), bits16(out_o)), (split, dump)
    finally:
        lib.qs_gemm_force_split(0)
