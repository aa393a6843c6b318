"""GPU parity of the GEMM at the edges of its INT32 -> fp16 epilogue, at prompt-sized M, and behind a producer kernel under programmatic
dependent launch.  Every launch runs on both instantiations of the kernel: the one the decode runner launches (no accumulator dump) and the
one that also writes the INT32 accumulators.

  * edge cases (tests/gemm_edge_cases.py): fp16 bits equal to the oracle's (NaN by position), at every forced tile size with a split > 1,
    and at 1000 rows (the rows repeated) on the unsplit 128-token tile.  The activations are views [:M] of buffers whose rows past M hold
    -128 codes and NaN scales and sums, as the runner's row views of its activation buffers do; the output rows past M must stay untouched;
  * prompt-sized M (1000, 4096, 8192 = 8 prompts of 1024 tokens) on the automatic, unsplit multi-wave plan, against the torch restatement of
    the oracle on the device (exact float64 accumulators, the fp32 epilogue op by op), which is checked against oracle/w4a8.py at a small
    slice of the same problem;
  * a captured chain quantiser -> GEMM -> the runner's next kernel (silu_and_mul_quant after gate_up, add_rms_norm_general after o), with
    programmatic dependent launch on and fresh activations copied in before every replay: the GEMM must read what the quantiser wrote in
    this replay, and one variant writes the GEMM's output over the quantiser's input, as the runner's o output aliases its qkv buffer."""
import numpy as np
import pytest
import torch

from oracle import ops
from tests import gemm_edge_cases as edges
from tests.util import np_of, to_dev

pytestmark = pytest.mark.gpu

PLANS = ((32, 1), (64, 2), (128, 1), (128, 4))  # forced (tokens per tile, cluster split)
PROMPT_ROWS = 1000
PAD = 64  # poisoned / sentinel rows behind row M


def gemm(mode, aq, args, sa, asum, out, acc=None):
    """The drop-in op of `mode` on device tensors; args as Weights.args.  acc=None launches the instantiation the runner uses."""
    if mode == "chn":
        import qserve_backend.qgemm_w4a8_per_chn as op
        qw, s1, s1z = args
        op.gemm_forward_cuda(aq, qw, s1, sa, s1z, asum, out, _acc_out=acc)
    elif mode == "grp":
        import qserve_backend.qgemm_w4a8_per_group as op
        qw, s2z, s2s, s1 = args
        op.gemm_forward_cuda(aq, qw, s2z, s2s, s1, sa, out, _acc_out=acc)
    else:
        import qserve_backend.qgemm_w8a8 as op
        w, sw = args
        op.w8a8_gemm_forward_cuda(aq, w, sw, sa, out, _acc_out=acc)


def _poisoned(aq, sa, asum, dev):
    """Device views [:M] of buffers whose rows past M hold -128 codes and NaN scales / sums."""
    M, K = aq.shape
    a = torch.full((M + PAD, K), -128, dtype=torch.int8, device=dev)
    s = torch.full((M + PAD,), float("nan"), dtype=torch.half, device=dev)
    u = torch.full((M + PAD,), float("nan"), dtype=torch.half, device=dev)
    a[:M], s[:M], u[:M] = to_dev(aq, dev), to_dev(sa, dev), to_dev(asum, dev)
    return a[:M], s[:M], u[:M]


def _force(nt, split):
    from qserve_b200._lib import lib
    lib.qs_gemm_force_tile_tokens(nt)
    lib.qs_gemm_force_split(split)


@pytest.mark.parametrize("name", edges.CASE_NAMES)
def test_edge_case_bits(dev, name):
    c = edges.build(name)
    M, N = c.out.shape
    args = [to_dev(a, dev) for a in c.wt.args]
    reps = -(-PROMPT_ROWS // M)
    runs = [(M, plan) for plan in PLANS] + [(PROMPT_ROWS, (128, 1))]
    try:
        for rows, plan in runs:
            aq, sa, asum = (np.tile(x, (reps,) + (1,) * (x.ndim - 1))[:rows] for x in (c.aq, c.sa, c.asum))
            out_o, acc_o = np.tile(c.out, (reps, 1))[:rows], np.tile(c.acc, (reps, 1))[:rows]
            d_aq, d_sa, d_asum = _poisoned(aq, sa, asum, dev)
            _force(*plan)
            for dump in (True, False):
                out = torch.full((rows + PAD, N), float("nan"), dtype=torch.half, device=dev)
                acc = torch.full((rows + PAD, N), -1, dtype=torch.int32, device=dev) if dump else None
                gemm(c.wt.mode, d_aq, args, d_sa, d_asum, out[:rows], acc[:rows] if dump else None)
                torch.cuda.synchronize()
                what = (name, rows, plan, dump)
                assert edges.same_bits(np_of(out[:rows]), out_o), what
                assert bool(torch.isnan(out[rows:]).all()), what
                if dump:
                    assert np.array_equal(np_of(acc[:rows]), acc_o), what
                    assert bool((acc[rows:] == -1).all()), what
    finally:
        _force(0, 0)


def _synth(mode, rng, N, K):
    """Random weights of `mode` as keyword arguments of edges.weights (slice every value [:n] for the first n channels)."""
    p = {"q": rng.integers(0, 16, (N, K), dtype=np.uint8), "ws": rng.uniform(0.005, 0.02, N)}
    if mode == "chn":
        p["wsz"] = rng.integers(0, 16, N) * p["ws"]
    elif mode == "grp":
        p["s2"], p["z"] = rng.integers(1, 17, (N, K // 128)), rng.integers(0, 16, (N, K // 128))
    else:
        p["w"] = rng.integers(-128, 128, (N, K), dtype=np.int8)
    return p


def _device_weights(wt, dev):
    t = lambda a: None if a is None else to_dev(a, dev)  # noqa: E731
    return [t(a) for a in wt.args], t(wt.w8), t(wt.ws), t(wt.wsz)


PROMPT_SHAPES = {"chn": (4096, 14336), "grp": (6144, 4096), "w8": (4096, 4096)}  # Llama-3-8B down, qkv; Mistral-7B o


@pytest.mark.parametrize("mode", edges.MODES)
def test_prompt_sized_m(dev, mode):
    N, K = PROMPT_SHAPES[mode]
    rng = np.random.default_rng(N + K)
    p = _synth(mode, rng, N, K)
    wt = edges.weights(mode, **p)
    args, w8, ws, wsz = _device_weights(wt, dev)
    Mmax = 8192
    g = torch.Generator(device=dev).manual_seed(N + K)
    aq = torch.randint(-128, 128, (Mmax, K), dtype=torch.int8, device=dev, generator=g)
    sa = (torch.rand(Mmax, device=dev, generator=g) * 0.015 + 0.005).half()
    asum = (torch.randn(Mmax, device=dev, generator=g) * 64).half()
    ref, ref_acc = edges.restated(mode, aq, w8, ws, wsz, sa, asum)
    ref_acc = ref_acc.to(torch.int32)
    # the restatement against the oracle on the first 16 rows x 256 channels
    small = edges.weights(mode, **{k: v[:256] for k, v in p.items()})
    out_o, acc_o = edges.oracle(small, np_of(aq[:16]), np_of(sa[:16]), np_of(asum[:16]))
    assert np.array_equal(np_of(ref_acc[:16, :256]), acc_o)
    assert edges.same_bits(np_of(ref[:16, :256]), out_o)
    for M in (1000, 4096, 8192):
        for dump in (True, False):
            out = torch.full((M + PAD, N), float("nan"), dtype=torch.half, device=dev)
            acc = torch.zeros((M, N), dtype=torch.int32, device=dev) if dump else None
            gemm(mode, aq[:M], args, sa[:M], asum[:M], out[:M], acc)
            torch.cuda.synchronize()
            assert torch.equal(out[:M].view(torch.int16), ref[:M].view(torch.int16)), (M, dump)
            assert bool(torch.isnan(out[M:]).all()), (M, dump)
            if dump:
                assert torch.equal(acc, ref_acc[:M]), M


CHAIN_SHAPES = {"gate_up": (7168, 4096), "o": (4096, 4096)}  # Llama-3-8B: gate_up at TP = 4, o
CHAIN = [(mode, layer, alias) for mode in edges.MODES for layer, alias in (("gate_up", False), ("o", False), ("o", True))]
CHAIN_PLANS = ((32, 1), (32, 2), (64, 1), (64, 4), (128, 1), (128, 8), (0, 0))  # (0, 0): the automatic plan
REPLAYS = 10


@pytest.mark.parametrize("mode,layer,alias", CHAIN, ids=[f"{m}-{l}" + ("-out_over_x" if a else "") for m, l, a in CHAIN])
def test_pdl_producer_chain(dev, mode, layer, alias):
    """invoke_quant[_fuse_sum] of a static x -> GEMM (no accumulator dump) -> the runner's next kernel, captured once per forced plan with
    programmatic dependent launch on.  After every replay (fresh x each time) the GEMM output equals the oracle of quant_per_token(x), and
    the consumer's outputs equal the same consumer run eagerly, PDL off, on that GEMM output."""
    from qserve_b200 import backend
    N, K = CHAIN_SHAPES[layer]
    M = 64
    rng = np.random.default_rng(N * 3 + K + alias)
    wt = edges.weights(mode, **_synth(mode, rng, N, K))
    args, w8, ws, wsz = _device_weights(wt, dev)
    fuse = mode == "chn"
    half = lambda *s: torch.empty(s, dtype=torch.half, device=dev)  # noqa: E731
    x = half(M, K)
    q, scale, qsum = torch.empty((M, K), dtype=torch.int8, device=dev), half(M), half(M) if fuse else None
    out = x if alias else half(M, N)  # alias: the GEMM writes over the buffer the quantiser read
    if layer == "gate_up":
        def bufs():
            return [torch.empty((M, N // 2), dtype=torch.int8, device=dev), half(M), half(M) if fuse else None]

        def consume(o, b):
            backend.silu_and_mul_quant(b[0], o, b[2], b[1])
    else:
        resid = to_dev(rng.standard_normal((M, N)).astype(np.float16), dev)
        gamma = to_dev(rng.uniform(0.5, 1.5, N).astype(np.float16), dev)

        def bufs():
            return [torch.empty((M, N), dtype=torch.int8, device=dev), half(M, N), half(M), half(M) if fuse else None]

        def consume(o, b):
            backend.add_rms_norm_general(b[0], b[1], resid, o, gamma, b[3], b[2], 1e-5)
    cb = bufs()

    def step():
        if fuse:
            backend.invoke_quant_fuse_sum(q, x, qsum, scale)
        else:
            backend.invoke_quant(q, x, scale)
        gemm(mode, q, args, scale, qsum, out)
        consume(out, cb)

    bits = lambda t: t.view(torch.int16) if t.dtype == torch.half else t  # noqa: E731
    was = backend.set_pdl(True)
    try:
        for plan in CHAIN_PLANS:
            _force(*plan)
            x.copy_(to_dev(rng.standard_normal((M, K)).astype(np.float16), dev))
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                step()  # first launches (function attributes, workspaces) outside the capture
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
            for rep in range(REPLAYS):
                xs = rng.standard_normal((M, K)).astype(np.float16)
                x.copy_(to_dev(xs, dev))
                graph.replay()
                torch.cuda.synchronize()
                aq_o, sa_o, asum_o = ops.quant_per_token(xs)
                ref = edges.restated(mode, to_dev(aq_o, dev), w8, ws, wsz, to_dev(sa_o, dev), to_dev(asum_o, dev))[0]
                assert torch.equal(bits(out), bits(ref)), (plan, rep)
                backend.set_pdl(False)
                eager = bufs()
                consume(out.clone(), eager)
                torch.cuda.synchronize()
                backend.set_pdl(True)
                for i, (a, b) in enumerate(zip(cb, eager)):
                    assert a is None or torch.equal(bits(a), bits(b)), (plan, rep, i)
            del graph
    finally:
        backend.set_pdl(was)
        _force(0, 0)
