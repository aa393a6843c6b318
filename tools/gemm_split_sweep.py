#!/usr/bin/env python
"""Time the decode GEMM shapes for the automatic plan and every tile size / cluster split factor (qs_gemm_force_tile_tokens,
qs_gemm_force_split) -- tuning aid for plan_gemm() in csrc/gemm.cu, and the per-shape A/B timer of two builds.

Each number is microseconds per launch of a CUDA graph that launches the shape once per layer over --layers weight sets, replayed
back to back (as bench.py's time_kernel): every launch streams its weights from HBM, as in the decode step.  For the automatic plan
the tool also prints the (tokens per tile, split) the planner chose, read back from a profiled launch.

  python tools/gemm_split_sweep.py [--shapes llama-3-8b] [--precision w4a8kv4] [--batch 64] [--reps 20] [--auto-only]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qserve_b200._lib import lib  # noqa: E402
from qserve_b200.decode import _Linear  # noqa: E402

# (N, K) per launch.  qwen72b-tp4: the per-rank shards of Qwen1.5-72B at tensor parallelism 4
SHAPES = {
    "llama-3-8b": {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)},
    "w8a8-b128": {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)},
    "qwen72b-tp4": {"qkv": (6144, 8192), "o": (8192, 2048), "gate_up": (12288, 8192), "down": (8192, 6144)},
}

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="llama-3-8b", choices=sorted(SHAPES), help="w8a8-b128: the Llama-3-8B / Mistral-7B shapes as W8A8 at batch 128")
ap.add_argument("--precision", default="w4a8kv4")
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--layers", type=int, default=32, help="weight sets per shape (enough that a replay never finds its weights in L2)")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--auto-only", action="store_true", help="only the automatic plan (A/B of two builds)")
args = ap.parse_args()
if args.shapes == "w8a8-b128":
    args.precision, args.batch = "w8a8", 128
mode = "w8" if args.precision.startswith("w8a8") else ("grp" if args.precision.endswith("g128") else "chn")

dev = torch.device("cuda:0")
gen = torch.Generator(device=dev)
gen.manual_seed(0)
M = args.batch
scale = torch.full((M,), 0.01, dtype=torch.half, device=dev)
asum = torch.full((M,), 0.1, dtype=torch.half, device=dev)
prof = torch.zeros(8192 * 16, dtype=torch.int64, device=dev)


def time_op(lins, xq, buf):
    def fn():
        for lin in lins:
            lin(xq, scale, asum, buf)
    fn()  # warm (attributes, tensor maps, plan)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    del g
    return e0.elapsed_time(e1) * 1e3 / (args.reps * len(lins))


def plan_of(lin, xq, buf):
    """(tokens per tile, split) of one profiled launch: thread 0 of every CTA stamps them into slots 13 and 14."""
    prof.zero_()
    lib.qs_gemm_set_profile_buffer(prof.data_ptr())
    lin(xq, scale, asum, buf)
    torch.cuda.synchronize()
    lib.qs_gemm_set_profile_buffer(None)
    nt, split = prof[13].item(), prof[14].item()
    return f"NT={nt} S={split}" if nt else "plan not stamped by this build"


print(f"-- {args.shapes} {args.precision} batch {M}, {args.layers} weight sets, us per launch")
nts = (0,) if args.auto_only else (0, 32, 64, 128)
for name, (N, K) in SHAPES[args.shapes].items():
    lins = [_Linear(N, K, mode, dev, gen) for _ in range(args.layers)]
    xq = torch.randint(-127, 128, (M, K), dtype=torch.int8, device=dev, generator=gen)
    buf = torch.empty((M, N), dtype=torch.half, device=dev)
    for nt in nts:
        lib.qs_gemm_force_tile_tokens(nt)
        line = f"{name:8s} N={N:5d} K={K:5d} tokens per tile = {nt if nt else 'auto':>4}"
        for S in ((0,) if nt == 0 else (1, 2, 4, 8)):
            lib.qs_gemm_force_split(S)
            try:
                line += f"  S={S if S else 'auto'}: {time_op(lins, xq, buf):6.2f}"
            except Exception as ex:  # noqa: BLE001
                line += f"  S={S}: failed ({str(ex)[:40]})"
        if nt == 0:
            line += f"  ({plan_of(lins[0], xq, buf)})"
        print(line, flush=True)
    del lins
lib.qs_gemm_force_split(0)
lib.qs_gemm_force_tile_tokens(0)
