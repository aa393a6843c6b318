#!/usr/bin/env python
"""Time the four decode GEMM shapes for the automatic plan and every tile size / cluster split factor (qs_gemm_force_tile_tokens,
qs_gemm_force_split) -- tuning aid for dispatch_gemm() / choose_split(), and the per-shape A/B timer of two builds.

Each number is microseconds per launch of a CUDA graph that launches the shape once per layer over ALL the model's layers, replayed
back to back (as bench.py's time_kernel): every launch streams its weights from HBM, as in the decode step.

  python tools/gemm_split_sweep.py [--precision w4a8kv4] [--batch 64] [--reps 20] [--auto-only]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qserve_b200._lib import lib  # noqa: E402
from qserve_b200.decode import DecodeRunner  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--precision", default="w4a8kv4")
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--auto-only", action="store_true", help="only the automatic plan (A/B of two builds)")
args = ap.parse_args()

run = DecodeRunner("llama-3-8b", args.precision, args.batch, 1024, torch.device("cuda:0"))
run.q_scale.fill_(0.01)
run.q_sum.fill_(0.1)
ops = {"qkv": (run.q_hidden, run.qkv_buf), "o": (run.q_attn, run.out_buf), "gate_up": (run.q_hidden, run.gate_up_buf), "down": (run.q_mlp, run.out_buf)}


def time_op(name, xq, buf):
    def fn():
        for ly in run.layers:
            ly[name](xq, run.q_scale, run.q_sum, buf)
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
    return e0.elapsed_time(e1) * 1e3 / (args.reps * len(run.layers))


print(f"-- {args.precision} batch {args.batch}, {len(run.layers)} layers, us per launch")
for nt in ((0,) if args.auto_only else (0, 64, 32)):
    lib.qs_gemm_force_tile_tokens(nt)
    print(f"-- tokens per tile = {nt if nt else 'auto'}")
    for name, (xq, buf) in ops.items():
        line = f"{name:8s}"
        for S in ((0,) if args.auto_only else (0, 1, 2, 4, 8)):
            lib.qs_gemm_force_split(S)
            try:
                line += f"  S={S if S else 'auto'}: {time_op(name, xq, buf):6.2f}"
            except Exception as ex:  # noqa: BLE001
                line += f"  S={S}: failed ({str(ex)[:40]})"
        print(line, flush=True)
lib.qs_gemm_force_split(0)
lib.qs_gemm_force_tile_tokens(0)
