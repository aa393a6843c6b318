#!/usr/bin/env python
"""Launch one hot-path op a few times at a BASELINE shape (for ncu captures and quick timing).
usage: python tools/run_op.py {gemm_qkv|gemm_o|gemm_gate_up|gemm_down|attention|norm|quant|silu} [--reps N] [--precision P] [--batch B] [--ctx C]"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qserve_b200 import backend  # noqa: E402
from qserve_b200.decode import DecodeRunner  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("op")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--precision", default="w4a8kv4")
ap.add_argument("--model", default="llama-3-8b")
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--ctx", type=int, default=1024)
ap.add_argument("--layers", type=int, default=4)
ap.add_argument("--no-pdl", action="store_true")
ap.add_argument("--time", action="store_true")
a = ap.parse_args()
backend.set_pdl(not a.no_pdl)
run = DecodeRunner(a.model, a.precision, a.batch, a.ctx, torch.device("cuda:0"), layers=a.layers)
D = run.cfg.head_dim
q, k, v = run.qkv_buf.split([run.q_size, run.kv_size, run.kv_size], dim=-1)
q, k, v = q.reshape(a.batch, run.Hq, D), k.reshape(a.batch, run.Hkv, D), v.reshape(a.batch, run.Hkv, D)
run.qkv_buf.normal_()
hidden = torch.randn((a.batch, run.cfg.hidden), device="cuda", dtype=torch.half)
import qserve_backend.fused_attention as fa  # noqa: E402


def call(i):
    ly = run.layers[i % run.L]
    if a.op.startswith("gemm_"):
        name = a.op[5:]
        xq, buf = {"qkv": (run.q_hidden, run.qkv_buf), "o": (run.q_attn, run.out_buf), "gate_up": (run.q_hidden, run.gate_up_buf),
                   "down": (run.q_mlp, run.out_buf)}[name]
        ly[name](xq, run.q_scale, run.q_sum, buf)
    elif a.op == "attention":
        fa.single_query_attention(q, k, v, run.block_tables[i % run.L], run.context_lens, None, 8192, 64, run.size_per_token, run.max_seq_len, D,
                                  run.cfg.rope_theta, True, run.kv_bits == 4, True)
    elif a.op == "norm":
        run._norm_quant(run.rows, hidden, ly["ln1"])
    elif a.op == "quant":
        run._quant(run.rows, run.q_mlp, run.mlp_act)
    elif a.op == "silu":
        from qserve_backend import activation_ops
        activation_ops.silu_and_mul(run.mlp_act, run.gate_up_buf)
    else:
        raise SystemExit("unknown op")


run.q_scale.fill_(0.01); run.q_sum.fill_(0.1)
for i in range(2):
    call(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(a.reps):
    call(i)
e1.record()
torch.cuda.synchronize()
if a.time:
    print(f"{a.op}: {e0.elapsed_time(e1) * 1e3 / a.reps:.2f} us/launch over {a.reps} launches (pdl={not a.no_pdl})")
