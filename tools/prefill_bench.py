"""Prompt step (time to first token) of the decode runner: DecodeRunner.prefill on Llama-3-8B W4A8KV4, all layers.

    python tools/prefill_bench.py [--iters 3] [--warmup 1] [--layers N]

Cases: 8 prompts of 1024 tokens and 1 prompt of 8192 tokens, each whole (chunk=None: flash_attn_varlen_func over the prompt) and in pieces
of 512 and 2048 tokens (prefix_prefill_attention over the dequantised prefix).  A prefill is eager and ends in the first token; it is timed
with CUDA events from the call to the token, the median of --iters calls after --warmup.  Reported per case: prompt-step ms, prompt
tokens/s and the INT8 TOP/s that the GEMMs alone would need to fill that time (2 * tokens * sum of N * K over the four GEMMs of every layer;
attention, norms and the lm_head are not counted).  The device name, power limit and maximum SM clock are read in the same run.  Prints one
JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.tree_verify_bench import _device_info  # noqa: E402


def run_case(batch, length, chunks, iters, warmup, layers, dev):
    from qserve_b200.decode import DecodeRunner

    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=batch, ctx=length, device=dev, layers=layers, prompt_tokens=batch * length)
    g = torch.Generator(device=dev).manual_seed(batch * length)
    prompts = torch.randint(0, run.cfg.vocab, (batch, length), device=dev, generator=g)
    lens = torch.full((batch,), length, dtype=torch.int32, device=dev)
    gemm_ops = 2 * batch * length * sum(ly[n].N * ly[n].K for ly in run.layers for n in ("qkv", "o", "gate_up", "down"))
    out = []
    with torch.no_grad():
        for chunk in chunks:
            for _ in range(warmup):
                run.prefill(prompts, lens, chunk=chunk)
            times = []
            for _ in range(iters):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                run.prefill(prompts, lens, chunk=chunk)
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b))
            ms = sorted(times)[len(times) // 2]
            out.append({"batch": batch, "prompt_len": length, "chunk": chunk, "ms": round(ms, 3), "runs_ms": [round(t, 3) for t in times],
                        "tokens_per_s": round(batch * length / ms * 1e3, 1), "gemm_int8_tops": round(gemm_ops / ms * 1e-9, 1)})
    del run
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--layers", type=int, default=None, help="decoder layers (default: all 32)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"model": "llama-3-8b", "precision": "w4a8kv4", "layers": args.layers or 32, **_device_info()}
    res["cases"] = run_case(8, 1024, (None, 512, 2048), args.iters, args.warmup, args.layers, dev) + \
        run_case(1, 8192, (None, 512, 2048), args.iters, args.warmup, args.layers, dev)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
