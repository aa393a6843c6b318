"""GPU penalties and log-probabilities: time apply_penalties and logprobs_rows, and their cost inside the captured sampled decode step.

    python tools/logprobs_bench.py --out DIR [--iters 200] [--rounds 3] [--e2e-iters 50] [--no-e2e]

apply_penalties: fp16 logits [B, 128256], B in (1, 8, 64), histories of 1024 / 4096 / 8192 tokens per row (half prompt, half generated, ids
drawn from 4096 tokens so that runs repeat), repetition 1.1, presence 0.5, frequency 0.3.  logprobs_rows: the same logits, n in (0, 5, 20).
Each op is timed as the decode runner runs it, inside a CUDA graph: 50 calls per graph, the median of --iters replays over 50
(tools/tree_verify_bench._graph_time; single eager calls would time the host's argument checks); --rounds rounds show the spread.
End to end (unless --no-e2e): one decode runner (Llama-3-8B W4A8KV4, batch 64, ctx 1024, all layers, CUDA graphs, sampling
(0.8, -1, 0.95)) with two captured steps, the plain sampled step and the sampled step with penalties and logprobs = 5, replayed
alternately.  The device name, power limit and maximum SM clock are read in the same run.  Writes DIR/logprobs_bench.json.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from qserve_b200 import backend  # noqa: E402
from tools.tree_verify_bench import _alternate, _device_info, _graph_time  # noqa: E402

V = 128256


def penalties_case(B, H, iters, rounds, dev):
    g = torch.Generator(device=dev).manual_seed(B * H)
    logits = (torch.randn((B, V), device=dev, generator=g) * 3).half()
    hist = torch.randint(0, 4096, (B, H), device=dev, generator=g)
    prompt = torch.full((B,), H // 2, dtype=torch.int32, device=dev)
    seq = torch.full((B,), H, dtype=torch.int32, device=dev)
    rep, pres, freq = (torch.full((B,), v, device=dev) for v in (1.1, 0.5, 0.3))
    fn = lambda: backend.apply_penalties(logits, hist, prompt, seq, rep, pres, freq)
    runs = [_graph_time(fn, iters) for _ in range(rounds)]
    return {"batch": B, "history": H, "vocab": V, "apply_penalties_us": [round(r, 2) for r in runs]}


def logprobs_case(B, n, iters, rounds, dev):
    g = torch.Generator(device=dev).manual_seed(B + n)
    logits = (torch.randn((B, V), device=dev, generator=g) * 3).half()
    tok = torch.randint(0, V, (B,), device=dev, generator=g)
    outs = (torch.empty(B, device=dev), torch.empty((B, n), dtype=torch.int64, device=dev), torch.empty((B, n), device=dev))
    fn = lambda: backend.logprobs_rows(logits, tok, n, *outs)
    runs = [_graph_time(fn, iters) for _ in range(rounds)]
    return {"batch": B, "n": n, "vocab": V, "logprobs_rows_us": [round(r, 2) for r in runs], "bytes_read": B * V * 2}


def run_e2e(iters, rounds, dev):
    from qserve_b200.decode import DecodeRunner
    B, ctx = 64, 1024
    res = {"model": "llama-3-8b", "precision": "w4a8kv4", "batch": B, "ctx": ctx, "sampling": [0.8, -1, 0.95],
           "penalties": [1.1, 0.5, 0.3], "logprobs": 5}
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=ctx, device=dev, max_new_tokens=1024)
    g = torch.Generator(device=dev).manual_seed(0)
    run.s_history[:, :ctx] = torch.randint(0, 4096, (B, ctx), device=dev, generator=g)
    run.s_prompt_lens.fill_(ctx // 2)
    run.s_temperature.fill_(0.8); run.s_top_k.fill_(-1); run.s_top_p.fill_(0.95)
    run.s_repetition.fill_(1.1); run.s_presence.fill_(0.5); run.s_frequency.fill_(0.3)
    run.capture(sample=True)
    run.capture(sample=True, penalties=True, logprobs=5)
    plain, extra = (True, False, 0), (True, True, 5)
    runs = [_alternate([lambda: run.step(plain), lambda: run.step(extra)], iters, 3) for _ in range(rounds)]
    res["sampled_ms"] = [round(r[0] / 1e3, 4) for r in runs]
    res["sampled_penalties_logprobs_ms"] = [round(r[1] / 1e3, 4) for r in runs]
    res["overhead"] = [round(r[1] / r[0] - 1, 4) for r in runs]
    res["replays_with_history"] = int(run.s_seq_lens[0].item()) - ctx  # the history stays below its last column: no clamped appends
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-iters", type=int, default=50)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    res = {"config": {"iters": args.iters, "rounds": args.rounds}, **_device_info(), "apply_penalties": [], "logprobs_rows": []}
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}), flush=True)
    for B in (1, 8, 64):
        for H in (1024, 4096, 8192):
            r = penalties_case(B, H, args.iters, args.rounds, dev)
            res["apply_penalties"].append(r)
            print(json.dumps(r), flush=True)
        for n in (0, 5, 20):
            r = logprobs_case(B, n, args.iters, args.rounds, dev)
            res["logprobs_rows"].append(r)
            print(json.dumps(r), flush=True)
    if not args.no_e2e:
        res["end_to_end"] = run_e2e(args.e2e_iters, args.rounds, dev)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "logprobs_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
