"""Prompt-lookup speculative decoding: time ngram_propose and spec_commit, and generation end to end against plain decoding.

    python tools/speculative_bench.py --out DIR [--iters 100] [--tokens 64] [--batches 1,8,64] [--rounds 2] [--no-e2e]

Kernels: each op timed as the runner runs it, 50 calls inside a CUDA graph (tools/tree_verify_bench._graph_time), at B in (1, 8, 64),
histories of H in (1024, 4096, 32768) full tokens (ids from a 64-token alphabet, so that many positions match the key's last id and the
scan extends past the first compare), n in (4, 8, 16) and, for ngram_propose, branches in (1, 4).
End to end: one runner per batch (Llama-3-8B W4A8KV4, ctx 1024, all layers, verify_len 8, --tokens generated tokens per row), every arm a
captured generation step replayed until every row is finished: plain decoding (n = 1) and speculative steps at n in (4, 8), branches in
(1, 2), ngram (1, 4).  Two workloads: "planted" (each row's greedy continuation, found by the plain arm, is planted in its prompt behind the
prompt's last four ids: the best case) and "random" (a random prompt: few drafts are accepted, the pure overhead).  The arms alternate over
--rounds rounds.  Reported per arm: ms per step, mean tokens emitted per row and step, tokens/s, the speedup over plain and the break-even
tokens per step (ms per step over the plain arm's).  The device name, power limit and maximum SM clock are read in the same run.  Writes
DIR/speculative_bench.json.
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
from tools.tree_verify_bench import _device_info, _graph_time  # noqa: E402


def kernel_cases(iters, dev):
    out = []
    for B in (1, 8, 64):
        for H in (1024, 4096, 32768):
            g = torch.Generator(device=dev).manual_seed(B * H)
            hist = torch.randint(0, 64, (B, H), device=dev, generator=g)
            lens = torch.full((B,), H, dtype=torch.int32, device=dev)
            for n in (4, 8, 16):
                tok = torch.empty((B, n), dtype=torch.int64, device=dev)
                mask = torch.empty((B, n), dtype=torch.int32, device=dev)
                for br in (1, 4):
                    t = _graph_time(lambda: backend.ngram_propose(hist, lens, n, 1, 4, br, tokens=tok, tree_mask=mask), iters)
                    out.append({"op": "ngram_propose", "batch": B, "history": H, "n": n, "branches": br, "us": round(t, 2),
                                "bytes_read_bound": B * H * 8})
                # the commit: every row accepts all n nodes (path 0 .. n - 1); the history is large enough that nothing is dropped early
                h2 = torch.full((B, H), -1, dtype=torch.int64, device=dev)
                path = torch.arange(n, dtype=torch.int32, device=dev).repeat(B, 1).contiguous()
                acc = torch.full((B,), n, dtype=torch.int32, device=dev)
                bonus = torch.zeros(B, dtype=torch.int64, device=dev)
                L = torch.full((B,), H // 2, dtype=torch.int32, device=dev)
                prompt = L.clone()
                budget = torch.full((B,), 1 << 30, dtype=torch.int32, device=dev)
                eos = torch.full((B,), -1, dtype=torch.int64, device=dev)
                fin = torch.zeros(B, dtype=torch.int32, device=dev)
                start, ctxl, roots = L.clone(), L.clone(), bonus.clone()
                t = _graph_time(lambda: backend.spec_commit(tok, path, acc, bonus, h2, L, prompt, budget, eos, fin, start, ctxl, roots), iters)
                out.append({"op": "spec_commit", "batch": B, "history": H, "n": n, "us": round(t, 2)})
                print(json.dumps(out[-1]), flush=True)
    return out


ARMS = [(1, 1), (4, 1), (4, 2), (8, 1), (8, 2)]


def _run_until_done(run, key, prompt, T):
    """Replay the captured step `key` from reset_generation(prompt) until every row is finished: (device ms summed over the steps, steps,
    tokens generated).  Each replay is timed by its own events; the host checks g_finished between replays, outside the timed spans."""
    run.reset_generation(prompt)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms, steps = 0.0, 0
    while not bool(run.g_finished.all()):
        e0.record()
        run.generate_step(*key)
        e1.record()
        torch.cuda.synchronize()
        ms += e0.elapsed_time(e1)
        steps += 1
        assert steps <= T
    return ms, steps, int((run.s_seq_lens - run.s_prompt_lens).sum())


def e2e(B, T, rounds, dev):
    from qserve_b200.decode import DecodeRunner

    ctx = 1024
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=0, verify_len=8, max_new_tokens=T, generate=True)
    g = torch.Generator(device=dev).manual_seed(B)
    random_prompt = torch.randint(0, run.cfg.vocab, (B, ctx + 1), device=dev, generator=g)
    keys = [(n, br, (1, 4), False) for n, br in ARMS]
    run.reset_generation(random_prompt)
    for k in keys:
        run.capture_generate(*k)
        run.reset_generation(random_prompt)
    # the plain loop's output, planted behind a copy of the key
    _run_until_done(run, keys[0], random_prompt, T)
    plain_out = run.s_history[:, ctx + 1:].clone()
    planted = random_prompt.clone()
    planted[:, 10:14] = random_prompt[:, ctx - 3:ctx + 1]
    planted[:, 14:14 + T] = plain_out
    res = []
    for name, prompt in (("planted", planted), ("random", random_prompt)):
        acc = {k: [] for k in keys}
        for _ in range(rounds):
            for k in keys:
                acc[k].append(_run_until_done(run, k, prompt, T))
        base = None
        for k in keys:
            ms = min(a[0] for a in acc[k])  # every round replays the same steps (the loop is deterministic)
            steps, toks = acc[k][0][1], acc[k][0][2]
            ms_step = ms / steps
            row = {"workload": name, "batch": B, "n": k[0], "branches": k[1], "steps": steps, "ms_per_step": round(ms_step, 3),
                   "tokens_per_row_step": round(toks / (B * steps), 3), "tokens_per_s": round(toks / (ms / 1e3), 1),
                   "ms_rounds": [round(a[0], 2) for a in acc[k]]}
            if k[0] == 1:
                base = row
            row["speedup"] = round(row["tokens_per_s"] / base["tokens_per_s"], 3)
            row["break_even_tokens_per_step"] = round(row["ms_per_step"] / base["ms_per_step"], 3)
            res.append(row)
            print(json.dumps(row), flush=True)
    del run
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--tokens", type=int, default=64)
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("speculative_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"device_info": _device_info()}
    print(json.dumps(res["device_info"]), flush=True)
    if not a.no_kernels:
        res["kernels"] = kernel_cases(a.iters, dev)
    if not a.no_e2e:
        res["e2e"] = {"model": "llama-3-8b", "precision": "w4a8kv4", "ctx": 1024, "tokens": a.tokens, "rows": []}
        for B in (int(x) for x in a.batches.split(",")):
            res["e2e"]["rows"] += e2e(B, a.tokens, a.rounds, dev)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "speculative_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
