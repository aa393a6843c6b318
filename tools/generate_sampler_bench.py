"""The generation loop's sampler: time apply_penalties_tree against the composition it replaces, logprobs_accepted, and the captured
generation step with and without penalties and log-probabilities.

    python tools/generate_sampler_bench.py --out DIR [--iters 50] [--tokens 32] [--rounds 2] [--no-e2e]

Kernels (timed inside CUDA graphs, tools/tree_verify_bench._graph_time; the arms of one shape alternate):
  * apply_penalties_tree on [B, n, V = 128256] verify logits against (a) the composition: the expanded per-node histories built with torch
    ops, then apply_penalties over B n rows, and (b) apply_penalties over the B root rows alone (the sequential step's cost), at B in
    (1, 8, 64), n in (4, 8, 16), H in (1024, 2048, 4096, 8192) full histories (ids from a 64-token alphabet), trees from ngram_propose;
  * logprobs_accepted with n_top = 5 at acc = 1 and acc = n (B = 64, n in (4, 8)), and logprobs_rows over the B rows for scale.
End to end: Llama-3-8B W4A8KV4, batch 64, ctx 1024, all layers, --tokens generated tokens per row; arms: plain (n = 1) and speculative
n = 4 (branches 1) / n = 8 (branches 2), each without and with penalties (presence 0.5, frequency 0.5; the repetition penalty would count
the planted prompt ids) and logprobs = 5, every arm a captured step replayed until every row is finished.  "planted": each arm's own plain
output planted in the prompt behind the last four ids; "random": a random prompt.  Arms alternate over --rounds rounds.  The device name,
power limit and maximum SM clock are read in the same run.  Writes DIR/generate_sampler_bench.json.
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
from tools.speculative_bench import _run_until_done  # noqa: E402
from tools.tree_verify_bench import _alternate, _device_info, _graph_time  # noqa: E402

VOCAB = 128256


def _capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(20):
            fn()
    return g


def _composition(logits, tok, mask, hist, pl, L, rep, pres, freq, buf):
    """The expanded per-node histories with torch ops (graph-capturable), then apply_penalties over the B n rows."""
    B, n = tok.shape
    H = hist.size(1)
    i = torch.arange(n, device=tok.device)
    below = torch.where(i > 0, (1 << i) - 1, 0) & ~1
    word = (mask & below) | torch.where(i > 0, 1 << i, 0)                        # [B, n] path words
    bits = (word.unsqueeze(-1) >> torch.arange(16, device=tok.device)) & 1        # [B, n, 16]
    pos = L.view(B, 1, 1).long() + bits.cumsum(-1) - 1
    col = torch.where(bits.bool(), pos, H + 15)                                   # non-path nodes go to a dump column
    buf[:, :, :H].copy_(hist.unsqueeze(1).expand(B, n, H))
    buf.scatter_(2, col, torch.nn.functional.pad(tok, (0, 16 - n), value=-1).unsqueeze(1).expand(B, n, 16).contiguous())
    sl = (L.view(B, 1) + bits.sum(-1)).to(torch.int32).view(-1)
    r = lambda a: a.repeat_interleave(n)
    backend.apply_penalties(logits.view(B * n, -1), buf.view(B * n, H + 16), r(pl), sl, r(rep), r(pres), r(freq))


def kernel_cases(iters, dev):
    out = []
    shapes = [(B, n, H) for B in (1, 8, 64) for n in (4, 8, 16) for H in (1024, 4096, 8192)] + [(64, 8, 2048)]
    for B, n, H in shapes:
        g = torch.Generator(device=dev).manual_seed(B * 131 + n * 7 + H)
        hist = torch.randint(0, 64, (B, H), device=dev, generator=g)
        L = torch.full((B,), H - n, dtype=torch.int32, device=dev)  # the expanded histories fit H + 16 columns
        pl = torch.full((B,), H // 2, dtype=torch.int32, device=dev)
        rep, pres, freq = (torch.full((B,), v, dtype=torch.float32, device=dev) for v in (1.2, 0.5, 0.5))
        tok, mask = backend.ngram_propose(hist, L, n, 1, 4, 4)
        logits = torch.randn((B, n, VOCAB), device=dev, generator=g).half()
        root = logits[:, 0].contiguous()
        buf = torch.full((B, n, H + 16), -1, dtype=torch.int64, device=dev)
        graphs = [_capture(lambda: backend.apply_penalties_tree(logits, tok, mask, hist, pl, L, rep, pres, freq)),
                  _capture(lambda: _composition(logits, tok, mask, hist, pl, L, rep, pres, freq, buf)),
                  _capture(lambda: backend.apply_penalties(root, hist, pl, L, rep, pres, freq))]
        t = [x / 20 for x in _alternate([gr.replay for gr in graphs], iters, 5)]
        row = {"op": "apply_penalties_tree", "batch": B, "n": n, "history": H, "kernel_us": round(t[0], 2), "composition_us": round(t[1], 2),
               "roots_only_us": round(t[2], 2), "composition_over_kernel": round(t[1] / t[0], 2)}
        out.append(row)
        print(json.dumps(row), flush=True)
        del graphs
    B, K, W = 64, 5, 1300
    for n in (4, 8):
        g = torch.Generator(device=dev).manual_seed(n)
        logits = torch.randn((B, n, VOCAB), device=dev, generator=g).half()
        tok = torch.randint(0, VOCAB, (B, n), device=dev, generator=g)
        path = torch.arange(n, dtype=torch.int32, device=dev).repeat(B, 1).contiguous()
        bonus = torch.zeros(B, dtype=torch.int64, device=dev)
        L = torch.full((B,), 1025, dtype=torch.int32, device=dev)
        fin = torch.zeros(B, dtype=torch.int32, device=dev)
        lp = torch.zeros((B, W), dtype=torch.float32, device=dev)
        ids = torch.zeros((B, W, K), dtype=torch.int64, device=dev)
        tlp = torch.zeros((B, W, K), dtype=torch.float32, device=dev)
        for acc_v in (1, n):
            acc = torch.full((B,), acc_v, dtype=torch.int32, device=dev)
            t = _graph_time(lambda: backend.logprobs_accepted(logits, tok, path, acc, bonus, L, fin, K, lp, ids, tlp), iters)
            row = {"op": "logprobs_accepted", "batch": B, "n": n, "acc": acc_v, "us": round(t, 2)}
            out.append(row)
            print(json.dumps(row), flush=True)
        rows = logits[:, 0].contiguous()
        t = _graph_time(lambda: backend.logprobs_rows(rows, bonus, K, lp[:, 0].contiguous(), ids[:, 0].contiguous(), tlp[:, 0].contiguous()), iters)
        row = {"op": "logprobs_rows", "rows": B, "us": round(t, 2)}
        out.append(row)
        print(json.dumps(row), flush=True)
    return out


ARMS = [(1, 1), (4, 1), (8, 2)]


def e2e(B, T, rounds, dev):
    from qserve_b200.decode import DecodeRunner

    ctx = 1024
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=ctx, device=dev, seed=0, verify_len=8, max_new_tokens=T, generate=True)
    run.s_presence.fill_(0.5)
    run.s_frequency.fill_(0.5)
    g = torch.Generator(device=dev).manual_seed(B)
    random_prompt = torch.randint(0, run.cfg.vocab, (B, ctx + 1), device=dev, generator=g)
    keys = [(n, br, (1, 4), False, 2, pen, 5 if pen else 0) for pen in (False, True) for n, br in ARMS]
    step_key = lambda k: k[:4] + k[5:]
    for k in keys:
        run.reset_generation(random_prompt)
        run.capture_generate(*k)
    planted = {}
    for pen in (False, True):  # each mode's own plain output, planted behind a copy of the key
        plain_key = next(k for k in keys if k[0] == 1 and k[5] == pen)
        _run_until_done(run, step_key(plain_key), random_prompt, T)
        p = random_prompt.clone()
        p[:, 10:14] = random_prompt[:, ctx - 3:ctx + 1]
        p[:, 14:14 + T] = run.s_history[:, ctx + 1:ctx + 1 + T]
        planted[pen] = p
    res = []
    for name in ("planted", "random"):
        acc = {k: [] for k in keys}
        for _ in range(rounds):
            for k in keys:
                prompt = planted[k[5]] if name == "planted" else random_prompt
                acc[k].append(_run_until_done(run, step_key(k), prompt, T))
        base = {}
        for k in keys:
            ms = min(a[0] for a in acc[k])
            steps, toks = acc[k][0][1], acc[k][0][2]
            row = {"workload": name, "batch": B, "n": k[0], "branches": k[1], "penalties_logprobs": k[5], "steps": steps,
                   "ms_per_step": round(ms / steps, 3), "tokens_per_row_step": round(toks / (B * steps), 3), "tokens_per_s": round(toks / (ms / 1e3), 1),
                   "ms_rounds": [round(a[0], 2) for a in acc[k]]}
            if not k[5]:
                base[k[:2]] = row
            else:
                row["ms_per_step_over_unpenalised"] = round(row["ms_per_step"] / base[k[:2]]["ms_per_step"], 3)
            res.append(row)
            print(json.dumps(row), flush=True)
    del run
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generate_sampler_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"device_info": _device_info()}
    print(json.dumps(res["device_info"]), flush=True)
    if not a.no_kernels:
        res["kernels"] = kernel_cases(a.iters, dev)
    if not a.no_e2e:
        res["e2e"] = {"model": "llama-3-8b", "precision": "w4a8kv4", "ctx": 1024, "tokens": a.tokens, "rows": e2e(64, a.tokens, a.rounds, dev)}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "generate_sampler_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
