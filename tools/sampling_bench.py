"""GPU sampling: time sample_rows against argmax_rows and against a torch restatement of the reference's Sampler.forward, tree_accept_sampling
against tree_accept_greedy, and the sampled decode / tree steps end to end.

    python tools/sampling_bench.py --out DIR [--iters 200] [--rounds 3] [--e2e-iters 50] [--no-e2e]

sample_rows: fp16 logits [B, 128256], B in (1, 8, 64), settings (T, top_k, top_p) in (1.0, 1, 1.0) (the reference ModelRunner's default),
(0.7, 50, 0.9), (0.8, -1, 0.95) and (1.0, -1, 1.0).  The torch arm restates Sampler.forward (qserve/modeling/layers/sampler.py): the
TemperatureLogitsWarper division (skipped at T = 1), TopPLogitsWarper (sort, softmax, cumsum, scatter of the mask; skipped at top_p = 1),
TopKLogitsWarper (topk, masked_fill; skipped at top_k = -1), softmax and torch.multinomial, all in fp16 as the reference runs them.  Each arm
is the median of --iters launches timed one by one with CUDA events, the arms alternating launch by launch; --rounds rounds show the spread.
tree_accept_sampling: batch 64, V = 128256, a random tree of n in (4, 8, 16) nodes, with and without draft_probs, against
tree_accept_greedy (which reads target tokens the verify step's argmax_rows produced: its time plus argmax_rows over the B n rows is the
greedy arm's full cost).  Bytes read are computed from the shapes.
End to end (unless --no-e2e): the decode runner (Llama-3-8B W4A8KV4, batch 64, ctx 1024, all layers, CUDA graphs): the sampled decode step
(0.8, -1, 0.95) against the greedy step, and the sampled tree step of n = 8 nodes against the greedy tree step, alternating.
The device name, power limit and maximum SM clock are read in the same run.  Writes DIR/sampling_bench.json.
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
from tools.tree_verify_bench import _alternate, _device_info, random_tree  # noqa: E402

V = 128256
SETTINGS = [(1.0, 1, 1.0), (0.7, 50, 0.9), (0.8, -1, 0.95), (1.0, -1, 1.0)]


def torch_sampler(logits, T, top_k, top_p):
    """Sampler.forward with one SamplingParams for the batch, in the reference's order and dtype."""
    x = logits
    if T >= 1e-5 and T != 1.0:
        x = x / T
    if 1e-8 <= top_p < 1.0:
        sx, idx = torch.sort(x, descending=False)
        cum = sx.softmax(dim=-1).cumsum(dim=-1)
        drop = cum <= (1 - top_p)
        drop[..., -1:] = 0
        x = x.masked_fill(drop.scatter(1, idx, drop), -float("inf"))
    if top_k > 0:
        kth = torch.topk(x, min(top_k, x.size(-1)))[0][..., -1, None]
        x = x.masked_fill(x < kth, -float("inf"))
    if T < 1e-5 or top_p < 1e-8:
        return torch.argmax(x, dim=-1)
    return torch.multinomial(torch.softmax(x, dim=-1), num_samples=1).view(-1)


def rows_case(Bn, setting, iters, rounds, dev):
    g = torch.Generator(device=dev).manual_seed(Bn)
    logits = (torch.randn((Bn, V), device=dev, generator=g) * 3).half()
    off = torch.zeros(Bn, dtype=torch.int64, device=dev)
    T = torch.full((Bn,), setting[0], device=dev)
    K = torch.full((Bn,), setting[1], dtype=torch.int32, device=dev)
    P = torch.full((Bn,), setting[2], device=dev)
    out = torch.empty(Bn, dtype=torch.int64, device=dev)
    fns = [lambda: backend.sample_rows(logits, T, K, P, 1, off, out=out), lambda: backend.argmax_rows(logits, out=out),
           lambda: torch_sampler(logits, *setting)]
    runs = [_alternate(fns, iters) for _ in range(rounds)]
    return {"batch": Bn, "vocab": V, "setting": list(setting), "sample_rows_us": [round(r[0], 2) for r in runs],
            "argmax_rows_us": [round(r[1], 2) for r in runs], "torch_sampler_us": [round(r[2], 2) for r in runs]}


def tree_case(n, probs, iters, rounds, dev, B=64):
    g = torch.Generator(device=dev).manual_seed(n)
    gc = torch.Generator().manual_seed(n)
    logits = (torch.randn((B, n, V), device=dev, generator=g) * 3).half()
    mask = torch.tensor([random_tree(n, gc) for _ in range(B)], dtype=torch.int32, device=dev)
    target = backend.argmax_rows(logits.view(B * n, V)).view(B, n)
    draft = torch.where(torch.rand((B, n), device=dev, generator=g) < 0.5, target, torch.randint(0, V, (B, n), device=dev, generator=g))
    q = torch.softmax(torch.randn((B, n, V), device=dev, generator=g), -1) if probs else None
    off = torch.zeros(B, dtype=torch.int64, device=dev)
    outs = (torch.empty(B, dtype=torch.int32, device=dev), torch.empty((B, n), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int64, device=dev))
    fns = [lambda: backend.tree_accept_sampling(draft, mask, logits, 0.8, -1, 0.95, 1, off, q, *outs),
           lambda: backend.tree_accept_greedy(draft, mask, target, *outs),
           lambda: backend.argmax_rows(logits.view(B * n, V), out=target.view(-1))]
    runs = [_alternate(fns, iters) for _ in range(rounds)]
    acc = backend.tree_accept_sampling(draft, mask, logits, 0.8, -1, 0.95, 1, off, q)[0].float().mean().item()
    return {"batch": B, "nodes": n, "vocab": V, "draft_probs": probs, "mean_accept_len": round(acc, 2),
            "tree_accept_sampling_us": [round(r[0], 2) for r in runs], "tree_accept_greedy_us": [round(r[1], 2) for r in runs],
            "argmax_rows_all_nodes_us": [round(r[2], 2) for r in runs],
            # logits of every visited node (at least the root) + q rows of every tried child, against the greedy op's int64 / int32 inputs
            "bytes_read_min": B * V * 2 + (B * (n - 1) * V * 4 if probs else 0), "bytes_read_greedy": B * n * (8 + 8 + 4)}


def run_e2e(iters, rounds, dev):
    from qserve_b200.decode import DecodeRunner
    B = 64
    res = {"model": "llama-3-8b", "precision": "w4a8kv4", "batch": B, "ctx": 1024}
    greedy = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=1024, device=dev, verify_len=8)
    greedy.capture()
    sampled = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=1024, device=dev, verify_len=8)
    sampled.s_temperature.fill_(0.8); sampled.s_top_k.fill_(-1); sampled.s_top_p.fill_(0.95)
    sampled.capture(sample=True)
    runs = [_alternate([greedy.step, sampled.step], iters, 3) for _ in range(rounds)]
    res["decode_greedy_ms"] = [round(r[0] / 1e3, 3) for r in runs]
    res["decode_sampled_ms"] = [round(r[1] / 1e3, 3) for r in runs]
    res["decode_sampled_over_greedy"] = [round(r[1] / r[0], 4) for r in runs]
    print(json.dumps(res), flush=True)
    n = 8
    gc = torch.Generator().manual_seed(5)
    m = torch.tensor([random_tree(n, gc) for _ in range(B)], dtype=torch.int32)
    for r in (greedy, sampled):
        r.v_tree_mask[:, :n].copy_(m)
    greedy.capture_verify(n, tree=True)
    sampled.capture_verify(n, tree=True, sampled=True)
    runs = [_alternate([lambda: greedy.verify_step(n, tree=True), lambda: sampled.verify_step(n, tree=True, sampled=True)], iters, 3)
            for _ in range(rounds)]
    res["tree_n8_greedy_ms"] = [round(r[0] / 1e3, 3) for r in runs]
    res["tree_n8_sampled_ms"] = [round(r[1] / 1e3, 3) for r in runs]
    print(json.dumps({k: res[k] for k in ("tree_n8_greedy_ms", "tree_n8_sampled_ms")}), flush=True)
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
    res = {"config": {"iters": args.iters, "rounds": args.rounds}, **_device_info(), "sample_rows": [], "tree_accept": []}
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}), flush=True)
    for Bn in (1, 8, 64):
        for s in SETTINGS:
            r = rows_case(Bn, s, args.iters, args.rounds, dev)
            res["sample_rows"].append(r)
            print(json.dumps(r), flush=True)
    for n in (4, 8, 16):
        for probs in (False, True):
            r = tree_case(n, probs, args.iters, args.rounds, dev)
            res["tree_accept"].append(r)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    if not args.no_e2e:
        res["end_to_end"] = run_e2e(args.e2e_iters, args.rounds, dev)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "sampling_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
