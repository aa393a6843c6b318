"""Speculative decoding with draft trees: time tree-mask verify attention against the chain verify, the compaction and the acceptance.

    python tools/tree_verify_bench.py --out DIR [--iters 200] [--rounds 3] [--e2e-iters 50] [--no-e2e]

Attention: Llama-3-8B heads (32 query / 8 KV heads, head_dim 128), batch 64, cached prefix P in (1024, 4096), n in (4, 8, 16) nodes per
sequence, KV4 and KV8.  The tree is a random tree of n nodes (every sequence its own); the chain is the same n tokens without a mask.  Both
run on the same pages and q / k / v; per round each is the median of --iters launches timed one by one with CUDA events, the two alternating
launch by launch, and --rounds rounds show the run-to-run spread.
kv_cache_compact: 32 layers, batch 64, 8 KV heads, every sequence accepting 4 nodes of 16 (path 0, 3, 7, 12), KV4 and KV8; the bytes moved
(read + written) are 32 * 64 * 3 moved slots * 2 (K, V) * 8 heads * (code row + 4) * 2.
tree_accept_greedy: batch 64, 16 nodes.  Both are timed as 50 back-to-back calls in a CUDA graph (per call: the replay time / 50), which
is how the runner's step issues them; an eager call of these small kernels would time the host.
End to end (unless --no-e2e): the decode runner (Llama-3-8B W4A8KV4, batch 64, ctx 1024, all layers), captured verify graphs: the chain
verify of n tokens against the tree step (tree verify + acceptance + compaction of every layer) of n nodes, n in (4, 8, 16), alternating.
The device name, power limit and maximum SM clock are read in the same run.  Writes DIR/tree_verify_bench.json.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from qserve_b200 import backend  # noqa: E402

HQ, HKV, D = 32, 8, 128
B = 64
ROPE = 500000.0


def _device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=60)
        power, clock = (x.strip() for x in r.stdout.strip().split(","))
        info.update(power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        info.update(power_limit=None, max_sm_clock=None, nvidia_smi_error=str(e))
    return info


def _alternate(fns, iters, warmup=20):
    """Median time (us) of each function, launches interleaved one by one."""
    for _ in range(warmup):
        for f in fns:
            f()
    ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for _ in fns]
    for i in range(iters):
        for f, e in zip(fns, ev):
            e[i][0].record()
            f()
            e[i][1].record()
    torch.cuda.synchronize()
    out = []
    for e in ev:
        t = sorted(s.elapsed_time(x) for s, x in e)
        out.append(t[len(t) // 2] * 1e3)
    return out


def _graph_time(fn, iters, per_graph=50):
    """Device time (us) of one call of a small kernel: per_graph calls captured in a CUDA graph (as the runner runs them), the median of
    iters replays over per_graph.  Timing single eager calls would measure the host's launch and argument checks instead."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            fn()
    t, = _alternate([g.replay], iters, 5)
    return t / per_graph


def _pool(pages, bits, dev, g, hkv=HKV):
    code_bytes = hkv * 64 * D * bits // 8
    page_bytes = code_bytes + hkv * 64 * 4
    p = torch.randint(0, 256, (pages, page_bytes), dtype=torch.uint8, device=dev, generator=g)
    meta = p[:, code_bytes:].view(torch.float16).view(pages, 2, hkv * 64)
    meta[:, 0] = (torch.rand(pages, hkv * 64, device=dev, generator=g) * 0.09 + 0.01).half()
    meta[:, 1] = (torch.rand(pages, hkv * 64, device=dev, generator=g) * (15.0 if bits == 4 else 255.0)).half()
    return p, page_bytes


def random_tree(n, g):
    m = [0] * n
    for i in range(1, n):
        p = int(torch.randint(0, i, (1,), generator=g))
        m[i] = m[p] | (1 << p)
    return m


def attention_case(P, n, bits, iters, rounds, dev):
    g = torch.Generator(device=dev).manual_seed(P * 7 + n + bits)
    gc = torch.Generator().manual_seed(P + n)
    nb = (P + n + 63) // 64
    kp, pb = _pool(B * nb, bits, dev, g)
    vp, _ = _pool(B * nb, bits, dev, g)
    bt = torch.arange(B * nb, device=dev, dtype=torch.int64).view(B, nb)
    table = torch.stack([kp.data_ptr() + bt * pb, vp.data_ptr() + bt * pb], dim=1).contiguous()
    spt = HKV * D * bits // 8
    T = B * n
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, device=dev, generator=g).half()
    cu = torch.arange(0, T + 1, n, dtype=torch.int32, device=dev)
    prefix = torch.full((B,), P, dtype=torch.int32, device=dev)
    mask = torch.tensor([w for _ in range(B) for w in random_tree(n, gc)], dtype=torch.int32, device=dev)
    backend.apply_bias_rope_update_kv_cache_at(qkv, torch.full((B,), n, dtype=torch.int32, device=dev), backend.compute_padding_offsets(cu, n, T), prefix,
                                               table, HQ, HKV, n, 64, spt, D, ROPE, 8192, True, bits == 4, True, tree_mask=mask)
    q, k, v = (x.reshape(T, -1, D) for x in qkv.split([HQ * D, HKV * D, HKV * D], dim=-1))
    chain = lambda: backend.multi_token_decode_attention(q, k, v, cu, n, prefix, P, table, 64, spt, bits == 4)
    tree = lambda: backend.multi_token_decode_attention(q, k, v, cu, n, prefix, P, table, 64, spt, bits == 4, tree_mask=mask)
    runs = [_alternate([chain, tree], iters) for _ in range(rounds)]
    return {"batch": B, "prefix": P, "n": n, "kv_bits": bits, "chain_us": [round(r[0], 2) for r in runs], "tree_us": [round(r[1], 2) for r in runs],
            "tree_over_chain": [round(r[1] / r[0], 3) for r in runs]}


def compact_case(bits, iters, dev, layers=32, a=4, n=16):
    g = torch.Generator(device=dev).manual_seed(bits)
    P = 1024
    nb = (P + n + 63) // 64
    pools, tables = [], []
    bt = torch.arange(B * nb, device=dev, dtype=torch.int64).view(B, nb)
    for _ in range(layers):
        kp, pb = _pool(B * nb, bits, dev, g)
        vp, _ = _pool(B * nb, bits, dev, g)
        pools += [kp, vp]
        tables.append(torch.stack([kp.data_ptr() + bt * pb, vp.data_ptr() + bt * pb], dim=1))
    table = torch.stack(tables).contiguous()
    start = torch.full((B,), P, dtype=torch.int32, device=dev)
    path = torch.full((B, n), -1, dtype=torch.int32, device=dev)
    path[:, :a] = torch.tensor([0, 3, 7, 12][:a], dtype=torch.int32)
    acc = torch.full((B,), a, dtype=torch.int32, device=dev)
    spt = HKV * D * bits // 8
    t = _graph_time(lambda: backend.kv_cache_compact(table, start, path, acc, HKV, 64, spt, bits == 4), iters)
    moved = layers * B * (a - 1) * 2 * HKV * (D * bits // 8 + 4) * 2
    return {"layers": layers, "batch": B, "accept_len": a, "kv_bits": bits, "time_us": round(t, 2), "bytes_moved": moved,
            "achieved_gb_s": round(moved / (t * 1e-6) / 1e9, 1)}


def accept_case(iters, dev, n=16):
    g = torch.Generator(device=dev).manual_seed(1)
    gc = torch.Generator().manual_seed(1)
    draft = torch.randint(0, 3, (B, n), device=dev, generator=g)
    target = torch.randint(0, 3, (B, n), device=dev, generator=g)
    mask = torch.tensor([random_tree(n, gc) for _ in range(B)], dtype=torch.int32, device=dev)
    outs = (torch.empty(B, dtype=torch.int32, device=dev), torch.empty((B, n), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int64, device=dev))
    t = _graph_time(lambda: backend.tree_accept_greedy(draft, mask, target, *outs), iters)
    return {"batch": B, "nodes": n, "time_us": round(t, 2)}


def run_e2e(iters, rounds, dev):
    from qserve_b200.decode import DecodeRunner
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=1024, device=dev, verify_len=16)
    gc = torch.Generator().manual_seed(5)
    res = {"model": "llama-3-8b", "precision": "w4a8kv4", "batch": B, "ctx": 1024}
    for n in (4, 8, 16):
        run.v_tree_mask[:, :n].copy_(torch.tensor([random_tree(n, gc) for _ in range(B)], dtype=torch.int32))
        run.capture_verify(n)
        run.capture_verify(n, tree=True)
        runs = [_alternate([lambda: run.verify_step(n), lambda: run.verify_step(n, tree=True)], iters, 3) for _ in range(rounds)]
        res[f"n{n}"] = {"chain_verify_ms": [round(r[0] / 1e3, 3) for r in runs], "tree_step_ms": [round(r[1] / 1e3, 3) for r in runs]}
        print(json.dumps({f"n{n}": res[f"n{n}"]}), flush=True)
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
    res = {"config": {"num_heads": HQ, "num_kv_heads": HKV, "head_dim": D, "batch": B, "iters": args.iters, "rounds": args.rounds}, **_device_info(),
           "attention": [], "compact": [], "accept": None}
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}), flush=True)
    for bits in (4, 8):
        for P in (1024, 4096):
            for n in (4, 8, 16):
                r = attention_case(P, n, bits, args.iters, args.rounds, dev)
                res["attention"].append(r)
                print(json.dumps(r), flush=True)
                torch.cuda.empty_cache()
    for bits in (4, 8):
        r = compact_case(bits, args.iters, dev)
        res["compact"].append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    res["accept"] = accept_case(args.iters, dev)
    print(json.dumps(res["accept"]), flush=True)
    if not args.no_e2e:
        res["end_to_end"] = run_e2e(args.e2e_iters, args.rounds, dev)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "tree_verify_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
