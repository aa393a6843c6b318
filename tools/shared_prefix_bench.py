"""Shared-prefix decode attention: time qs_shared_prefix_decode_attention against single_query_attention_quant on the same pages.

    python tools/shared_prefix_bench.py --out DIR [--iters 200] [--e2e-iters 100] [--no-e2e]

Per launch: Llama-3-8B heads (32 query / 8 KV heads, head_dim 128), batch 64 split into groups of m in (1, 2, 4, 8, 16, 64) rows that share a
prefix of P in (1024, 4096) tokens (S = P / 64 pages), each row with its own suffix of s in (1, 64, 256) tokens (the last one the new token), KV4
and KV8.  Both arms write the fused per-token quantisation (the runner's form).  Each time is the median of --iters launches per arm, timed one
by one with CUDA events, the two arms alternated launch by launch after a warm-up.  Unique page bytes per arm: the baseline streams every
row's P + s - 1 cached tokens, the op each group's P once plus every row's s - 1.
End to end (unless --no-e2e): the decode runner (Llama-3-8B W4A8KV4, batch 64 = 8 prompts x 8 rows forked from each, ctx 1024 and 4096, all
layers, captured plain step) with and without shared_prefix=True, ms per step, the two graphs alternated.  The device name, power limit and
maximum SM clock are read in the same run.  Writes DIR/shared_prefix_bench.json.
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

HQ, HKV, D, B = 32, 8, 128, 64
GROUPS, PREFIXES, SUFFIXES = (1, 2, 4, 8, 16, 64), (1024, 4096), (1, 64, 256)
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


def _time_pair(fa, fb, iters, warmup=20):
    """Median µs of fa and fb, launched alternately, each launch between its own pair of events."""
    for _ in range(warmup):
        fa(); fb()
    ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for _ in range(2)]
    for i in range(iters):
        for f, e in zip((fa, fb), ev):
            e[i][0].record()
            f()
            e[i][1].record()
    torch.cuda.synchronize()
    med = []
    for e in ev:
        t = sorted(s.elapsed_time(x) for s, x in e)
        med.append(t[len(t) // 2] * 1e3)
    return med


def _pool(pages, bits, dev, g):
    code_bytes = HKV * 64 * D * bits // 8
    page_bytes = code_bytes + HKV * 64 * 4
    p = torch.randint(0, 256, (pages, page_bytes), dtype=torch.uint8, device=dev, generator=g)
    meta = p[:, code_bytes:].view(torch.float16).view(pages, 2, HKV * 64)
    meta[:, 0] = (torch.rand(pages, HKV * 64, device=dev, generator=g) * 0.09 + 0.01).half()
    meta[:, 1] = (torch.rand(pages, HKV * 64, device=dev, generator=g) * (15.0 if bits == 4 else 255.0)).half()
    return p, page_bytes


def run_case(m, P, s, bits, iters, dev):
    g = torch.Generator(device=dev).manual_seed(m * 131 + P * 7 + s + bits)
    L = P + s  # context length including the new token
    nb = (L + 63) // 64
    kp, pb = _pool(B * nb, bits, dev, g)
    vp, _ = _pool(B * nb, bits, dev, g)
    bt = torch.arange(B * nb, device=dev, dtype=torch.int64).view(B, nb)
    S = P // 64
    first = (torch.arange(B, device=dev) // m) * m
    bt[:, :S] = bt[first, :S]
    table = torch.stack([kp.data_ptr() + bt * pb, vp.data_ptr() + bt * pb], dim=1).contiguous()
    spt = HKV * D * bits // 8
    qkv = torch.randn(B, (HQ + 2 * HKV) * D, device=dev, generator=g).half()
    q, k, v = (x.reshape(B, -1, D) for x in qkv.split([HQ * D, HKV * D, HKV * D], dim=-1))
    lens = torch.full((B,), L, dtype=torch.int32, device=dev)
    layout = backend.shared_prefix_layout([list(range(j, j + m)) for j in range(0, B, m)], [S] * (B // m), B, device=dev)
    oq = torch.empty((B, HQ * D), dtype=torch.int8, device=dev)
    sc = torch.empty(B, dtype=torch.half, device=dev)
    sm = torch.empty(B, dtype=torch.half, device=dev)
    op = lambda: backend.shared_prefix_decode_attention(q, k, v, table, lens, layout, 64, spt, L, D, ROPE, bits == 4, True, out_q=oq, out_scale=sc,
                                                        out_sum=sm)
    base = lambda: backend.single_query_attention_quant(q, k, v, table, lens, 8192, 64, spt, L, D, ROPE, bits == 4, True, oq, sc, sm)
    t_op, t_base = _time_pair(op, base, iters)
    per_tok = HKV * (D * bits // 8 * 2 + 8)
    return {"group": m, "prefix": P, "suffix": s, "kv_bits": bits, "op_us": round(t_op, 2), "decode_us": round(t_base, 2),
            "op_over_decode": round(t_op / t_base, 3), "op_page_bytes": (B // m * P + B * (s - 1)) * per_tok, "decode_page_bytes": B * (L - 1) * per_tok}


def run_e2e(iters, dev):
    from qserve_b200.decode import DecodeRunner
    res = []
    for ctx in (1024, 4096):
        runs = []
        for flag in (False, True):
            run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=ctx, device=dev, shared_prefix=flag)
            for p in range(0, B, 8):
                run.fork(p, list(range(p + 1, p + 8)))
            run.capture()
            runs.append(run)
        t_off, t_on = _time_pair(runs[0].step, runs[1].step, iters, 5)
        res.append({"model": "llama-3-8b", "precision": "w4a8kv4", "batch": B, "ctx": ctx, "forks": "8 prompts x 8 rows",
                    "routed_to_op": runs[1]._sp_layout is not None, "step_ms": round(t_off / 1e3, 3), "shared_prefix_step_ms": round(t_on / 1e3, 3)})
        del runs
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--e2e-iters", type=int, default=100)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    assert args.iters >= 200
    dev = torch.device("cuda:0")
    res = {"config": {"num_heads": HQ, "num_kv_heads": HKV, "head_dim": D, "batch": B, "iters": args.iters}, **_device_info(), "cases": []}
    for bits in (4, 8):
        for P in PREFIXES:
            for s in SUFFIXES:
                for m in GROUPS:
                    r = run_case(m, P, s, bits, args.iters, dev)
                    res["cases"].append(r)
                    print(json.dumps(r), flush=True)
                    torch.cuda.empty_cache()
    if not args.no_e2e:
        res["end_to_end"] = run_e2e(args.e2e_iters, dev)
        print(json.dumps(res["end_to_end"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "shared_prefix_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}))


if __name__ == "__main__":
    main()
