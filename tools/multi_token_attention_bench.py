"""Speculative-decoding verification: time qs_multi_token_decode_attention against the ways the library could verify n draft tokens before it.

    python tools/multi_token_attention_bench.py --out DIR [--iters 200] [--e2e-iters 100] [--no-e2e]

Attention cases: Llama-3-8B heads (32 query / 8 KV heads, head_dim 128), batch in (8, 64), cached prefix P in (1024, 4096), n in (1, 2, 4, 8, 16)
draft tokens per sequence, KV4 and KV8.  Per case, each the median of --iters launches timed one by one with CUDA events after a warm-up:
  * the new op;
  * prefix_prefill_attention on the same inputs (the prompt-chunk path, which is not what decoding computes);
  * one single_query_attention launch on the same cache (one decode step), and n times it;
  * the bytes the op must move, B * Hkv * (P + n) * (D * bits / 8 * 2 + 8) of KV pages plus q / k / v in and the output, and the achieved share
    of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM.
End to end (unless --no-e2e): the decode runner's verify graph (Llama-3-8B W4A8KV4, batch 64, ctx 1024, all layers, n in (1, 2, 4, 8)) against
its decode-step graph, ms per step.  The device name, power limit and maximum SM clock are read in the same run.  Writes
DIR/multi_token_attention_bench.json.
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
BATCHES, PREFIXES, DRAFTS = (8, 64), (1024, 4096), (1, 2, 4, 8, 16)
PEAK_BW = 3.35e12
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


def _time(fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for s, e in ev:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    t = sorted(s.elapsed_time(e) for s, e in ev)
    return t[len(t) // 2] * 1e3  # us


def _pool(pages, bits, dev, g):
    """Random pages: codes uniform, scale ~ U(0.01, 0.1), zero ~ U(0, 15 | 255) (the statistics of the parity tests)."""
    code_bytes = HKV * 64 * D * bits // 8
    page_bytes = code_bytes + HKV * 64 * 4
    p = torch.randint(0, 256, (pages, page_bytes), dtype=torch.uint8, device=dev, generator=g)
    meta = p[:, code_bytes:].view(torch.float16).view(pages, 2, HKV * 64)
    meta[:, 0] = (torch.rand(pages, HKV * 64, device=dev, generator=g) * 0.09 + 0.01).half()
    meta[:, 1] = (torch.rand(pages, HKV * 64, device=dev, generator=g) * (15.0 if bits == 4 else 255.0)).half()
    return p, page_bytes


def run_case(B, P, n, bits, iters, dev):
    g = torch.Generator(device=dev).manual_seed(B * 131 + P * 7 + n + bits)
    nb = (P + n + 63) // 64
    pages = B * nb
    kp, pb = _pool(pages, bits, dev, g)
    vp, _ = _pool(pages, bits, dev, g)
    bt = torch.arange(pages, device=dev, dtype=torch.int64).view(B, nb)
    table = torch.stack([kp.data_ptr() + bt * pb, vp.data_ptr() + bt * pb], dim=1).contiguous()
    spt = HKV * D * bits // 8
    T = B * n
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, device=dev, generator=g).half()
    cu = torch.arange(0, T + 1, n, dtype=torch.int32, device=dev)
    prefix = torch.full((B,), P, dtype=torch.int32, device=dev)
    backend.apply_bias_rope_update_kv_cache_at(qkv, torch.full((B,), n, dtype=torch.int32, device=dev), backend.compute_padding_offsets(cu, n, T), prefix,
                                               table, HQ, HKV, n, 64, spt, D, ROPE, 8192, True, bits == 4, True)
    q, k, v = (x.reshape(T, -1, D) for x in qkv.split([HQ * D, HKV * D, HKV * D], dim=-1))
    t_new = _time(lambda: backend.multi_token_decode_attention(q, k, v, cu, n, prefix, P, table, 64, spt, bits == 4), iters)
    t_prefix = _time(lambda: backend.prefix_prefill_attention(q, k, v, cu, n, prefix, P, table, 64, spt, bits == 4), iters)
    # one decode step over the same cache (it appends its token at slot P, which the verify above has already written)
    dq, dk, dv = (x.reshape(B, n, -1, D)[:, 0].contiguous() for x in (q, k, v))
    lens = torch.full((B,), P + 1, dtype=torch.int32, device=dev)
    t_dec = _time(lambda: backend.single_query_attention(dq, dk, dv, table, lens, None, 8192, 64, spt, P + 1, D, ROPE, True, bits == 4, True), iters)
    kv_bytes = B * HKV * (P + n) * (D * bits // 8 * 2 + 8)
    io_bytes = T * (HQ + 2 * HKV) * D * 2 + T * HQ * D * 2
    bw = (kv_bytes + io_bytes) / (t_new * 1e-6)
    return {"batch": B, "prefix": P, "n": n, "kv_bits": bits, "time_us": round(t_new, 2), "prefix_prefill_us": round(t_prefix, 2),
            "decode_launch_us": round(t_dec, 2), "n_decode_launches_us": round(n * t_dec, 2), "over_one_decode": round(t_new / t_dec, 3),
            "bytes": kv_bytes + io_bytes, "achieved_tb_s": round(bw / 1e12, 3), "share_of_3p35_tb_s": round(bw / PEAK_BW, 4),
            "faster_than_prefix": t_new < t_prefix, "faster_than_n_decodes": t_new < n * t_dec}


def run_e2e(iters, dev):
    from qserve_b200.decode import DecodeRunner
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=64, ctx=1024, device=dev, verify_len=8)
    run.capture()
    res = {"model": "llama-3-8b", "precision": "w4a8kv4", "batch": 64, "ctx": 1024, "decode_step_ms": round(_time(run.step, iters, 5) / 1e3, 3)}
    for n in (1, 2, 4, 8):
        run.capture_verify(n)
        res[f"verify_n{n}_ms"] = round(_time(lambda: run.verify_step(n), iters, 5) / 1e3, 3)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--e2e-iters", type=int, default=100)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    assert args.iters >= 100
    dev = torch.device("cuda:0")
    res = {"config": {"num_heads": HQ, "num_kv_heads": HKV, "head_dim": D, "iters": args.iters}, **_device_info(), "cases": []}
    for bits in (4, 8):
        for B in BATCHES:
            for P in PREFIXES:
                for n in DRAFTS:
                    r = run_case(B, P, n, bits, args.iters, dev)
                    res["cases"].append(r)
                    print(json.dumps(r), flush=True)
                    torch.cuda.empty_cache()
    if not args.no_e2e:
        res["end_to_end"] = run_e2e(args.e2e_iters, dev)
        print(json.dumps(res["end_to_end"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "multi_token_attention_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}))


if __name__ == "__main__":
    main()
