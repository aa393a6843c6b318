"""Prompt chunks over a cached prefix: time qs_prefix_prefill_attention against recomputing the whole prompt with the prompt attention.

    python tools/prefix_attention_bench.py --out DIR [--iters 200]

Llama-3-8B heads (32 query / 8 KV heads, head_dim 128), 8 sequences, (prefix, chunk) in (0,1024) (512,512) (1024,512) (3072,1024) (1024,128),
KV4 and KV8.  Per case: the median of --iters launches timed one by one with CUDA events after a warm-up; the FLOPs the chunk needs,
4 * D * Hq * sum_b C_b * (P_b + (C_b + 1) / 2); the achieved TFLOP/s and its share of the 989 TFLOP/s dense FP16 data-sheet figure of the H100
SXM; and the time of flash_attn_varlen_func (the library's prompt attention) over the same sequences as one fp16 prompt of P + C tokens.
The device name, power limit and maximum SM clock are read in the same run.  Writes DIR/prefix_attention_bench.json.
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

HQ, HKV, D, B = 32, 8, 128, 8
CASES = [(0, 1024), (512, 512), (1024, 512), (3072, 1024), (1024, 128)]
PEAK_TFLOPS = 989.0
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


def run_case(P, C, bits, iters, dev):
    g = torch.Generator(device=dev).manual_seed(P * 7 + C + bits)
    nb = (P + C + 63) // 64
    pages = B * nb
    kp, pb = _pool(pages, bits, dev, g)
    vp, _ = _pool(pages, bits, dev, g)
    bt = torch.arange(pages, device=dev, dtype=torch.int64).view(B, nb)
    table = torch.stack([kp.data_ptr() + bt * pb, vp.data_ptr() + bt * pb], dim=1).contiguous()
    spt = HKV * D * bits // 8
    T = B * C
    qkv = torch.randn(T, (HQ + 2 * HKV) * D, device=dev, generator=g).half()
    cu = torch.arange(0, T + 1, C, dtype=torch.int32, device=dev)
    prefix = torch.full((B,), P, dtype=torch.int32, device=dev)
    backend.apply_bias_rope_update_kv_cache_at(qkv, torch.full((B,), C, dtype=torch.int32, device=dev), backend.compute_padding_offsets(cu, C, T), prefix,
                                               table, HQ, HKV, C, 64, spt, D, ROPE, 8192, True, bits == 4, True)
    q, k, v = (x.reshape(T, -1, D) for x in qkv.split([HQ * D, HKV * D, HKV * D], dim=-1))
    t_new = _time(lambda: backend.prefix_prefill_attention(q, k, v, cu, C, prefix, P, table, 64, spt, bits == 4), iters)
    # full recompute: the same sequences as one fp16 prompt of P + C tokens
    L = P + C
    fqkv = torch.randn(B * L, (HQ + 2 * HKV) * D, device=dev, generator=g).half()
    fq, fk, fv = (x.reshape(B * L, -1, D) for x in fqkv.split([HQ * D, HKV * D, HKV * D], dim=-1))
    fcu = torch.arange(0, B * L + 1, L, dtype=torch.int32, device=dev)
    t_full = _time(lambda: backend.flash_attn_varlen_func(fq, fk, fv, fcu, fcu, L, L, dropout_p=0.0, causal=True), iters)
    flops = 4.0 * D * HQ * B * C * (P + (C + 1) / 2)
    tflops = flops / (t_new * 1e-6) / 1e12
    return {"prefix": P, "chunk": C, "kv_bits": bits, "batch": B, "time_us": round(t_new, 2), "flops": flops, "tflops": round(tflops, 1),
            "share_of_989_tflops": round(tflops / PEAK_TFLOPS, 4), "full_recompute_tokens": L, "full_recompute_time_us": round(t_full, 2),
            "time_over_full_recompute": round(t_new / t_full, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    assert args.iters >= 100
    dev = torch.device("cuda:0")
    res = {"config": {"num_heads": HQ, "num_kv_heads": HKV, "head_dim": D, "batch": B, "iters": args.iters}, **_device_info(), "cases": []}
    for bits in (4, 8):
        for P, C in CASES:
            r = run_case(P, C, bits, args.iters, dev)
            res["cases"].append(r)
            print(json.dumps(r), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "prefix_attention_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("device", "power_limit", "max_sm_clock")}))


if __name__ == "__main__":
    main()
