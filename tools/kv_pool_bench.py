"""In-flight batching over a shared KV page pool against rows that own their pages (DESIGN.md 3.12, 5).

    python tools/kv_pool_bench.py --out DIR [--requests 384] [--layers 32] [--profile-steps 20]

Llama-3-8B W4A8KV4-g128, ctx 1024, max_new_tokens 512, chunk C = 512.  One seeded script of mixed requests, all submitted at t = 0: prompt
lengths uniform over 64 .. 1024 and max_tokens uniform over 16 .. 512 (no eos, so rows end at their budgets).  Runs:
  (a) own pages, B = 64: 64 x 25 pages, enough for the worst case of every row;
  (b) a pool of the same 1600 pages at B = 128 and at B = 96;
  (c) a pool of half the pages (800) at B = 64.
Each run captures the mixed and decode-only in-flight steps, replays the mixed step while prompt tokens are pending and the decode-only one
otherwise, and polls after every step (tools/inflight_bench.py's loop).  Reported per run: generated tokens/s over the wall-clock of the
script, time-to-first-token and inter-token time (mean and p90, ms), mean step times (CUDA events), preemptions, starts and peak pages in use,
and, from a separate eager profile of --profile-steps mixed steps (torch.profiler), the schedule kernel's mean device time per step.  The
device name and power limit are read in the same run.  Writes DIR/kv_pool_bench.json.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from inflight_bench import _device_info, _stats  # noqa: E402
from qserve_b200.decode import DecodeRunner  # noqa: E402

CTX, NEW, CHUNK = 1024, 512, 512
OWN_BLOCKS = (max(CTX + NEW + 1, CTX - 1 + CHUNK) + 63) // 64  # the own-pages runner's pages per row
RUNS = [("a_own_B64", 64, 0), ("b_pool_B128", 128, 64 * OWN_BLOCKS), ("b_pool_B96", 96, 64 * OWN_BLOCKS), ("c_pool_half_B64", 64, 32 * OWN_BLOCKS)]


def _script(n, vocab):
    rng = random.Random(4321)
    lens = [rng.randint(64, CTX) for _ in range(n)]
    budgets = [rng.randint(16, NEW) for _ in range(n)]
    prompts = torch.randint(0, vocab, (n, CTX), generator=torch.Generator().manual_seed(77))
    return prompts, lens, budgets


def _schedule_us(run, script, steps):
    """Mean device time of the schedule kernel over `steps` eager mixed steps, under torch.profiler."""
    prompts, lens, budgets = script
    k = min(len(lens), 2 * run.batch)
    run.submit(prompts[:k], lens[:k], max_tokens=budgets[:k])
    for _ in range(3):
        run.inflight_forward(True)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run.inflight_forward(True)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "inflight_schedule_kernel" in e.name]
    return {"mean_us": sum(times) / len(times) if times else None, "launches": len(times)}


def run_one(name, B, pages, script, layers, profile_steps, dev):
    prompts, lens, budgets = script
    n = len(lens)
    run = DecodeRunner("llama-3-8b", "w4a8kv4-g128", B, CTX, dev, layers=layers, generate=True, max_new_tokens=NEW, prompt_tokens=CHUNK, inflight=n,
                       kv_pool_pages=pages)
    run.capture_inflight(True)
    run.capture_inflight(False)
    torch.cuda.synchronize()
    ev, kinds = [], []
    first, last_tok, gaps_ms, counts, generated, finished = {}, {}, [], {}, 0, 0
    t0 = time.perf_counter()
    run.submit(prompts, lens, max_tokens=budgets)
    pending = sum(lens)
    while finished < n:
        mixed = pending > 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run.inflight_step(mixed)
        e1.record()
        ev.append((e0, e1))
        kinds.append(mixed)
        polled = run.poll()
        pending = polled.pending_tokens
        tend = time.perf_counter() - t0
        req, seq, plen = (t.tolist() for t in (run.i_rows.request, run.s_seq_lens, run.s_prompt_lens))
        for b in range(B):
            r = req[b]
            if r < 0:
                continue
            c = seq[b] - plen[b]
            if c > counts.get(r, 0):
                if r in last_tok:
                    gaps_ms.append((tend - last_tok[r]) * 1e3)
                first.setdefault(r, tend)
                last_tok[r] = tend
                counts[r] = c
        for e in polled.finished:
            finished += 1
            generated += len(e[1])
            first.setdefault(e[0], tend)
    wall = time.perf_counter() - t0
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    stats = run.pool_stats()._asdict() if pages else {"free_pages": None, "peak_pages": None, "preemptions": 0, "starts": None}
    res = {"batch": B, "pages": pages or B * run.table_blocks, "pool": bool(pages), "generated_tokens": generated, "wall_s": wall,
           "generated_tokens_per_s": generated / wall, "steps": len(ms), "mixed_step_ms": _stats([m for m, k in zip(ms, kinds) if k]),
           "decode_only_step_ms": _stats([m for m, k in zip(ms, kinds) if not k]), "ttft_ms": _stats([first[r] * 1e3 for r in range(n)]),
           "itl_ms": _stats(gaps_ms), **stats}
    if profile_steps:
        res["schedule_kernel"] = _schedule_us(run, script, profile_steps)
    del run
    torch.cuda.empty_cache()
    print(json.dumps({name: res}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--requests", type=int, default=384)
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--runs", default=",".join(r[0] for r in RUNS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_pool_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"workload": {"model": "llama-3-8b", "precision": "w4a8kv4-g128", "ctx": CTX, "max_new_tokens": NEW, "chunk": CHUNK,
                        "prompt_len": "uniform 64 .. 1024", "max_tokens": "uniform 16 .. 512", "requests": args.requests, "arrivals": "all at t = 0",
                        "layers": args.layers or 32}, **_device_info()}
    script = _script(args.requests, 128256)
    want = set(args.runs.split(","))
    with torch.no_grad():
        for name, B, pages in RUNS:
            if name in want:
                res[name] = run_one(name, B, pages, script, args.layers, args.profile_steps, dev)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "kv_pool_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
