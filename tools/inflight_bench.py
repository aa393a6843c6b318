"""In-flight batching against static batching on BASELINE config 3 (DESIGN.md 3.12, 5).

    python tools/inflight_bench.py --out DIR [--requests 256] [--layers 32] [--bench-json FILE]

Llama-3-8B W4A8KV4-g128, all layers, batch 64, prompts of 1024 tokens, per-request max_tokens drawn from a seeded uniform distribution over
16 .. 512 (no eos, so rows finish at their budgets, at different times).  The script runs twice: every request submitted at t = 0, and with
seeded Poisson arrivals (40 requests/s).
  * In-flight: DecodeRunner(inflight=256, prompt_tokens=C) for C in 128, 256, 512; the captured mixed step while prompt tokens are pending,
    the captured decode-only step otherwise, a poll (one host synchronisation) after every step.  Per step the host reads which rows advanced,
    so each request's first-token step and its inter-token gaps are known in steps and in wall-clock ms.
  * Static: batches of 64 requests in arrival order, prefill(chunk=512), then the captured generate_step until every row is done (checked
    every 16 steps).  A batch starts when its last request has arrived.
Reported: generated tokens/s over the wall-clock of the whole script, time-to-first-token and inter-token time (mean and p90, steps and ms;
the in-flight ITL is the wall-clock gap between the polls after a request's consecutive tokens, the static ITL is each batch's decode-loop
wall-clock divided by its steps, given to every token of the batch, because the static loop does not synchronise per step),
mean ms of the mixed and decode-only steps (CUDA events) against the static run's generate_step, and bench.py's config3_ifb_round estimate
(from --bench-json, a bench.py output line, when given).  The device name and power limit are read in the same run.  Writes
DIR/inflight_bench.json.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from qserve_b200.decode import DecodeRunner  # noqa: E402

B, CTX, NEW = 64, 1024, 512
RATE = 40.0  # Poisson arrivals, requests per second


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


def _stats(xs):
    if not xs:
        return {"mean": None, "p90": None}
    xs = sorted(xs)
    return {"mean": sum(xs) / len(xs), "p90": xs[min(len(xs) - 1, int(0.9 * len(xs)))]}


def _script(n, vocab, poisson):
    rng = random.Random(1234)
    prompts = torch.randint(0, vocab, (n, CTX), generator=torch.Generator().manual_seed(99))
    budgets = [rng.randint(16, NEW) for _ in range(n)]
    t, arrivals = 0.0, []
    for _ in range(n):
        arrivals.append(t if poisson else 0.0)
        t += rng.expovariate(RATE)
    return prompts, budgets, arrivals


def run_inflight(C, script, layers, dev):
    prompts, budgets, arrivals = script
    n = len(budgets)
    run = DecodeRunner("llama-3-8b", "w4a8kv4-g128", B, CTX, dev, layers=layers, generate=True, max_new_tokens=NEW, prompt_tokens=C, inflight=n)
    run.capture_inflight(True)
    run.capture_inflight(False)
    torch.cuda.synchronize()
    ev = []
    step_kind, step_end = [], []
    first, last_tok, gaps_steps, gaps_ms, generated = {}, {}, [], [], 0
    counts = {}
    nxt, pending, finished = 0, 0, 0
    t0 = time.perf_counter()
    while finished < n:
        now = time.perf_counter() - t0
        k = nxt
        while k < n and arrivals[k] <= now:
            k += 1
        if k > nxt:
            run.submit(prompts[nxt:k], [CTX] * (k - nxt), max_tokens=budgets[nxt:k])
            pending += CTX * (k - nxt)
            nxt = k
        if finished == nxt and nxt < n:
            time.sleep(max(0.0, arrivals[nxt] - now))  # nothing to run until the next arrival
            continue
        mixed = pending > 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run.inflight_step(mixed)
        e1.record()
        ev.append((e0, e1))
        step_kind.append(mixed)
        polled = run.poll()
        pending = polled.pending_tokens
        tend = time.perf_counter() - t0
        step_end.append(tend)
        s = len(step_end) - 1
        req, seq, plen = (t.tolist() for t in (run.i_rows.request, run.s_seq_lens, run.s_prompt_lens))
        for b in range(B):
            r = req[b]
            if r < 0:
                continue
            c = seq[b] - plen[b]
            if c > counts.get(r, 0):
                if r not in first:
                    first[r] = (s, tend)
                else:
                    ps, pt = last_tok[r]
                    gaps_steps.append(s - ps)
                    gaps_ms.append((tend - pt) * 1e3)
                last_tok[r] = (s, tend)
                counts[r] = c
        for e in polled.finished:
            finished += 1
            generated += len(e[1])
            if e[0] not in first:  # admitted and finished between two reads (cannot happen: a request lives at least one step)
                first[e[0]] = (s, tend)
    wall = time.perf_counter() - t0
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    mixed_ms = [m for m, k in zip(ms, step_kind) if k]
    dec_ms = [m for m, k in zip(ms, step_kind) if not k]
    arr_step = {}
    for r in range(n):  # the first step that ended after the arrival
        arr_step[r] = next(i for i, t in enumerate(step_end) if t >= arrivals[r])
    ttft_steps = [first[r][0] - arr_step[r] + 1 for r in range(n)]
    ttft_ms = [(first[r][1] - arrivals[r]) * 1e3 for r in range(n)]
    del run
    torch.cuda.empty_cache()
    return {"chunk": C, "generated_tokens": generated, "wall_s": wall, "generated_tokens_per_s": generated / wall, "steps": len(ms),
            "mixed_steps": len(mixed_ms), "decode_only_steps": len(dec_ms), "mixed_step_ms": _stats(mixed_ms), "decode_only_step_ms": _stats(dec_ms),
            "ttft_steps": _stats(ttft_steps), "ttft_ms": _stats(ttft_ms), "itl_steps": _stats(gaps_steps), "itl_ms": _stats(gaps_ms)}


def run_static(script, layers, dev):
    prompts, budgets, arrivals = script
    n = len(budgets)
    run = DecodeRunner("llama-3-8b", "w4a8kv4-g128", B, CTX, dev, layers=layers, generate=True, max_new_tokens=NEW, prompt_tokens=B * 512)
    p0 = prompts[:B].to(dev)
    lens = torch.full((B,), CTX, dtype=torch.int32, device=dev)
    # bench.py's config3_ifb_round formula over this runner: one prompt step of 8 x 1024 tokens (the other rows take a 1-token prompt), then
    # 512 decode steps at batch 64 per 8 admitted prompts
    few = torch.tensor([CTX] * 8 + [1] * (B - 8), dtype=torch.int32, device=dev)
    run.prefill(p0, few, chunk=512)
    torch.cuda.synchronize()
    t = time.perf_counter()
    run.prefill(p0, few, chunk=512)
    torch.cuda.synchronize()
    prompt_ms = (time.perf_counter() - t) * 1e3
    run.prefill(p0, lens, chunk=512)
    run.capture_generate(1)
    torch.cuda.synchronize()
    gen_ms, generated, ttft_ms, itl_ms = [], 0, [], []
    t0 = time.perf_counter()
    for i in range(0, n, B):
        idx = list(range(i, min(n, i + B)))
        wait = arrivals[idx[-1]] - (time.perf_counter() - t0)
        if wait > 0:
            time.sleep(wait)
        p = prompts[idx + [idx[-1]] * (B - len(idx))].to(dev)
        run.g_budget.copy_(torch.tensor([budgets[r] for r in idx] + [1] * (B - len(idx)), dtype=torch.int32))
        run.prefill(p, lens, chunk=512)
        torch.cuda.synchronize()
        tf = time.perf_counter() - t0
        ttft_ms += [(tf - arrivals[r]) * 1e3 for r in idx]
        steps = 0
        ts = time.perf_counter()
        while True:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run.generate_step(1)
            e1.record()
            gen_ms.append((e0, e1))
            steps += 1
            if steps % 16 == 0 and bool(run.g_finished.all()):
                break
        torch.cuda.synchronize()
        dt = (time.perf_counter() - ts) * 1e3 / steps
        itl_ms += [dt] * sum(budgets[r] - 1 for r in idx)
        generated += int((run.s_seq_lens - run.s_prompt_lens)[: len(idx)].sum())
    wall = time.perf_counter() - t0
    ms = [a.elapsed_time(b) for a, b in gen_ms]
    del run
    torch.cuda.empty_cache()
    dec = _stats(ms)["mean"]
    est = 8 * 512 / ((prompt_ms + 512 * dec * 8 / B) * 1e-3)
    return {"generated_tokens": generated, "wall_s": wall, "generated_tokens_per_s": generated / wall, "generate_step_ms": _stats(ms),
            "prompt_step_8x1024_ms": prompt_ms, "config3_ifb_round_formula_tokens_per_s": est,
            "ttft_ms": _stats(ttft_ms), "itl_ms": _stats(itl_ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--layers", type=int, default=None)
    ap.add_argument("--chunks", default="128,256,512")
    ap.add_argument("--bench-json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"workload": {"model": "llama-3-8b", "precision": "w4a8kv4-g128", "batch": B, "prompt_len": CTX, "max_tokens": "uniform 16 .. 512",
                        "requests": args.requests, "poisson_rate_per_s": RATE, "layers": args.layers or 32}, **_device_info()}
    if args.bench_json and os.path.exists(args.bench_json):
        for line in open(args.bench_json):
            try:
                rec = json.loads(line)
            except ValueError:
                continue
            if "config3_ifb_round" in rec:
                res["bench_config3_ifb_round_tokens_per_s"] = rec["config3_ifb_round"]["tokens_per_s"]
    with torch.no_grad():
        for mode, poisson in (("all_at_t0", False), ("poisson", True)):
            script = _script(args.requests, 128256, poisson)
            out = {"static": run_static(script, args.layers, dev)}
            for C in (int(c) for c in args.chunks.split(",")):
                out[f"inflight_C{C}"] = run_inflight(C, script, args.layers, dev)
            res[mode] = out
            print(json.dumps({mode: out}), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "inflight_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
