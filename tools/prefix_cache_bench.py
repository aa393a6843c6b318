"""Automatic prefix caching over the shared KV page pool, on and off (DESIGN.md 3.12 "Prefix cache", 5).

    python tools/prefix_cache_bench.py --out DIR [--requests 128] [--reps 2] [--profile-steps 20]

Llama-3-8B W4A8KV4-g128, ctx 1024, max_new_tokens 512, chunk C = 512, B = 64, a pool of half the own-pages footprint (32 x 25 = 800 pages,
tools/kv_pool_bench.py's run c), so that pages are evicted and rows preempted.  Workloads (max_tokens uniform over 16 .. 256, no eos):
  (a) system: one 512-token system prompt followed by 64 .. 512 unique tokens, all submitted at t = 0;
  (b) chat: requests / 3 three-turn conversations; turn k + 1 (turn k's prompt, its answer and 64 new tokens) is submitted when turn k is
      polled, turn 1 of every conversation at t = 0 (prompts 64 .. 512 tokens);
  (c) no sharing: tools/kv_pool_bench.py's script of unique prompts (64 .. 1024 tokens), to bound the cache's overhead.
One runner with the cache and one without are built once; every workload runs on both, alternated, --reps times.  Each run replays the
captured mixed step while prompt tokens are pending and the decode-only step otherwise, and polls after every step.  Reported per run:
generated tokens/s over the wall-clock of the script, time to first token (mean, p90), prompt tokens submitted and computed (chunk tokens
carried), hit tokens, evictions and preemptions (counter deltas).  A separate eager profile of --profile-steps mixed steps of workload (a)
(torch.profiler) gives the schedule kernel's mean device time with and without the cache.  The device name and power limit are read in the
same run.  Writes DIR/prefix_cache_bench.json.
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
from kv_pool_bench import OWN_BLOCKS, _schedule_us  # noqa: E402
from kv_pool_bench import _script as _unique_script  # noqa: E402
from qserve_b200.decode import DecodeRunner  # noqa: E402

CTX, NEW, CHUNK, B, VOCAB = 1024, 512, 512, 64, 128256
PAGES = 32 * OWN_BLOCKS
QUEUE = 512


def _workloads(n):
    rng = random.Random(99)
    system = [rng.randrange(VOCAB) for _ in range(512)]
    a = [(system + [rng.randrange(VOCAB) for _ in range(rng.randint(64, 512))], rng.randint(16, 256)) for _ in range(n)]
    chats = [([rng.randrange(VOCAB) for _ in range(rng.randint(64, 512))], [rng.randint(16, 256) for _ in range(3)],
              [[rng.randrange(VOCAB) for _ in range(64)] for _ in range(2)]) for _ in range(n // 3)]
    prompts, lens, budgets = _unique_script(n, VOCAB)
    c = [(prompts[i, : lens[i]].tolist(), min(budgets[i], 256)) for i in range(n)]
    return {"a_system": a, "b_chat": chats, "c_unique": c}


def _serve(run, kind, work):
    """Serve one workload to the end; returns the run's figures."""
    st0 = run.prefix_cache_stats() if run.prefix_cache else None
    pre0 = run.pool_stats().preemptions
    queue, chats, submitted_at = [], {}, {}
    if kind == "b_chat":
        for ci, (p, budgets, news) in enumerate(work):
            queue.append((p, budgets[0], (ci, 0)))
    else:
        queue = [(p, m, None) for p, m in work]
    prompt_tokens = computed = generated = 0
    first, n_req = {}, 0
    t0 = time.perf_counter()

    def submit(items):
        nonlocal prompt_tokens, n_req
        if not items:
            return
        width = max(len(p) for p, _, _ in items)
        t = torch.tensor([p + [0] * (width - len(p)) for p, _, _ in items], dtype=torch.int64)
        ids = run.submit(t, [len(p) for p, _, _ in items], max_tokens=[m for _, m, _ in items])
        for r, (p, m, tag) in zip(ids, items):
            submitted_at[r] = time.perf_counter() - t0
            prompt_tokens += len(p)
            if tag is not None:
                chats[r] = (tag, p)
        n_req += len(items)

    submit(queue)
    finished, pending = 0, 1
    while finished < n_req:
        mixed = pending > 0
        run.inflight_step(mixed)
        if mixed:
            computed += int(run.i_plan.cu_seqlens[-1])
        polled = run.poll()
        pending = polled.pending_tokens
        now = time.perf_counter() - t0
        for r in run.i_rows.request.tolist():
            if r >= 0 and r not in first:
                first[r] = None
        seq, plen, req = run.s_seq_lens.tolist(), run.s_prompt_lens.tolist(), run.i_rows.request.tolist()
        for b in range(run.batch):
            if req[b] >= 0 and first.get(req[b]) is None and seq[b] > plen[b]:
                first[req[b]] = now
        nxt = []
        for e in polled.finished:
            finished += 1
            generated += len(e[1])
            if first.get(e[0]) is None:
                first[e[0]] = now
            if e[0] in chats:
                (ci, k), p = chats.pop(e[0])
                if k < 2:
                    _, budgets, news = work[ci]
                    q = (p + e[1] + news[k])[:CTX]
                    nxt.append((q, budgets[k + 1], (ci, k + 1)))
        submit(nxt)
        pending = max(pending, len(nxt))
    wall = time.perf_counter() - t0
    res = {"requests": n_req, "generated_tokens": generated, "wall_s": wall, "generated_tokens_per_s": generated / wall,
           "ttft_ms": _stats([(first[r] - submitted_at[r]) * 1e3 for r in submitted_at]), "prompt_tokens_submitted": prompt_tokens,
           "prompt_tokens_computed": computed, "preemptions": run.pool_stats().preemptions - pre0}
    if st0 is not None:
        st = run.prefix_cache_stats()
        res.update(hit_tokens=st.hit_tokens - st0.hit_tokens, evictions=st.evictions - st0.evictions)
    else:
        res.update(hit_tokens=0, evictions=0)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefix_cache_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"workload": {"model": "llama-3-8b", "precision": "w4a8kv4-g128", "ctx": CTX, "max_new_tokens": NEW, "chunk": CHUNK, "batch": B,
                        "pool_pages": PAGES, "requests": args.requests, "max_tokens": "uniform 16 .. 256"}, **_device_info(), "runs": []}
    work = _workloads(args.requests)
    with torch.no_grad():
        runs = {}
        for cache in (False, True):
            run = DecodeRunner("llama-3-8b", "w4a8kv4-g128", B, CTX, dev, generate=True, max_new_tokens=NEW, prompt_tokens=CHUNK, inflight=QUEUE,
                               kv_pool_pages=PAGES, prefix_cache=cache)
            run.capture_inflight(True)
            run.capture_inflight(False)
            runs[cache] = run
        torch.cuda.synchronize()
        for rep in range(args.reps):
            for kind in ("a_system", "b_chat", "c_unique"):
                for cache in (False, True):
                    r = {"rep": rep, "workload": kind, "prefix_cache": cache, **_serve(runs[cache], kind, work[kind])}
                    res["runs"].append(r)
                    print(json.dumps(r), flush=True)
        if args.profile_steps:
            a = work["a_system"]
            width = max(len(p) for p, _ in a)
            script = (torch.tensor([p + [0] * (width - len(p)) for p, _ in a], dtype=torch.int64), [len(p) for p, _ in a], [m for _, m in a])
            res["schedule_kernel"] = {str(cache): _schedule_us(runs[cache], script, args.profile_steps) for cache in (False, True)}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "prefix_cache_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res.get("schedule_kernel")))


if __name__ == "__main__":
    main()
