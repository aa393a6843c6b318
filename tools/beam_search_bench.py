"""Beam search in the decode runner: the captured beam step against the captured greedy step, and its three beam launches.

    python tools/beam_search_bench.py --out DIR [--steps 100] [--layers 32]

Llama-3-8B W4A8KV4, all layers, batch 64 as (requests, beams) = (16, 4) and (8, 8); 1024-token prompts (prefilled in 512-token chunks) and
256 new tokens (length_penalty 1, early_stopping False, no eos).  Per configuration:
  * step: after beam_start, the captured beam step (decode + logprobs_rows(2 W) + beam_select + beam_reorder) and the captured greedy decode step
    (decode + argmax_rows) of the same runner, replayed alternately --steps times, each replay between its own pair of CUDA events; medians and
    their ratio.  The beams advance through the timed window.
  * kernels: logprobs_rows(n = 2 W), beam_select and beam_reorder on the state the last beam step left, each captured alone in a CUDA graph of 20
    launches and replayed 10 times; µs per launch.  Every beam_select launch writes its own copy of the beam state, reset from a snapshot
    between replays, so each launch does the step that follows the snapshot (the requests done after it are reported).  The bytes the
    reorder moves are counted on the host from that state: table entries, filled tail slots (codes, scale, zero) of every layer, K / V and KV
    head, and history columns, read and written.
The device name, power limit and maximum SM clock are read in the same run.  Writes DIR/beam_search_bench.json.
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
from qserve_b200.decode import DecodeRunner  # noqa: E402

B, CTX, NEW, CHUNK = 64, 1024, 256, 512
CONFIGS = ((16, 4), (8, 8))


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


def _median(ms):
    ms = sorted(ms)
    return ms[len(ms) // 2]


def _graph_time(fn, reps=20, replays=10):
    """µs per call of fn, captured `reps` times in one CUDA graph and replayed `replays` times."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    t = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b) * 1e3 / reps)
    return _median(t)


def _select_time(run, reps=20, replays=10):
    """µs per beam_select launch from the state the last beam step left: `reps` launches in one CUDA graph, each on its own copy of the state
    it writes (the copies are reset from a snapshot before every replay, outside the timed window), so every launch does one full step."""
    names = ("b_live", "b_cum", "s_seq_lens", "context_lens", "tokens_in", "b_parent", "b_done")
    snap = {k: getattr(run, k).clone() for k in names}
    pool_snap = [t.clone() for t in run.b_pool]
    copies = [({k: v.clone() for k, v in snap.items()}, backend.BeamPool(*(t.clone() for t in pool_snap))) for _ in range(reps)]

    def reset():
        for st, pool in copies:
            for k, v in st.items():
                v.copy_(snap[k])
            for t, t0 in zip(pool, pool_snap):
                t.copy_(t0)

    def launch(st, pool):
        backend.beam_select(run.b_top_ids, run.b_top_logprobs, st["b_live"], st["b_cum"], st["s_seq_lens"], st["context_lens"], st["tokens_in"],
                            st["b_parent"], run.s_prompt_lens, run.s_history, run.b_length_penalty, run.b_early_stopping, run.b_eos, run.b_stop,
                            run.b_budget, st["b_done"], pool, run.max_model_len)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch(*copies[0])
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for c in copies:
            launch(*c)
    t = []
    for _ in range(replays):
        reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b) * 1e3 / reps)
    done = int(copies[0][0]["b_done"].sum())
    return _median(t), done


def _reorder_bytes(run):
    """Bytes beam_reorder reads and writes for the current parents (2 x what it moves)."""
    W = run.beam_width
    par, ctx, p0 = run.b_parent.tolist(), run.context_lens.tolist(), run.s_prompt_lens.tolist()
    kRow = 128 * run.kv_bits // 8
    moved = rows = 0
    for s, p in enumerate(par):
        if p < 0 or p == s or not s - s % W <= p < s - s % W + W:
            continue
        rows += 1
        P = ctx[s] - 1
        moved += run.L * 2 * (P // 64 * 8 + run.Hkv * (P % 64) * (kRow + 4)) + (P - p0[s]) * 8
    return 2 * moved, rows


def bench(R, W, steps, layers):
    run = DecodeRunner("llama-3-8b", "w4a8kv4", batch=B, ctx=CTX, seed=0, layers=layers, prompt_tokens=R * CHUNK + B, max_new_tokens=NEW, beam_width=W)
    g = torch.Generator(device=run.dev).manual_seed(1)
    prompts = torch.randint(0, run.cfg.vocab, (R, CTX), device=run.dev, generator=g)
    lens = torch.full((R,), CTX, dtype=torch.int32, device=run.dev)
    with torch.no_grad():
        run.capture_beam()
        run.capture()
        run.beam_start(prompts, lens, chunk=CHUNK)
        ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)] for _ in range(2)]
        for i in range(steps):
            for f, e in zip((run.beam_step, run.step), ev):
                e[i][0].record()
                f()
                e[i][1].record()
        torch.cuda.synchronize()
        beam_ms, greedy_ms = (_median([a.elapsed_time(b) for a, b in e]) for e in ev)
        live = int(run.b_live.sum())
        done = int(run.b_done.sum())
        rb, rows = _reorder_bytes(run)
        logits = run.last_logits
        k = {"logprobs_rows_us": _graph_time(lambda: backend.logprobs_rows(logits, run.tokens_in, 2 * W, run.b_logprob, run.b_top_ids,
                                                                          run.b_top_logprobs))}
        k["beam_select_us"], k["beam_select_done_requests_after"] = _select_time(run)
        k["beam_reorder_us"] = _graph_time(lambda: backend.beam_reorder(run.block_tables, run.b_parent, run.context_lens, run.s_prompt_lens,
                                                                        run.tokens_in, run.s_history, W, run.Hkv, 64, run.size_per_token,
                                                                        run.kv_bits == 4))
    out = {"requests": R, "beam_width": W, "batch": B, "layers": layers, "prompt": CTX, "new_tokens": NEW, "steps": steps,
           "beam_step_ms": beam_ms, "greedy_step_ms": greedy_ms, "ratio": beam_ms / greedy_ms, "live_slots_at_end": live, "done_requests_at_end": done,
           "reorder_rows_moved": rows, "reorder_bytes": rb, **k}
    out["reorder_GBps"] = rb / (k["beam_reorder_us"] * 1e3)
    del run
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--layers", type=int, default=32)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"device": _device_info(), "configs": [bench(R, W, a.steps, a.layers) for R, W in CONFIGS]}
    with open(os.path.join(a.out, "beam_search_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
