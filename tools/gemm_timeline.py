#!/usr/bin/env python
"""Per-CTA phase timeline of the decode GEMM (Llama-3-8B, M = 64) from the kernel's %globaltimer stamps (qs_gemm_set_profile_buffer).

For each of the four decode shapes: the number of waves (CTAs that enter only after the first CTA has exited ran in a later wave), CTAs
per SM, the planned tokens per tile and split, and the median per-CTA phase times: entry -> first stage on chip, PDL wait, mainloop (and
per 256-K stage), epilogue up to the issue of the split-K bulk copies (staging the partials, row loads and the ring-drain cluster barrier
included), the wait for the peers' partials, the finish.  A profiled launch prints its plan, with the occupancy API's answer for it, on
stderr (qs_gemm_plan ... resident_clusters=N).

  python tools/gemm_timeline.py [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qserve_b200._lib import lib  # noqa: E402
from qserve_b200.decode import DecodeRunner  # noqa: E402

# stamp slots written by gemm_kernel (slots 13 / 14 / 15: tokens per tile, split, SM id)
ENTRY, PDL, FIRST_STAGE, MAIN_DONE, ROWS, PUSHED, CLUSTER, FINISHED, EXIT = 0, 2, 4, 6, 8, 9, 10, 11, 12

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--layers", type=int, default=8)
ap.add_argument("--out", default=None, help="write the summary as DIR/gemm_timeline.json")
args = ap.parse_args()

run = DecodeRunner("llama-3-8b", "w4a8kv4", 64, 1024, torch.device("cuda:0"), layers=args.layers)
run.q_scale.fill_(0.01)
run.q_sum.fill_(0.1)
ops = {"qkv": (run.q_hidden, run.qkv_buf), "o": (run.q_attn, run.out_buf), "gate_up": (run.q_hidden, run.gate_up_buf), "down": (run.q_mlp, run.out_buf)}
prof = torch.zeros(8192 * 16, dtype=torch.int64, device="cuda")
summary = {}
for name, (xq, buf) in ops.items():
    lin = run.layers[0][name]
    stages = -(-lin.K // 256)
    reps = []
    for r in range(args.reps):
        for i in range(1, args.layers):  # stream the other layers' weights first: the profiled launch reads layer 0 from HBM
            run.layers[i][name](xq, run.q_scale, run.q_sum, buf)
        torch.cuda.synchronize()
        prof.zero_()
        lib.qs_gemm_set_profile_buffer(prof.data_ptr())
        run.layers[0][name](xq, run.q_scale, run.q_sum, buf)
        torch.cuda.synchronize()
        lib.qs_gemm_set_profile_buffer(None)
        p = prof.cpu().numpy().reshape(-1, 16)
        p = p[p[:, ENTRY] > 0]
        sm = p[:, 15].copy()
        t = (p[:, :15] - p[:, ENTRY].min()).astype(np.float64) / 1e3  # us from the first CTA's entry
        ctas, nt, split = len(p), int(p[0, 13]), int(p[0, 14])
        late = int((t[:, ENTRY] > t[:, EXIT].min()).sum())
        med = lambda a, b: float(np.median(t[:, b] - t[:, a]))  # noqa: E731
        reps.append({
            "ctas": ctas, "tile_tokens": nt, "split": split, "stages_per_cta": stages / split, "ctas_after_first_exit": late, "waves": 1 if late == 0 else 2,
            "max_ctas_per_sm": int(np.bincount(sm.astype(np.int64)).max()) if sm.any() else None,
            "span_us": float(t[:, EXIT].max()), "entry_spread_us": float(t[:, ENTRY].max()),
            "entry_to_first_stage_us": med(ENTRY, FIRST_STAGE), "pdl_wait_us": med(ENTRY, PDL),
            "mainloop_us": med(FIRST_STAGE, MAIN_DONE), "mainloop_per_stage_us": med(FIRST_STAGE, MAIN_DONE) / (stages / split),
            "epilogue_push_us": med(MAIN_DONE, PUSHED), "cluster_barrier_us": med(PUSHED, CLUSTER), "finish_us": med(CLUSTER, FINISHED),
        })
    agg = {k: (float(np.median([r[k] for r in reps])) if isinstance(reps[0][k], (int, float)) and reps[0][k] is not None else reps[0][k]) for k in reps[0]}
    agg["waves_per_rep"] = [r["waves"] for r in reps]
    summary[name] = agg
    print(f"== {name:8s} N={lin.N} K={lin.K}: " + "  ".join(f"{k}={v:.2f}" if isinstance(v, float) else f"{k}={v}" for k, v in agg.items()), flush=True)
if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemm_timeline.json"), "w") as f:
        json.dump(summary, f, indent=1)
