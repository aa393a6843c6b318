"""GPU: every step kind of the decode runner reproduces pinned output bits (tests/golden/runner_steps.npz).

The tiny model (vocab 1024) at three precisions runs each step kind from fixed seeds: the greedy decode step (eager and graph replay),
the sampled step, the step with penalties and log-probabilities, the chain verify (eager and replayed), the greedy and sampled tree verify
with their acceptance and KV compaction, the generation loop (plain and prompt-lookup steps, greedy and sampled, eager and captured), one
tensor-parallel rank's fused step with tp_exact on and off, and the reference op sequence.  Tokens, logits, sampler state and acceptance
results are compared with torch.equal, and the KV pools by SHA-256 digest: a change to the runner that is meant to keep the arithmetic
must keep every one of them."""
import contextlib
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "runner_steps.npz")
PRECISIONS = ("w4a8kv4", "w4a8kv4-g128", "w8a8kv8")
B, CTX, V = 4, 100, 1024


def _digest(pools) -> np.ndarray:
    h = hashlib.sha256()
    for p in pools:
        h.update(p.cpu().numpy().tobytes())
    return np.frombuffer(h.digest(), np.uint8).copy()


def _sampling(run, temperature=0.8, top_k=-1, top_p=0.9):
    run.s_temperature.fill_(temperature); run.s_top_k.fill_(top_k); run.s_top_p.fill_(top_p)


def runner_step_outputs(dev, precision, around=lambda name: contextlib.nullcontext()):
    """name -> CPU tensor of every pinned output.  around(name) wraps one eager step of each kind (the golden generator records the
    kernels it launches)."""
    from qserve_b200.decode import DecodeRunner

    out = {}

    def put(name, t):
        out[name] = t.detach().cpu().clone()

    def pools(name, run):
        out[name] = torch.from_numpy(_digest(run.kpools + run.vpools + run.kpools_gen + run.vpools_gen))

    g = torch.Generator(device=dev).manual_seed(17)
    ids = lambda shape, hi=V: torch.randint(0, hi, shape, device=dev, generator=g)
    with torch.no_grad():
        # ---- decode: greedy (eager, replayed), sampled, penalties + logprobs (eager, replayed) ------------------------------------------
        run = DecodeRunner("tiny", precision, batch=B, ctx=CTX, device=dev, seed=1, max_new_tokens=8)
        run.tokens_in.copy_(ids((B,)))
        with around("decode_greedy"):
            put("decode_greedy", run.forward(run.tokens_in))
        put("decode_logits", run.last_logits)
        out["decode_launches"] = torch.tensor(run.launches_per_step)
        run.capture()
        run.tokens_out.zero_()
        run.step()
        put("decode_graph", run.tokens_out)
        _sampling(run)
        with around("decode_sampled"):
            put("decode_sampled", run.forward(run.tokens_in, sample=True))
        put("decode_sampled_offsets", run.s_offsets)
        run.s_history[:, :CTX].copy_(ids((B, CTX), 64))
        run.s_history[:, 0] = run.tokens_in  # the step's own argmax is likely penalised
        run.s_repetition.copy_(torch.tensor([1.3, 1.0, 0.8, 1.1], device=dev))
        run.s_presence.copy_(torch.tensor([0.5, 0.0, -1.0, 0.2], device=dev))
        run.s_frequency.copy_(torch.tensor([0.2, 0.0, 1.5, 0.1], device=dev))
        _sampling(run, 0.0, -1, 1.0)
        with around("decode_penalties_logprobs"):
            put("decode_penalties_tokens", run.forward(run.tokens_in, penalties=True, logprobs=5))
        put("decode_penalties_logits", run.last_logits)
        put("decode_penalties_logprob", run.s_logprob)
        put("decode_penalties_top_ids", run.top_logprobs_view(5)[0])
        put("decode_penalties_top_logprobs", run.top_logprobs_view(5)[1])
        _sampling(run)
        run.capture(sample=True, penalties=True, logprobs=5)
        run.step((True, True, 5))
        put("decode_penalties_graph", run.tokens_out)
        put("decode_penalties_graph_logprob", run.s_logprob)
        put("decode_penalties_graph_top_ids", run.top_logprobs_view(5)[0])
        put("decode_penalties_graph_top_logprobs", run.top_logprobs_view(5)[1])
        put("decode_s_history", run.s_history)
        put("decode_s_seq_lens", run.s_seq_lens)
        put("decode_s_offsets", run.s_offsets)
        pools("decode_pools", run)
        del run

        # ---- verify: chain (eager, replayed), a decode step on the same runner, greedy and sampled tree ----------------------------------
        n = 4
        run = DecodeRunner("tiny", precision, batch=B, ctx=CTX, device=dev, seed=2, verify_len=n, max_new_tokens=8)
        drafts = ids((B, n))
        with around("verify_chain"):
            put("verify_chain", run.verify_forward(drafts))
        put("verify_chain_logits", run.last_verify_logits)
        run.v_tokens_in.copy_(ids((B, n)))
        run.capture_verify(n)
        run.verify_step(n)
        put("verify_chain_graph", run.v_tokens_out)
        put("verify_chain_graph_logits", run.last_verify_logits)
        run.tokens_in.copy_(drafts[:, 0])
        put("verify_then_decode", run.forward(run.tokens_in))
        put("verify_then_decode_logits", run.last_logits)
        mask = torch.tensor([0, 1, 1, 3], dtype=torch.int32, device=dev).repeat(B, 1)  # 0 -> {1, 2}, 1 -> 3
        first = run.verify_forward(drafts, tree_mask=mask)
        drafts[:, 1] = first[:, 0]  # node 1 is accepted, so the compaction moves a path of two or more
        with around("verify_tree_greedy"):
            target = run.verify_forward(drafts, tree_mask=mask)
            run.accept_and_compact(drafts, mask, target)
        put("verify_tree_target", target)
        put("verify_tree_logits", run.last_verify_logits)
        put("verify_tree_accept_len", run.v_accept_len)
        put("verify_tree_path", run.v_path)
        put("verify_tree_bonus", run.v_bonus)
        pools("verify_tree_pools", run)
        _sampling(run)
        with around("verify_tree_sampled"):
            logits = run.verify_forward(drafts, return_logits=True, tree_mask=mask)
            run.accept_sampled_and_compact(drafts, mask, logits)
        put("verify_sampled_logits", logits)
        put("verify_sampled_accept_len", run.v_accept_len)
        put("verify_sampled_path", run.v_path)
        put("verify_sampled_bonus", run.v_bonus)
        run.v_tokens_in.copy_(drafts)
        run.v_tree_mask.copy_(mask)
        run.capture_verify(n, tree=True, sampled=True, draft_probs=True)
        run.draft_probs_view(n).copy_(torch.softmax(torch.randn((B, n, V), device=dev, generator=g), dim=-1))
        run.verify_step(n, tree=True, sampled=True, draft_probs=True)
        put("verify_sampled_q_accept_len", run.v_accept_len)
        put("verify_sampled_q_path", run.v_path)
        put("verify_sampled_q_bonus", run.v_bonus)
        put("verify_s_offsets", run.s_offsets)
        pools("verify_pools", run)
        del run

        # ---- generation: plain (n = 1) and prompt-lookup (n = 4, two branches), greedy and sampled, eager and captured --------------
        run = DecodeRunner("tiny", precision, batch=B, ctx=CTX, device=dev, seed=3, verify_len=n, max_new_tokens=12, generate=True)
        prompt = ids((B, CTX + 1), 16)  # a small alphabet: the n-gram drafter finds matches
        run.g_budget.copy_(torch.tensor([12, 5, 12, 12], dtype=torch.int32, device=dev))
        for steps, branches, sampled in ((1, 1, False), (1, 1, True), (4, 2, False), (4, 2, True)):
            tag = f"generate_n{steps}_{'sampled' if sampled else 'greedy'}"
            _sampling(run)
            for captured in (False, True):
                if captured:
                    run.reset_generation(prompt)
                    run.capture_generate(steps, branches, sampled=sampled)
                run.reset_generation(prompt)
                run.s_offsets.zero_()
                for i in range(3):
                    if captured:
                        run.generate_step(steps, branches, sampled=sampled)
                    else:
                        with around(tag) if i == 0 else contextlib.nullcontext():
                            run.generate_forward(steps, branches, sampled=sampled)
                key = tag + ("_graph" if captured else "")
                put(key + "_s_history", run.s_history)
                put(key + "_s_seq_lens", run.s_seq_lens)
                put(key + "_g_finished", run.g_finished)
                put(key + "_tokens_in", run.tokens_in)
                put(key + "_context_lens", run.context_lens)
                put(key + "_logits", run.last_logits if steps == 1 else run.last_verify_logits)
                pools(key + "_pools", run)
        del run

        # ---- one tensor-parallel rank's fused step on one GPU, tp_exact off and on ---------------------------------------------------
        for exact in (False, True):
            tag = f"tp_exact{int(exact)}"
            run = DecodeRunner("tiny", precision, batch=B, ctx=CTX, device=dev, seed=4, tp_rank=1, tp_size=2, no_comm=True, tp_exact=exact)
            run.tokens_in.copy_(ids((B,)))
            with around(tag):
                put(tag, run.forward(run.tokens_in))
            put(tag + "_logits", run.last_logits)
            out[tag + "_launches"] = torch.tensor(run.launches_per_step)
            run.capture()
            run.step()
            put(tag + "_graph", run.tokens_out)
            pools(tag + "_pools", run)
            del run

        # ---- the reference op sequence: greedy and sampled -------------------------------------------------------------------------
        run = DecodeRunner("tiny", precision, batch=B, ctx=CTX, device=dev, seed=5, fused=False)
        run.tokens_in.copy_(ids((B,)))
        with around("reference_greedy"):
            put("reference_greedy", run.forward(run.tokens_in))
        put("reference_logits", run.last_logits)
        out["reference_launches"] = torch.tensor(run.launches_per_step)
        _sampling(run)
        with around("reference_sampled"):
            put("reference_sampled", run.forward(run.tokens_in, sample=True))
        pools("reference_pools", run)
        del run
    torch.cuda.synchronize()
    return out


def _as_numpy(t: torch.Tensor) -> np.ndarray:
    return t.view(torch.int16).numpy() if t.dtype == torch.half else t.numpy()  # fp16 as its bits


@pytest.mark.parametrize("precision", PRECISIONS)
def test_runner_steps_reproduce_the_pinned_bits(dev, precision):
    golden = np.load(GOLDEN)
    got = runner_step_outputs(dev, precision)
    want = {k.split(".", 1)[1]: golden[k] for k in golden.files if k.startswith(precision + ".")}
    assert sorted(got) == sorted(want)
    for k, t in got.items():
        assert torch.equal(torch.from_numpy(_as_numpy(t)), torch.from_numpy(want[k])), f"{precision}: {k} differs from the pinned bits"
