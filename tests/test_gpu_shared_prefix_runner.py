"""GPU: DecodeRunner(shared_prefix=True) -- fork records groups, the plain step attends through shared_prefix_decode_attention.

The measured routing rule sends only long shared prefixes to the op; these tests lower its page threshold to 1 so that the op runs on the
tiny model's short prompts.  Tolerance against the runner without the flag (same seed, same calls): the attention differs only in its fp32
summation order, which the per-token INT8 requantisation of every later layer amplifies: the first step's logits agree to
max |a - b| <= 5e-2 * max(1, max |b|) (seen on an H100: 0.122 at max |b| about 4; rows outside groups agree bit for bit), and layer-0 pages are
byte-identical (layer 0 appends the same k / v with the decode kernel's code).  Later steps are not compared: on the random tiny model a last-bit difference can flip
a near-tied greedy token, and the trajectories then part.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
B, CTX = 8, 200


@pytest.fixture(autouse=True)
def _route_short_prefixes(monkeypatch):
    from qserve_b200 import decode
    monkeypatch.setattr(decode, "SHARED_PREFIX_MIN_PAGES", 1)


def _runner(dev, **kw):
    from qserve_b200.decode import DecodeRunner

    return DecodeRunner("tiny", "w4a8kv4", batch=B, ctx=CTX, device=dev, seed=3, prompt_tokens=B * CTX, max_new_tokens=80, generate=True, **kw)


def _prompts(dev, lens, seed=13):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 1024, (B, CTX), device=dev, generator=g), torch.tensor(lens, dtype=torch.int32, device=dev)


def _own_pages(run, b, n_blocks):
    return torch.cat([pool[b * run.blocks_per_seq + j] for li in range(run.L) for pool in (run.kpools[li], run.vpools[li]) for j in range(n_blocks)])


def test_fork_children_follow_the_parent(dev):
    lens = [193, 150, 1, 1, 1, 130, 1, 1]
    with torch.no_grad():
        run = _runner(dev, shared_prefix=True)
        prompts, lens_d = _prompts(dev, lens)
        run.prefill(prompts, lens_d)
        snap = _own_pages(run, 0, 3)
        run.fork(0, [2, 3, 4])
        run.fork(5, [6])
        assert run.sp_groups == [((0, 2, 3, 4), 3), ((5, 6), 2)] and run._sp_layout is not None
        run.generate_forward(1)
        for c in (2, 3, 4):
            assert torch.equal(run.last_logits[c], run.last_logits[0]), f"child {c}: logits differ from the parent's"
        assert torch.equal(run.last_logits[6], run.last_logits[5])
        for _ in range(69):  # 193 + 70 crosses the page boundary at 256
            run.generate_forward(1)
        for c in (2, 3, 4):
            assert torch.equal(run.s_history[c], run.s_history[0]), f"greedy child {c} left its parent"
        assert torch.equal(_own_pages(run, 0, 3), snap), "a child wrote into the parent's pages"
        run.prefill(prompts, lens_d)
        assert run.sp_groups == [] and run._sp_layout is None and torch.equal(run.block_tables, run.own_tables)


def test_matches_the_runner_without_the_flag(dev):
    lens = [193, 150, 1, 1, 1, 130, 1, 1]
    with torch.no_grad():
        runs = [_runner(dev, shared_prefix=f) for f in (False, True)]
        logits, pages = [], []
        for run in runs:
            prompts, lens_d = _prompts(dev, lens)
            run.prefill(prompts, lens_d)
            run.fork(0, [2, 3, 4])
            run.fork(5, [6, 7])
            run.generate_forward(1)
            logits.append(run.last_logits.float().clone())
            pages.append((run.kpools[0].clone(), run.vpools[0].clone()))
        a, b = logits
        assert torch.isfinite(a).all()
        assert torch.equal(a[1], b[1]), "a row outside every group changed"
        tol = 5e-2 * max(1.0, b.abs().max().item())
        assert (a - b).abs().max().item() <= tol, (a - b).abs().max().item()
        assert torch.equal(pages[0][0], pages[1][0]) and torch.equal(pages[0][1], pages[1][1]), "layer-0 pages differ"


def test_flag_changes_nothing_else(dev):
    with torch.no_grad():
        runs = [_runner(dev, shared_prefix=f) for f in (False, True)]
        assert all(torch.equal(a, b) for a, b in zip(runs[0].kpools + runs[0].vpools, runs[1].kpools + runs[1].vpools))
        assert torch.equal(runs[0].embed, runs[1].embed) and torch.equal(runs[0].lm_head, runs[1].lm_head)
        g = torch.Generator(device=dev).manual_seed(21)
        toks = torch.randint(0, 1024, (B,), device=dev, generator=g)
        out = []
        for run in runs:
            t = run.forward(toks)
            lg = run.last_logits.clone()
            run.capture()
            run.tokens_in.copy_(toks)
            run.step()
            out.append((t, lg, run.tokens_out.clone(), run.kpools[0].clone()))
        for x, y in zip(*out):
            assert torch.equal(x, y)


def test_captured_equals_eager_and_stale_replay_raises(dev):
    lens = [193, 150, 1, 1, 1, 130, 1, 1]
    with torch.no_grad():
        runs = [_runner(dev, shared_prefix=True) for _ in range(2)]
        for run in runs:
            prompts, lens_d = _prompts(dev, lens)
            run.prefill(prompts, lens_d)
            run.fork(0, [2, 3, 4])
        eager, graph = runs
        graph.capture_generate(1)
        # the warm-up advanced the graph runner: start both again from the same prompt state
        for run in runs:
            run.prefill(prompts, lens_d)
            run.fork(0, [2, 3, 4])
        for _ in range(6):
            eager.generate_forward(1)
            graph.generate_step(1)
        assert torch.equal(eager.s_history, graph.s_history) and torch.equal(eager.context_lens, graph.context_lens)
        graph.capture()
        graph.step()
        # another layout plan: the old captures are not replayed
        graph.fork(5, [6, 7])
        with pytest.raises(KeyError):
            graph.generate_step(1)
        with pytest.raises(RuntimeError):
            graph.step()
        with pytest.raises(KeyError):
            graph.step((False, False, 0))
